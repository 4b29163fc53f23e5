// ring_tsan.cpp -- ThreadSanitizer harness for the host side of the coalescing ring (b2s_submit / b2s_wait / b2s_flush,
// the dispatcher thread) with b2s_run_host running beside it.  Built against a -fsanitize=thread build of the library
// (every unit of mlrun_b200/csrc compiled with `nvcc -gencode arch=compute_90a,code=sm_90a -O1 -g -std=c++17
// -Xcompiler -fPIC,-fsanitize=thread`, linked with -ltsan), then `g++ -std=c++17 -O1 -g -fsanitize=thread ring_tsan.cpp
// -lb200serve_tsan -lcudart -lpthread`; run on a GPU machine:  TSAN_OPTIONS="halt_on_error=0" ./ring_tsan
// Every result is also checked against a single-threaded b2s_run_host of the same rows.
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <thread>
#include <vector>

#include "../../include/b200serve.h"

#define CK(x)                                                                  \
  do {                                                                         \
    int rc_ = (x);                                                             \
    if (rc_) {                                                                 \
      fprintf(stderr, "%s -> %d: %s\n", #x, rc_, b2s_last_error());            \
      exit(2);                                                                 \
    }                                                                          \
  } while (0)

int main(int argc, char** argv) {
  const double seconds = argc > 1 ? atof(argv[1]) : 3.0;
  const int n_threads = argc > 2 ? atoi(argv[2]) : 16;
  const int F = 64, N = 8192;
  CK(b2s_init(0, nullptr));
  b2s_plan_t plan;
  CK(b2s_plan_create(F, &plan));
  std::mt19937 rng(1);
  std::normal_distribution<double> nd;
  std::vector<double> W(4 * F), b(4);
  for (auto& w : W) w = nd(rng);
  for (auto& v : b) v = nd(rng);
  for (int m = 0; m < 4; ++m) CK(b2s_plan_add_linear_model(plan, W.data() + m * F, b.data() + m, 1, B2S_LINK_IDENTITY, nullptr, 0));
  const double vw[4] = {0.25, 0.25, 0.25, 0.25};
  CK(b2s_plan_set_vote(plan, B2S_VOTE_MEAN, vw, 4));
  CK(b2s_plan_finalize(plan));
  std::vector<float> X((size_t)N * F);
  for (auto& v : X) v = (float)nd(rng);
  std::vector<float> want(N);
  CK(b2s_run_host(plan, X.data(), N, F * 4, want.data(), N * 4, nullptr, nullptr));

  std::atomic<long long> rows{0}, mismatches{0};
  const auto t_end = std::chrono::steady_clock::now() + std::chrono::duration_cast<std::chrono::steady_clock::duration>(std::chrono::duration<double>(seconds));
  std::vector<std::thread> threads;
  for (int t = 0; t < n_threads; ++t)
    threads.emplace_back([&, t] {
      std::mt19937 r(100 + t);
      std::vector<float> out(512);
      std::vector<int32_t> status(512);
      while (std::chrono::steady_clock::now() < t_end) {
        const int n = 1 + (int)(r() % 64), off = (int)(r() % (N - 64));
        if (t == 0 && (r() % 7) == 0) {  // the synchronous host path beside the ring
          CK(b2s_run_host(plan, X.data() + (size_t)off * F, n, F * 4, out.data(), n * 4, status.data(), nullptr));
        } else {
          uint64_t ticket = 0;
          CK(b2s_submit(plan, X.data() + (size_t)off * F, n, F * 4, &ticket));
          if ((r() % 5) == 0) CK(b2s_flush(plan));
          CK(b2s_wait(plan, ticket, out.data(), n * 4, status.data(), nullptr));
        }
        for (int i = 0; i < n; ++i)
          if (out[i] != want[off + i]) ++mismatches;
        rows += n;
      }
    });
  for (auto& th : threads) th.join();
  CK(b2s_plan_destroy(plan));
  CK(b2s_shutdown());
  printf("ring_tsan: %d threads, %.1f s, %lld rows served, %lld mismatches\n", n_threads, seconds, rows.load(), mismatches.load());
  return mismatches ? 1 : 0;
}
