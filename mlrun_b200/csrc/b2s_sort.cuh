// b2s_sort.cuh -- the stable LSD radix sort of 64-bit keys with a 32-bit payload that the point-in-time join (b2s_pit.cu)
// and the windowed aggregations (b2s_agg.cu) share: 8 passes of 8-bit digits, each pass histogram -> scan -> stable scatter.
// Included by one translation unit each, inside no namespace: the kernels live in that unit's anonymous namespace.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/b200serve.h"
#include "b2s_internal.h"
#include "b2s_stage.h"

namespace b2s_sort {

// A block sorts a tile of kSortThreads * kSortItems keys; element e of the tile is item e / kSortThreads of thread
// e % kSortThreads, so ranking items in (item, warp, lane) order is ranking them in input order (stability).
constexpr int kSortThreads = 256;
constexpr int kSortItems = 16;
constexpr int kSortTile = kSortThreads * kSortItems;
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kScanThreads = 1024;

// signed order: flipping the sign bit maps INT64_MIN..INT64_MAX onto 0..UINT64_MAX monotonically
__host__ __device__ inline uint32_t radix_digit(uint64_t key, int shift) {
  return (uint32_t)(((key ^ 0x8000000000000000ull) >> shift) & 0xffu);
}

}  // namespace b2s_sort

namespace {

using namespace b2s_sort;

// ---- radix sort ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kSortThreads) radix_hist_kernel(const uint64_t* __restrict__ keys, int64_t n, int shift,
                                                                  uint32_t* __restrict__ hist, int n_blocks) {
  __shared__ uint32_t s_hist[256];
  s_hist[threadIdx.x] = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * kSortTile;
#pragma unroll 4
  for (int j = 0; j < kSortItems; ++j) {
    const int64_t e = base + (int64_t)j * kSortThreads + threadIdx.x;
    if (e < n) atomicAdd(&s_hist[radix_digit(keys[e], shift)], 1u);
  }
  __syncthreads();
  hist[(int64_t)threadIdx.x * n_blocks + blockIdx.x] = s_hist[threadIdx.x];  // digit-major: the scan yields global offsets
}

// exclusive scan of m counters in place, one block (m = 256 * n_blocks is a few hundred thousand at most)
__global__ void __launch_bounds__(kScanThreads) radix_scan_kernel(uint32_t* __restrict__ v, int64_t m) {
  __shared__ uint32_t s_sum[kScanThreads];
  const int64_t chunk = (m + kScanThreads - 1) / kScanThreads;
  const int64_t b = threadIdx.x * chunk, e = (b + chunk < m) ? b + chunk : m;
  uint32_t sum = 0;
  for (int64_t i = b; i < e; ++i) sum += v[i];
  s_sum[threadIdx.x] = sum;
  __syncthreads();
  for (int off = 1; off < kScanThreads; off <<= 1) {  // Hillis-Steele over the per-thread sums
    const uint32_t add = threadIdx.x >= off ? s_sum[threadIdx.x - off] : 0u;
    __syncthreads();
    s_sum[threadIdx.x] += add;
    __syncthreads();
  }
  uint32_t run = s_sum[threadIdx.x] - sum;
  for (int64_t i = b; i < e; ++i) {
    const uint32_t c = v[i];
    v[i] = run;
    run += c;
  }
}

__global__ void __launch_bounds__(kSortThreads) radix_scatter_kernel(const uint64_t* __restrict__ kin, const uint32_t* __restrict__ vin,
                                                                     uint64_t* __restrict__ kout, uint32_t* __restrict__ vout,
                                                                     int64_t n, int shift, const uint32_t* __restrict__ hist, int n_blocks) {
  __shared__ uint32_t s_base[256];              // next free output position of each digit for this block
  __shared__ uint32_t s_warp[kSortWarps][256];  // per item: count, then first position, of each digit per warp
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  s_base[tid] = hist[(int64_t)tid * n_blocks + blockIdx.x];
  const unsigned lt_mask = (1u << lane) - 1u;
  const int64_t base = (int64_t)blockIdx.x * kSortTile;
  for (int j = 0; j < kSortItems; ++j) {
#pragma unroll
    for (int w = 0; w < kSortWarps; ++w) s_warp[w][tid] = 0;
    __syncthreads();
    const int64_t e = base + (int64_t)j * kSortThreads + tid;
    const bool valid = e < n;
    uint64_t k = 0;
    uint32_t d = 256;  // out-of-range items form their own group and are never stored
    if (valid) {
      k = kin[e];
      d = radix_digit(k, shift);
    }
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const unsigned rank = __popc(peers & lt_mask);
    if (valid && rank == 0) s_warp[warp][d] = __popc(peers);
    __syncthreads();
    {  // thread tid owns digit tid: warp counts -> positions, in warp order
      uint32_t run = s_base[tid];
#pragma unroll
      for (int w = 0; w < kSortWarps; ++w) {
        const uint32_t c = s_warp[w][tid];
        s_warp[w][tid] = run;
        run += c;
      }
      s_base[tid] = run;
    }
    __syncthreads();
    if (valid) {
      const uint32_t pos = s_warp[warp][d] + rank;
      kout[pos] = k;
      vout[pos] = vin ? vin[e] : (uint32_t)e;  // no payload: the input position
    }
    __syncthreads();
  }
}

// the sort's buffers, allocated on stream st and freed on it when they leave scope
struct SortBufs {
  explicit SortBufs(cudaStream_t s) : st(s) {}
  SortBufs(const SortBufs&) = delete;
  SortBufs& operator=(const SortBufs&) = delete;
  ~SortBufs() {
    for (int i = 0; i < 2; ++i) {
      if (k[i]) cudaFreeAsync(k[i], st);
      if (v[i]) cudaFreeAsync(v[i], st);
    }
    if (hist) cudaFreeAsync(hist, st);
  }
  int alloc(int64_t n) {
    const int64_t n_blocks = (n + kSortTile - 1) / kSortTile;
    for (int i = 0; i < 2; ++i) {
      B2S_CUDA_TRY(cudaMallocAsync(&k[i], n * 8, st));
      B2S_CUDA_TRY(cudaMallocAsync(&v[i], n * 4, st));
    }
    B2S_CUDA_TRY(cudaMallocAsync(&hist, n_blocks * 256 * 4, st));
    return B2S_OK;
  }

  cudaStream_t st;
  uint64_t* k[2] = {};
  uint32_t* v[2] = {};
  uint32_t* hist = nullptr;
};

// stable sort of k[0] (signed 64-bit keys) carrying v[0] (null: the payload is the input position); the result ends in
// k[0] / v[0] (an even number of passes)
int radix_sort(SortBufs& b, bool payload, int64_t n, Launches& launches) {
  const int n_blocks = (int)((n + kSortTile - 1) / kSortTile);
  const cudaStream_t st = b.st;
  for (int pass = 0; pass < 8; ++pass) {
    const int src = pass & 1, shift = pass * 8;
    radix_hist_kernel<<<n_blocks, kSortThreads, 0, st>>>(b.k[src], n, shift, b.hist, n_blocks);
    radix_scan_kernel<<<1, kScanThreads, 0, st>>>(b.hist, (int64_t)n_blocks * 256);
    radix_scatter_kernel<<<n_blocks, kSortThreads, 0, st>>>(b.k[src], (pass == 0 && !payload) ? nullptr : b.v[src], b.k[src ^ 1],
                                                            b.v[src ^ 1], n, shift, b.hist, n_blocks);
  }
  launches.add(24);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return b2s_int_fail(B2S_ERR_CUDA, "radix sort launch failed: %s", cudaGetErrorString(e));
  return B2S_OK;
}

// the n signed keys at d_keys (device memory) in order: b.k[0] ends as the sorted keys, b.v[0] as their input positions
int sort_keys(SortBufs& b, const int64_t* d_keys, int64_t n, Launches& launches) {
  if (int rc = b.alloc(n)) return rc;
  B2S_CUDA_TRY(cudaMemcpyAsync(b.k[0], d_keys, n * 8, cudaMemcpyDeviceToDevice, b.st));
  return radix_sort(b, false, n, launches);
}

}  // namespace
