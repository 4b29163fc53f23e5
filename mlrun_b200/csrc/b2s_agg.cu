// b2s_agg.cu -- per-entity time-window aggregations at feature-set ingest, sm_90a.
//
// Replaces storey.AggregateByKey as FeatureSet.add_aggregation places it in a feature set's graph (mlrun/feature_store/
// feature_set.py:715-851), emitting every event: each row gains, per (operation, window), the aggregate over the earlier
// rows of its key (itself included) whose timestamps fall in the row's window.  Rows are radix-sorted by key (stable: each
// key's rows are contiguous and still in input order, b2s_sort.cuh); one prep kernel gathers the timestamps and source
// values into that order, records each row's key-run start and counts the rows the semantics refuse.  With times sorted
// inside a run, a row's window is the contiguous range [lo, i] of sorted positions, lo found by binary search.  Range
// reduces come from a hierarchy of 32-wide blocks (prefix and suffix combines per block from warp scans; block totals form
// the next level): a range is suffix + middle + prefix, or a loop of at most 32 inside one block, so the work per row is
// bounded by the number of levels whatever the window length, and no sum is ever a difference of prefix sums.
// Bound: HBM, a few dozen 8-byte reads per (row, window) and one 8-byte write per output value.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <exception>
#include <vector>

#include "../../include/b200serve.h"
#include "b2s_internal.h"
#include "b2s_sort.cuh"
#include "b2s_stage.h"

namespace {

constexpr int kAllOps = (1 << 10) - 1;
constexpr int kMaxWindows = 16;    // per aggregation
constexpr int kMaxSpecs = 64;      // aggregations per call
constexpr int kMaxSources = 16;    // distinct source columns per call
constexpr int kMaxLevels = 8;      // n < 2^32: at most 7 levels hold more than one block
constexpr int kThreads = 256;

// monoid fields (a field is stored only when an operation of the column needs it)
enum Field { F_SUM = 0, F_SQR, F_MIN, F_MAX, F_MEAN, F_M2, kFields };

int fields_of(uint32_t ops) {
  int f = 0;
  if (ops & (B2S_AGG_SUM | B2S_AGG_AVG)) f |= 1 << F_SUM;
  if (ops & B2S_AGG_SQR) f |= 1 << F_SQR;
  if (ops & B2S_AGG_MIN) f |= 1 << F_MIN;
  if (ops & B2S_AGG_MAX) f |= 1 << F_MAX;
  if (ops & (B2S_AGG_STDVAR | B2S_AGG_STDDEV)) f |= (1 << F_MEAN) | (1 << F_M2);
  return f;
}

struct Mono {
  double c, s, q, mn, mx, mean, m2;
};

__device__ __forceinline__ Mono mono_empty() { return Mono{0.0, 0.0, 0.0, INFINITY, -INFINITY, 0.0, 0.0}; }
__device__ __forceinline__ Mono mono_leaf(double x) { return Mono{1.0, x, x * x, x, x, x, 0.0}; }

// (count, mean, M2) by Chan et al.'s pairwise update: no n * sum(x^2) - sum(x)^2 cancellation
__device__ __forceinline__ Mono combine(const Mono& a, const Mono& b) {
  if (a.c == 0.0) return b;
  if (b.c == 0.0) return a;
  Mono r;
  r.c = a.c + b.c;
  r.s = a.s + b.s;
  r.q = a.q + b.q;
  r.mn = fmin(a.mn, b.mn);
  r.mx = fmax(a.mx, b.mx);
  const double d = b.mean - a.mean;
  r.mean = a.mean + d * (b.c / r.c);
  r.m2 = a.m2 + b.m2 + d * d * (a.c * b.c / r.c);
  return r;
}

__device__ __forceinline__ Mono shfl_mono(const Mono& v, int src, bool up) {
  Mono r;
  r.c = up ? __shfl_up_sync(0xffffffffu, v.c, src) : __shfl_down_sync(0xffffffffu, v.c, src);
  r.s = up ? __shfl_up_sync(0xffffffffu, v.s, src) : __shfl_down_sync(0xffffffffu, v.s, src);
  r.q = up ? __shfl_up_sync(0xffffffffu, v.q, src) : __shfl_down_sync(0xffffffffu, v.q, src);
  r.mn = up ? __shfl_up_sync(0xffffffffu, v.mn, src) : __shfl_down_sync(0xffffffffu, v.mn, src);
  r.mx = up ? __shfl_up_sync(0xffffffffu, v.mx, src) : __shfl_down_sync(0xffffffffu, v.mx, src);
  r.mean = up ? __shfl_up_sync(0xffffffffu, v.mean, src) : __shfl_down_sync(0xffffffffu, v.mean, src);
  r.m2 = up ? __shfl_up_sync(0xffffffffu, v.m2, src) : __shfl_down_sync(0xffffffffu, v.m2, src);
  return r;
}

// one source column's range structure.  Level 0 has m[0] = n elements (the rows in sorted order, x); level L + 1 has one
// element per 32-wide block of level L, whose value is that block's total.  pre[L][f] / suf[L][f]: field f of the combine
// of element e's block from its start to e / from e to its end, stored for the n_levels levels with more than one block.
struct Tree {
  const double* x;
  int64_t n;
  int32_t n_levels;
  int32_t fields;
  int64_t m[kMaxLevels + 1];
  double* pre[kMaxLevels][kFields];
  double* suf[kMaxLevels][kFields];
};

// leaves (level-0 rows) under elements [a, b] of level L
__device__ __forceinline__ double leaves(const Tree& t, int L, int64_t a, int64_t b) {
  const int64_t hi = min((b + 1) << (5 * L), t.n);
  return (double)(hi - (a << (5 * L)));
}

__device__ __forceinline__ Mono load(double* const* arr, int fields, int64_t e, double c) {
  Mono r{c, 0.0, 0.0, INFINITY, -INFINITY, 0.0, 0.0};
  if (fields & (1 << F_SUM)) r.s = arr[F_SUM][e];
  if (fields & (1 << F_SQR)) r.q = arr[F_SQR][e];
  if (fields & (1 << F_MIN)) r.mn = arr[F_MIN][e];
  if (fields & (1 << F_MAX)) r.mx = arr[F_MAX][e];
  if (fields & (1 << F_MEAN)) {
    r.mean = arr[F_MEAN][e];
    r.m2 = arr[F_M2][e];
  }
  return r;
}

__device__ __forceinline__ void store(double* const* arr, int fields, int64_t e, const Mono& v) {
  if (fields & (1 << F_SUM)) arr[F_SUM][e] = v.s;
  if (fields & (1 << F_SQR)) arr[F_SQR][e] = v.q;
  if (fields & (1 << F_MIN)) arr[F_MIN][e] = v.mn;
  if (fields & (1 << F_MAX)) arr[F_MAX][e] = v.mx;
  if (fields & (1 << F_MEAN)) {
    arr[F_MEAN][e] = v.mean;
    arr[F_M2][e] = v.m2;
  }
}

// element e of level L as a monoid: a row (L = 0) or the total of block e of level L - 1 (its suffix from the block start)
__device__ __forceinline__ Mono element(const Tree& t, int L, int64_t e) {
  if (L == 0) return mono_leaf(t.x[e]);
  return load(t.suf[L - 1], t.fields, e << 5, leaves(t, L, e, e));
}

// combine of rows [lo, hi]: at each level the partial blocks at either end come from one suffix and one prefix, and the
// whole blocks between them form a range of the next level; a range inside one block is looped (<= 32 elements)
__device__ Mono range_reduce(const Tree& t, int64_t lo, int64_t hi) {
  Mono left = mono_empty(), right = mono_empty();
  int64_t a = lo, b = hi;
  for (int L = 0;; ++L) {
    if (L >= t.n_levels || (a >> 5) == (b >> 5)) {
      for (int64_t e = a; e <= b; ++e) left = combine(left, element(t, L, e));
      break;
    }
    left = combine(left, load(t.suf[L], t.fields, a, leaves(t, L, a, a | 31)));
    right = combine(load(t.pre[L], t.fields, b, leaves(t, L, b & ~(int64_t)31, b)), right);
    a = (a >> 5) + 1;
    b = (b >> 5) - 1;
    if (a > b) break;
  }
  return combine(left, right);
}

// one warp per 32-wide block of level L: prefix and suffix combines by warp scans (elements past the end are empty)
__global__ void __launch_bounds__(kThreads) build_level_kernel(const __grid_constant__ Tree t, int L) {
  const int lane = threadIdx.x & 31;
  const int64_t m = t.m[L], blocks = (m + 31) >> 5;
  const int64_t warps = (int64_t)gridDim.x * (kThreads / 32);
  for (int64_t blk = (int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5); blk < blocks; blk += warps) {
    const int64_t e = (blk << 5) + lane;
    const Mono v = e < m ? element(t, L, e) : mono_empty();
    Mono p = v, s = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const Mono up = shfl_mono(p, off, true);
      if (lane >= off) p = combine(up, p);
      const Mono down = shfl_mono(s, off, false);
      if (lane + off < 32) s = combine(s, down);
    }
    if (e < m) {
      store(t.pre[L], t.fields, e, p);
      store(t.suf[L], t.fields, e, s);
    }
  }
}

struct PrepParams {
  const uint64_t* keys;          // [n] sorted
  const uint32_t* order;         // [n] input row at each sorted position
  const int64_t* ts;             // [n] input order
  int64_t* ts_sorted;            // [n]
  int64_t* run_start;            // [n]
  int64_t n;
  int32_t n_src;
  int32_t kind[kMaxSources];     // B2S_COL_F32 / B2S_COL_I32
  const void* src[kMaxSources];  // [n] input order
  double* x[kMaxSources];        // [n] sorted order, widened
  unsigned long long* counters;  // [3] out-of-order rows, NaT rows, NaN values
};

__global__ void __launch_bounds__(kThreads) prep_kernel(const __grid_constant__ PrepParams p) {
  unsigned long long late = 0, nat = 0, nan = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = p.order[i];
    const int64_t t = p.ts[r];
    const uint64_t k = p.keys[i];
    p.ts_sorted[i] = t;
    int64_t lo = 0, hi = i;  // first sorted position of this key (keys are sorted by signed value)
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if ((int64_t)p.keys[mid] < (int64_t)k) lo = mid + 1; else hi = mid;
    }
    p.run_start[i] = lo;
    nat += t == INT64_MIN;
    late += (i > lo && t < p.ts[p.order[i - 1]]);
    for (int c = 0; c < p.n_src; ++c) {
      double v;
      if (p.kind[c] == B2S_COL_I32) {
        v = (double)static_cast<const int32_t*>(p.src[c])[r];
      } else {
        v = (double)static_cast<const float*>(p.src[c])[r];
        nan += isnan(v);
      }
      p.x[c][i] = v;
    }
  }
  for (int off = 16; off; off >>= 1) {
    late += __shfl_down_sync(0xffffffffu, late, off);
    nat += __shfl_down_sync(0xffffffffu, nat, off);
    nan += __shfl_down_sync(0xffffffffu, nan, off);
  }
  if ((threadIdx.x & 31) == 0) {
    if (late) atomicAdd(&p.counters[0], late);
    if (nat) atomicAdd(&p.counters[1], nat);
    if (nan) atomicAdd(&p.counters[2], nan);
  }
}

struct ReduceParams {
  Tree t;
  const int64_t* ts;         // [n] sorted order
  const int64_t* run_start;  // [n]
  const uint32_t* order;     // [n]
  uint32_t ops;
  int32_t n_windows;
  int64_t period;            // 0: fixed windows
  int64_t window[kMaxWindows];
  double* out[10][kMaxWindows];  // [op bit][window], [n] each in input order; null where the op is not asked
};

__device__ __forceinline__ int64_t floor_div(int64_t t, int64_t p) {
  const int64_t q = t / p;
  return (t % p != 0 && t < 0) ? q - 1 : q;
}

// the first timestamp of bucket b of width p, clamped at INT64_MIN (where b * p would leave the int64 range every
// timestamp is in the window)
__device__ __forceinline__ int64_t bucket_start(int64_t b, int64_t p) {
  return b <= floor_div(INT64_MIN, p) ? INT64_MIN : b * p;
}

__global__ void __launch_bounds__(kThreads) reduce_kernel(const __grid_constant__ ReduceParams p) {
  const Tree& t = p.t;
  const bool need_reduce = t.fields != 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < t.n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t ti = p.ts[i], rs = p.run_start[i], r = p.order[i];
    for (int w = 0; w < p.n_windows; ++w) {
      int64_t start;
      if (p.period) {
        // first bucket b - back, clamped before the subtraction: at a 1 ns period it leaves the int64 range near 1677
        const int64_t b = floor_div(ti, p.period), back = p.window[w] / p.period - 1;
        start = b < INT64_MIN + back ? INT64_MIN : bucket_start(b - back, p.period);
      } else {
        start = bucket_start(floor_div(ti, p.window[w]), p.window[w]);
      }
      int64_t lo = rs, hi = i;  // first position of the run with ts >= start (row i itself qualifies)
      while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(p.ts + mid) < start) lo = mid + 1; else hi = mid;
      }
      const Mono v = need_reduce ? range_reduce(t, lo, i) : mono_empty();
      const double cnt = (double)(i - lo + 1);
#define AGG_OUT(bit, value) \
      if (double* dst = p.out[bit][w]) dst[r] = (value);
      AGG_OUT(0, cnt)
      AGG_OUT(1, v.s)
      AGG_OUT(2, v.q)
      AGG_OUT(3, v.mx)
      AGG_OUT(4, v.mn)
      AGG_OUT(5, t.x[lo])
      AGG_OUT(6, t.x[i])
      AGG_OUT(7, v.s / cnt)
      AGG_OUT(8, cnt > 1.0 ? v.m2 / (cnt - 1.0) : (double)NAN)
      AGG_OUT(9, cnt > 1.0 ? sqrt(v.m2 / (cnt - 1.0)) : (double)NAN)
#undef AGG_OUT
    }
  }
}

int n_ops(uint32_t ops) { return __builtin_popcount(ops); }

// levels of the range structure that hold more than one 32-wide block
int levels_of(int64_t n, int64_t* m) {
  int L = 0;
  m[0] = n;
  while (m[L] > 32) {
    m[L + 1] = (m[L] + 31) >> 5;
    ++L;
  }
  return L;
}

int check_specs(const void* keys, const void* ts, int64_t n, const b2s_agg_spec* specs, int32_t n_specs, const void* counters,
                std::vector<const void*>* sources) {
  if (n < 0 || n >= (1ll << 32)) return b2s_int_fail(B2S_ERR_INVALID, "n = %lld: 0 <= n < 2^32 rows (the sort's 32-bit payload)", (long long)n);
  if (n_specs < 1 || n_specs > kMaxSpecs || !specs) return b2s_int_fail(B2S_ERR_INVALID, "1 .. %d aggregations", kMaxSpecs);
  if (!counters || misaligned(counters, 8)) return b2s_int_fail(B2S_ERR_INVALID, "counters: null or not 8-byte aligned");
  if (n && (!keys || !ts)) return b2s_int_fail(B2S_ERR_INVALID, "null keys / timestamps");
  if (misaligned(keys, 8) || misaligned(ts, 8)) return b2s_int_fail(B2S_ERR_INVALID, "keys / timestamps must be 8-byte aligned");
  sources->clear();
  for (int s = 0; s < n_specs; ++s) {
    const b2s_agg_spec& d = specs[s];
    if (d.kind != B2S_COL_F32 && d.kind != B2S_COL_I32) return b2s_int_fail(B2S_ERR_INVALID, "aggregation %d: kind must be F32 or I32", s);
    if (d.ops == 0 || (d.ops & ~(uint32_t)kAllOps)) return b2s_int_fail(B2S_ERR_INVALID, "aggregation %d: empty or unknown op mask 0x%x", s, d.ops);
    if (d.n_windows < 1 || d.n_windows > kMaxWindows || !d.windows_ns || !d.outs)
      return b2s_int_fail(B2S_ERR_INVALID, "aggregation %d: 1 .. %d windows, with outputs", s, kMaxWindows);
    if (d.period_ns < 0) return b2s_int_fail(B2S_ERR_INVALID, "aggregation %d: negative period", s);
    for (int w = 0; w < d.n_windows; ++w) {
      const int64_t win = d.windows_ns[w];
      if (win <= 0) return b2s_int_fail(B2S_ERR_INVALID, "aggregation %d: window %d is not positive", s, w);
      if (d.period_ns && win % d.period_ns)
        return b2s_int_fail(B2S_ERR_INVALID, "aggregation %d: period %lld ns does not divide window %lld ns", s, (long long)d.period_ns, (long long)win);
    }
    if ((n && !d.src) || misaligned(d.src, 4)) return b2s_int_fail(B2S_ERR_INVALID, "aggregation %d: source null or not 4-byte aligned", s);
    for (int j = 0; j < n_ops(d.ops) * d.n_windows; ++j)
      if ((n && !d.outs[j]) || misaligned(d.outs[j], 8)) return b2s_int_fail(B2S_ERR_INVALID, "aggregation %d output %d: null or not 8-byte aligned", s, j);
    if (std::find(sources->begin(), sources->end(), d.src) == sources->end()) sources->push_back(d.src);
  }
  if ((int)sources->size() > kMaxSources) return b2s_int_fail(B2S_ERR_INVALID, "more than %d distinct source columns", kMaxSources);
  for (int s = 0; s < n_specs; ++s)
    for (int u = 0; u < s; ++u)
      if (specs[u].src == specs[s].src && specs[u].kind != specs[s].kind)
        return b2s_int_fail(B2S_ERR_INVALID, "aggregations %d and %d read one column as two kinds", u, s);
  return B2S_OK;
}

// everything after the checks, over device arrays
int run(const int64_t* d_keys, const int64_t* d_ts, int64_t n, const b2s_agg_spec* specs, int32_t n_specs,
        const std::vector<const void*>& sources, unsigned long long* d_counters, cudaStream_t st, Launches& launches, cudaEvent_t sorted) {
  const int ns = (int)sources.size();
  std::vector<int> fields(ns, 0);
  for (int s = 0; s < n_specs; ++s) {
    const int c = (int)(std::find(sources.begin(), sources.end(), specs[s].src) - sources.begin());
    fields[c] |= fields_of(specs[s].ops);
  }
  // the intermediates in one block: sorted timestamps, run starts, and per source its widened rows and range structure
  DeviceBlock blk(st);
  PrepParams pp{};
  pp.ts = d_ts;
  pp.n = n;
  pp.n_src = ns;
  pp.counters = d_counters;
  blk.scratch(pp.ts_sorted, (size_t)n * 8);
  blk.scratch(pp.run_start, (size_t)n * 8);
  std::vector<Tree> trees(ns);
  for (int c = 0; c < ns; ++c) {
    Tree& t = trees[c];
    t = Tree{};
    t.n = n;
    t.fields = fields[c];
    t.n_levels = levels_of(n, t.m);
    for (const b2s_agg_spec* d = specs; d < specs + n_specs; ++d)
      if (d->src == sources[c]) pp.kind[c] = d->kind;
    pp.src[c] = sources[c];
    blk.scratch(pp.x[c], (size_t)n * 8);
    for (int L = 0; L < t.n_levels; ++L)
      for (int f = 0; f < kFields; ++f) {
        if (!(t.fields & (1 << f))) continue;
        blk.scratch(t.pre[L][f], (size_t)t.m[L] * 8);
        blk.scratch(t.suf[L][f], (size_t)t.m[L] * 8);
      }
  }
  SortBufs sb(st);
  if (int rc = sort_keys(sb, d_keys, n, launches)) return rc;
  if (sorted) B2S_CUDA_TRY(cudaEventRecord(sorted, st));
  if (int rc = blk.alloc()) return rc;  // while the sort runs
  for (int c = 0; c < ns; ++c) trees[c].x = pp.x[c];
  pp.keys = sb.k[0];
  pp.order = sb.v[0];
  prep_kernel<<<grid_for(n, kThreads), kThreads, 0, st>>>(pp);
  launches.add(1);
  for (int c = 0; c < ns; ++c) {
    if (!trees[c].fields) continue;  // count / first / last only: no reduce
    for (int L = 0; L < trees[c].n_levels; ++L) {
      build_level_kernel<<<grid_for((trees[c].m[L] + 31) / 32 * 32, kThreads), kThreads, 0, st>>>(trees[c], L);
      launches.add(1);
    }
  }
  for (int s = 0; s < n_specs; ++s) {
    const b2s_agg_spec& d = specs[s];
    const int c = (int)(std::find(sources.begin(), sources.end(), d.src) - sources.begin());
    ReduceParams rp{};
    rp.t = trees[c];
    rp.t.fields = fields_of(d.ops);  // this aggregation's fields only (the column's structure may hold more)
    rp.ts = pp.ts_sorted;
    rp.run_start = pp.run_start;
    rp.order = sb.v[0];
    rp.ops = d.ops;
    rp.n_windows = d.n_windows;
    rp.period = d.period_ns;
    for (int w = 0; w < d.n_windows; ++w) rp.window[w] = d.windows_ns[w];
    int j = 0;
    for (int bit = 0; bit < 10; ++bit) {
      if (!(d.ops & (1u << bit))) continue;
      for (int w = 0; w < d.n_windows; ++w) rp.out[bit][w] = d.outs[j * d.n_windows + w];
      ++j;
    }
    reduce_kernel<<<grid_for(n, kThreads), kThreads, 0, st>>>(rp);
    launches.add(1);
  }
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return b2s_int_fail(B2S_ERR_CUDA, "aggregation launch failed: %s", cudaGetErrorString(e));
  return B2S_OK;
}

}  // namespace

extern "C" int b2s_agg_run_device(const int64_t* d_keys, const int64_t* d_ts, int64_t n, const b2s_agg_spec* specs, int32_t n_specs,
                                  uint64_t* d_counters, void* stream) {
  try {  // no C++ exception crosses the C boundary
    std::vector<const void*> sources;
    if (int rc = check_specs(d_keys, d_ts, n, specs, n_specs, d_counters, &sources)) return rc;
    if (n == 0) return B2S_OK;
    if (!b2s_int_inited()) return b2s_int_fail(B2S_ERR_STATE, "b2s_init was not called (no CUDA device: there is no CPU fallback)");
    B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
    cudaStream_t st = stream ? (cudaStream_t)stream : b2s_int_stream();
    Launches launches;
    return run(d_keys, d_ts, n, specs, n_specs, sources, reinterpret_cast<unsigned long long*>(d_counters), st, launches, nullptr);
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_agg_run_host(const int64_t* keys, const int64_t* ts, int64_t n, const b2s_agg_spec* specs, int32_t n_specs,
                                uint64_t* counters, b2s_stats* stats) {
  try {  // no C++ exception crosses the C boundary
    std::vector<const void*> sources;
    if (int rc = check_specs(keys, ts, n, specs, n_specs, counters, &sources)) return rc;
    if (stats) {
      memset(stats, 0, sizeof(*stats));
      stats->rows = n;
    }
    if (n == 0) {
      counters[0] = counters[1] = counters[2] = 0;
      return B2S_OK;
    }
    if (!b2s_int_inited()) return b2s_int_fail(B2S_ERR_STATE, "b2s_init was not called (no CUDA device: there is no CPU fallback)");
    B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
    cudaStream_t st = b2s_int_stream();
    Events ev;
    if (int rc = ev.create(4)) return rc;
    // device mirrors: the counters, keys, timestamps, each distinct source, each output; one block
    SyncOnExit done{st};
    DeviceBlock blk(st);
    unsigned long long* d_cnt = nullptr;
    const int64_t* d_keys = nullptr;
    const int64_t* d_ts = nullptr;
    blk.scratch(d_cnt, 24);
    blk.input(d_keys, keys, (size_t)n * 8);
    blk.input(d_ts, ts, (size_t)n * 8);
    std::vector<const void*> dsources(sources);
    for (const void*& src : dsources) blk.input(src, src, (size_t)n * 4);
    std::vector<b2s_agg_spec> dspecs(specs, specs + n_specs);
    std::vector<std::vector<double*>> douts(n_specs);
    for (int s = 0; s < n_specs; ++s) {
      douts[s].assign(specs[s].outs, specs[s].outs + n_ops(specs[s].ops) * specs[s].n_windows);
      for (double*& o : douts[s]) blk.output(o, o, 8, n);
      dspecs[s].outs = douts[s].data();
    }
    if (int rc = blk.alloc()) return rc;
    for (int s = 0; s < n_specs; ++s)
      dspecs[s].src = dsources[std::find(sources.begin(), sources.end(), specs[s].src) - sources.begin()];
    B2S_CUDA_TRY(cudaMemsetAsync(d_cnt, 0, 24, st));
    B2S_CUDA_TRY(cudaEventRecord(ev[0], st));
    if (int rc = blk.upload()) return rc;
    B2S_CUDA_TRY(cudaEventRecord(ev[1], st));
    Launches launches;
    if (int rc = run(d_keys, d_ts, n, dspecs.data(), n_specs, dsources, d_cnt, st, launches, ev[2])) return rc;
    B2S_CUDA_TRY(cudaEventRecord(ev[3], st));
    if (int rc = blk.download(0, n, st)) return rc;
    B2S_CUDA_TRY(cudaMemcpyAsync(counters, d_cnt, 24, cudaMemcpyDeviceToHost, st));
    B2S_CUDA_TRY(cudaStreamSynchronize(st));
    if (stats) {
      float sort_ms = 0.f, agg_ms = 0.f;
      cudaEventElapsedTime(&stats->h2d_ms, ev[0], ev[1]);
      cudaEventElapsedTime(&sort_ms, ev[1], ev[2]);
      cudaEventElapsedTime(&agg_ms, ev[2], ev[3]);
      stats->kernel_ms = sort_ms + agg_ms;
      stats->kernels = launches.n;
    }
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_agg_time_device(const int64_t* d_keys, const int64_t* d_ts, int64_t n, const b2s_agg_spec* specs, int32_t n_specs,
                                   uint64_t* d_counters, int32_t n_iters, float* sort_ms, float* total_ms) {
  try {  // no C++ exception crosses the C boundary
    std::vector<const void*> sources;
    if (int rc = check_specs(d_keys, d_ts, n, specs, n_specs, d_counters, &sources)) return rc;
    if (n_iters < 1 || !sort_ms || !total_ms) return b2s_int_fail(B2S_ERR_INVALID, "n_iters >= 1 and both times are required");
    if (!b2s_int_inited()) return b2s_int_fail(B2S_ERR_STATE, "b2s_init was not called (no CUDA device: there is no CPU fallback)");
    B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
    cudaStream_t st = b2s_int_stream();
    *sort_ms = *total_ms = 0.f;
    Events ev;
    if (int rc = ev.create(3)) return rc;
    SyncOnExit done{st};
    for (int it = 0; it < n_iters && n; ++it) {
      Launches launches;
      B2S_CUDA_TRY(cudaEventRecord(ev[0], st));
      if (int rc = run(d_keys, d_ts, n, specs, n_specs, sources, reinterpret_cast<unsigned long long*>(d_counters), st, launches, ev[1])) return rc;
      B2S_CUDA_TRY(cudaEventRecord(ev[2], st));
      B2S_CUDA_TRY(cudaEventSynchronize(ev[2]));
      float a = 0.f, b = 0.f;
      cudaEventElapsedTime(&a, ev[0], ev[1]);
      cudaEventElapsedTime(&b, ev[0], ev[2]);
      *sort_ms += a;
      *total_ms += b;
    }
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}
