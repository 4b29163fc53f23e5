// b2s_table.cu -- device-resident online feature table: entity key -> feature vector (+ imputing), sm_90a.
//
// Replaces the lookup half of real-time feature enrichment: EnrichmentModelRouter / EnrichmentVotingEnsemble.preprocess
// (mlrun/serving/routers.py:1189-1196, 1335-1342) call OnlineVectorService.get (mlrun/feature_store/feature_vector.py:
// 975-1067), which emits every entity row into a storey graph that reads the online (NoSQL) store key by key, then fills
// missing / NaN / Inf values from the impute policy (:1046-1052).  Here the online table lives in HBM: an open-addressing
// hash table of 64-bit entity keys (linear probing, load factor <= 0.5, built once on the host) next to the
// [n_keys][n_features] float32 matrix; one kernel launch resolves a batch of keys: each lane probes for one key, then
// the warp copies the 32 rows it found with coalesced 16-byte accesses, imputing on the way, straight into the row
// matrix the scoring plan reads (no host round trip between enrichment and predict).
// Bound: HBM (random 4*F-byte row reads + the sequential output): algorithmic bytes = 8 (key) + 16 (slot) + 8*F per
// query.
#include <cuda_runtime.h>

#include <exception>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/b200serve.h"
#include "b2s_internal.h"
#include "b2s_hash.cuh"
#include "b2s_stage.h"

namespace {

using Slot = b2s::TableSlot;
using b2s::mix64;

struct LookupParams {
  const Slot* slots;
  uint64_t mask;            // capacity - 1
  const float* values;      // [n_keys][n_feat]
  const float* impute;      // [n_feat]; NaN: keep the stored value
  int32_t n_feat;
  int32_t any_impute;
  int32_t lanes_per_row;    // n_feat / 4 when that is a power of two <= 32 (rows are copied by sub-warps), else 0
  int32_t vec;              // 1: every output row is 16-byte aligned (n_feat % 4 == 0, out and out_stride 16-byte multiples)
  const int64_t* keys;      // [n]
  int64_t n;
  float* out;               // row i at out + i * out_stride (bytes)
  int64_t out_stride;
  int32_t* found;           // [n] 1 / 0 (rows of unknown keys are filled with NaN)
};

__global__ void __launch_bounds__(256) table_lookup_kernel(const __grid_constant__ LookupParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const bool vec = p.vec != 0;
  for (int64_t base = warp * 32; base < p.n; base += n_warps * 32) {
    const int64_t q = base + lane;
    int64_t row = -1;
    if (q < p.n) {  // every lane probes for its own key
      row = b2s::table_find(p.slots, p.mask, p.keys[q]);
      if (p.found) p.found[q] = row >= 0 ? 1 : 0;
    }
    const int cnt = (int)((p.n - base < 32) ? (p.n - base) : 32);
    if (vec && p.lanes_per_row) {
      // lanes_per_row = n_feat / 4 lanes copy one row with one 16-byte access each, so a warp moves 32 / lanes_per_row rows
      // per step (two for 64 features); kGather steps are loaded before any is stored (more rows in flight)
      const int lpr = p.lanes_per_row, rpi = 32 / lpr;
      const int sub = lane / lpr, c = (lane - sub * lpr) * 4;
      const float4 f = p.any_impute ? *reinterpret_cast<const float4*>(p.impute + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      constexpr int kGather = 4;
      for (int j0 = 0; j0 < cnt; j0 += rpi * kGather) {
        float4 v[kGather];
#pragma unroll
        for (int u = 0; u < kGather; ++u) {
          const int j = j0 + u * rpi + sub;
          const int64_t r = __shfl_sync(0xffffffffu, row, j & 31);
          v[u] = (j < cnt && r >= 0) ? __ldg(reinterpret_cast<const float4*>(p.values + r * p.n_feat + c))
                                     : make_float4(NAN, NAN, NAN, NAN);
        }
#pragma unroll
        for (int u = 0; u < kGather; ++u) {
          const int j = j0 + u * rpi + sub;
          if (j >= cnt) continue;
          float4 w = v[u];
          if (p.any_impute) {  // OnlineVectorService.get (:1046-1052): None / NaN / Inf -> impute value
            w.x = (!(fabsf(w.x) <= 3.402823466e38f) && f.x == f.x) ? f.x : w.x;
            w.y = (!(fabsf(w.y) <= 3.402823466e38f) && f.y == f.y) ? f.y : w.y;
            w.z = (!(fabsf(w.z) <= 3.402823466e38f) && f.z == f.z) ? f.z : w.z;
            w.w = (!(fabsf(w.w) <= 3.402823466e38f) && f.w == f.w) ? f.w : w.w;
          }
          *reinterpret_cast<float4*>(reinterpret_cast<char*>(p.out) + (base + j) * p.out_stride + c * 4) = w;
        }
      }
      continue;
    }
    for (int j = 0; j < cnt; ++j) {  // the warp copies query j's row together
      const int64_t r = __shfl_sync(0xffffffffu, row, j);
      float* dst = reinterpret_cast<float*>(reinterpret_cast<char*>(p.out) + (base + j) * p.out_stride);
      const float* src = p.values + r * p.n_feat;
      if (vec) {
        for (int c = lane * 4; c < p.n_feat; c += 128) {
          float4 v = r >= 0 ? *reinterpret_cast<const float4*>(src + c) : make_float4(NAN, NAN, NAN, NAN);
          if (p.any_impute) {  // OnlineVectorService.get (:1046-1052): None / NaN / Inf -> impute value
            const float4 f = *reinterpret_cast<const float4*>(p.impute + c);
            v.x = (!(fabsf(v.x) <= 3.402823466e38f) && f.x == f.x) ? f.x : v.x;
            v.y = (!(fabsf(v.y) <= 3.402823466e38f) && f.y == f.y) ? f.y : v.y;
            v.z = (!(fabsf(v.z) <= 3.402823466e38f) && f.z == f.z) ? f.z : v.z;
            v.w = (!(fabsf(v.w) <= 3.402823466e38f) && f.w == f.w) ? f.w : v.w;
          }
          *reinterpret_cast<float4*>(dst + c) = v;
        }
      } else {
        for (int c = lane; c < p.n_feat; c += 32) {
          float v = r >= 0 ? src[c] : NAN;
          if (p.any_impute) {
            const float f = p.impute[c];
            v = (!(fabsf(v) <= 3.402823466e38f) && f == f) ? f : v;
          }
          dst[c] = v;
        }
      }
    }
  }
}

// status[i] |= B2S_ROW_UNKNOWN_KEY where the key was not in the table (after the scoring plan wrote status)
__global__ void mark_unknown_kernel(const int32_t* __restrict__ found, int32_t* __restrict__ status, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (!found[i]) status[i] |= B2S_ROW_UNKNOWN_KEY;
}

}  // namespace

struct b2s_table_s {
  int64_t n_keys = 0;
  int32_t n_feat = 0;
  uint64_t cap = 0;
  int any_impute = 0;
  Slot* d_slots = nullptr;
  float* d_values = nullptr;
  float* d_impute = nullptr;
  std::vector<float> h_impute;  // host copy: the fused gather folds the policy into the scoring kernel's operands
  int grid = 0;
  // host-call staging
  std::mutex mu;
  int64_t cap_rows = 0;
  int64_t* d_keys = nullptr;
  float* d_out = nullptr;
  int32_t* d_found = nullptr;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  // enrich_host staging: votes + status on the device, one pinned block [keys | votes | status] on the host
  int64_t enr_rows = 0;
  int32_t enr_out_cols = 0;
  float* d_votes = nullptr;
  int32_t* d_status = nullptr;
  char* h_pin = nullptr;
};

// what both builds do once the slots and values are in place: the padded impute vector (NaN: keep the stored value),
// the lookup grid and the events of the host calls
static int table_finish(b2s_table_s* t, const float* impute) {
  const int n_features = t->n_feat;
  std::vector<float> imp(((size_t)n_features + 3) / 4 * 4, NAN);
  if (impute)
    for (int c = 0; c < n_features; ++c) {
      imp[c] = impute[c];
      if (impute[c] == impute[c]) t->any_impute = 1;
    }
  t->h_impute = imp;
  B2S_CUDA_TRY(cudaMalloc(&t->d_impute, imp.size() * 4));
  B2S_CUDA_TRY(cudaMemcpy(t->d_impute, imp.data(), imp.size() * 4, cudaMemcpyHostToDevice));
  int occ = 0;
  B2S_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, table_lookup_kernel, 256, 0));
  t->grid = b2s_int_sm_count() * std::max(occ, 1);
  for (int i = 0; i < 4; ++i) B2S_CUDA_TRY(cudaEventCreate(&t->ev[i]));
  return B2S_OK;
}

extern "C" int b2s_table_create(const int64_t* keys, int64_t n_keys, const float* values, int32_t n_features, const float* impute,
                                b2s_table_t* out) {
  try {  // no C++ exception crosses the C boundary
    if (!keys || !values || !out || n_keys <= 0 || n_features <= 0) return b2s_int_fail(B2S_ERR_INVALID, "bad arguments");
    if (!b2s_int_inited()) return b2s_int_fail(B2S_ERR_STATE, "b2s_init was not called (no CUDA device: there is no CPU fallback)");
    uint64_t cap = 16;
    while (cap < (uint64_t)n_keys * 2) cap <<= 1;
    std::vector<Slot> slots(cap, Slot{0, -1});
    for (int64_t i = 0; i < n_keys; ++i) {
      uint64_t h = mix64((uint64_t)keys[i]) & (cap - 1);
      while (slots[h].row >= 0) {
        if (slots[h].key == keys[i]) return b2s_int_fail(B2S_ERR_INVALID, "duplicate entity key %lld (rows %lld and %lld)", (long long)keys[i], (long long)slots[h].row, (long long)i);
        h = (h + 1) & (cap - 1);
      }
      slots[h] = Slot{keys[i], i};
    }
    auto* t = new b2s_table_s();
    t->n_keys = n_keys;
    t->n_feat = n_features;
    t->cap = cap;
    B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
    B2S_CUDA_TRY(cudaMalloc(&t->d_slots, cap * sizeof(Slot)));
    B2S_CUDA_TRY(cudaMemcpy(t->d_slots, slots.data(), cap * sizeof(Slot), cudaMemcpyHostToDevice));
    // one more row than keys: row n_keys is all NaN, what the fused gather copies for an unknown key
    B2S_CUDA_TRY(cudaMalloc(&t->d_values, ((size_t)n_keys + 1) * n_features * 4));
    B2S_CUDA_TRY(cudaMemcpy(t->d_values, values, (size_t)n_keys * n_features * 4, cudaMemcpyHostToDevice));
    {
      const std::vector<float> nan_row((size_t)n_features, NAN);
      B2S_CUDA_TRY(cudaMemcpy(t->d_values + (size_t)n_keys * n_features, nan_row.data(), (size_t)n_features * 4, cudaMemcpyHostToDevice));
    }
    if (int rc = table_finish(t, impute)) return rc;
    *out = t;
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

static int launch_lookup(b2s_table_t t, const int64_t* d_keys, int64_t n, float* d_rows, int64_t row_stride, int32_t* d_found, cudaStream_t st) {
  LookupParams p{};
  p.slots = t->d_slots;
  p.mask = t->cap - 1;
  p.values = t->d_values;
  p.impute = t->d_impute;
  p.n_feat = t->n_feat;
  p.any_impute = t->any_impute;
  {
    const int l = t->n_feat / 4;
    p.lanes_per_row = (t->n_feat % 4 == 0 && l >= 1 && l <= 32 && (l & (l - 1)) == 0) ? l : 0;
  }
  p.keys = d_keys;
  p.n = n;
  p.out = d_rows;
  p.out_stride = row_stride;
  // 16-byte stores only where every row starts on a 16-byte boundary: a caller may gather into a column offset of a
  // wider row matrix (stride a multiple of 16, base 4 bytes off), which takes the scalar path
  p.vec = (t->n_feat % 4) == 0 && (row_stride % 16) == 0 && ((uintptr_t)d_rows % 16) == 0;
  p.found = d_found;
  const int64_t warps = (n + 31) / 32;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(t->grid, (warps + 7) / 8));
  b2s_int_count_launches(1);
  table_lookup_kernel<<<grid, 256, 0, st>>>(p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return b2s_int_fail(B2S_ERR_CUDA, "table lookup launch failed: %s", cudaGetErrorString(e));
  return B2S_OK;
}

// the kernels load keys as 8-byte words and store rows, flags and status words as 4-byte words (rows also as 16-byte
// words where the base allows): a pointer off those boundaries is refused before anything is launched
extern "C" int b2s_table_lookup_device(b2s_table_t t, const int64_t* d_keys, int64_t n, float* d_rows, int64_t row_stride_bytes,
                                       int32_t* d_found, void* stream) {
  try {  // no C++ exception crosses the C boundary
    if (!t) return b2s_int_fail(B2S_ERR_INVALID, "null table");
    if (n < 0 || row_stride_bytes < (int64_t)t->n_feat * 4 || (row_stride_bytes & 3)) return b2s_int_fail(B2S_ERR_INVALID, "bad n / row stride");
    if (n > 0 && (!d_keys || !d_rows)) return b2s_int_fail(B2S_ERR_INVALID, "null keys / rows");
    if (misaligned(d_keys, 8) || misaligned(d_rows, 4) || misaligned(d_found, 4))
      return b2s_int_fail(B2S_ERR_INVALID, "keys must be 8-byte aligned, rows and found 4-byte aligned");
    if (n == 0) return B2S_OK;
    B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
    return launch_lookup(t, d_keys, n, d_rows, row_stride_bytes, d_found, stream ? (cudaStream_t)stream : b2s_int_stream());
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_table_lookup_host(b2s_table_t t, const int64_t* keys, int64_t n, float* rows, int32_t* found, b2s_stats* stats) {
  try {  // no C++ exception crosses the C boundary
    if (!t || !keys || !rows || n < 0) return b2s_int_fail(B2S_ERR_INVALID, "bad arguments");
    if (n == 0) return B2S_OK;
    std::lock_guard<std::mutex> lk(t->mu);
    B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
    if (n > t->cap_rows) {
      if (t->d_keys) { cudaFree(t->d_keys); cudaFree(t->d_out); cudaFree(t->d_found); t->d_keys = nullptr; }
      t->cap_rows = 0;
      const int64_t cap = std::max<int64_t>(n, 4096);
      B2S_CUDA_TRY(cudaMalloc(&t->d_keys, cap * 8));
      B2S_CUDA_TRY(cudaMalloc(&t->d_out, (size_t)cap * t->n_feat * 4));
      B2S_CUDA_TRY(cudaMalloc(&t->d_found, cap * 4));
      t->cap_rows = cap;
    }
    cudaStream_t st = b2s_int_stream();
    const int64_t stride = (int64_t)t->n_feat * 4;
    B2S_CUDA_TRY(cudaEventRecord(t->ev[0], st));
    B2S_CUDA_TRY(cudaMemcpyAsync(t->d_keys, keys, n * 8, cudaMemcpyHostToDevice, st));
    B2S_CUDA_TRY(cudaEventRecord(t->ev[1], st));
    if (int rc = launch_lookup(t, t->d_keys, n, t->d_out, stride, t->d_found, st)) return rc;
    B2S_CUDA_TRY(cudaEventRecord(t->ev[2], st));
    B2S_CUDA_TRY(cudaMemcpyAsync(rows, t->d_out, (size_t)n * stride, cudaMemcpyDeviceToHost, st));
    if (found) B2S_CUDA_TRY(cudaMemcpyAsync(found, t->d_found, n * 4, cudaMemcpyDeviceToHost, st));
    B2S_CUDA_TRY(cudaEventRecord(t->ev[3], st));
    B2S_CUDA_TRY(cudaStreamSynchronize(st));
    if (stats) {
      memset(stats, 0, sizeof(*stats));
      stats->rows = n;
      cudaEventElapsedTime(&stats->h2d_ms, t->ev[0], t->ev[1]);
      cudaEventElapsedTime(&stats->kernel_ms, t->ev[1], t->ev[2]);
      cudaEventElapsedTime(&stats->d2h_ms, t->ev[2], t->ev[3]);
      stats->kernels = 1;
    }
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

// A plan with merge targets or an attached communicator stores its votes there and never into the enrichment's output,
// which would then hand out memory no kernel wrote: both entry points refuse it before anything is enqueued.
static int refuse_merging(b2s_plan_t plan) {
  if (!b2s_int_plan_merges(plan)) return B2S_OK;
  return b2s_int_fail(B2S_ERR_UNSUPPORTED, "the plan stores its votes to merge targets or a communicator: enrich without them");
}

static int launch_fused(b2s_table_t t, b2s_plan_t plan, const int64_t* d_keys, int64_t n, void* d_out, int32_t* d_status, cudaStream_t st) {
  B2SGather g{};
  g.d_keys = reinterpret_cast<const long long*>(d_keys);
  g.d_slots = t->d_slots;
  g.mask = t->cap - 1;
  g.d_values = t->d_values;
  g.missing_row = t->n_keys;
  g.h_impute = t->h_impute.data();
  g.any_impute = t->any_impute;
  g.n_feat = t->n_feat;
  return b2s_int_launch_gathered(plan, g, n, d_out, d_status, st);
}

extern "C" int b2s_table_enrich_device(b2s_table_t t, b2s_plan_t plan, const int64_t* d_keys, int64_t n, void* d_out,
                                       int32_t* d_status, void* stream) {
  try {  // no C++ exception crosses the C boundary
    if (!t || !plan || !d_keys || !d_out || n < 0) return b2s_int_fail(B2S_ERR_INVALID, "bad arguments");
    if (misaligned(d_keys, 8) || misaligned(d_out, 4) || misaligned(d_status, 4))
      return b2s_int_fail(B2S_ERR_INVALID, "keys must be 8-byte aligned, out and status 4-byte aligned");
    if (int rc = refuse_merging(plan)) return rc;
    if (n == 0) return B2S_OK;
    B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
    return launch_fused(t, plan, d_keys, n, d_out, d_status, stream ? (cudaStream_t)stream : b2s_int_stream());
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

static bool host_pinned(const void* ptr) {
  cudaPointerAttributes attr{};
  const bool yes = cudaPointerGetAttributes(&attr, ptr) == cudaSuccess && attr.type == cudaMemoryTypeHost;
  cudaGetLastError();
  return yes;
}

extern "C" int b2s_table_enrich_host(b2s_table_t t, b2s_plan_t plan, const int64_t* keys, int64_t n, void* out, int64_t out_bytes,
                                     int32_t* row_status, b2s_stats* stats) {
  try {  // no C++ exception crosses the C boundary
    if (!t || !keys || !out || n < 0) return b2s_int_fail(B2S_ERR_INVALID, "bad arguments");
    int n_in = 0, out_cols = 0;
    if (int rc = b2s_int_plan_shape(plan, &n_in, &out_cols)) return rc;
    if (n_in != t->n_feat) return b2s_int_fail(B2S_ERR_INVALID, "the table has %d features, the plan takes %d", t->n_feat, n_in);
    if (out_bytes < n * out_cols * 4) return b2s_int_fail(B2S_ERR_INVALID, "out buffer too small");
    if (int rc = refuse_merging(plan)) return rc;
    if (n == 0) return B2S_OK;
    std::lock_guard<std::mutex> lk(t->mu);
    B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
    const int64_t stride = (int64_t)t->n_feat * 4;
    if (n > t->cap_rows) {
      if (t->d_keys) { cudaFree(t->d_keys); cudaFree(t->d_out); cudaFree(t->d_found); t->d_keys = nullptr; }
      t->cap_rows = 0;
      const int64_t cap = std::max<int64_t>(n, 4096);
      B2S_CUDA_TRY(cudaMalloc(&t->d_keys, cap * 8));
      B2S_CUDA_TRY(cudaMalloc(&t->d_out, (size_t)cap * stride));
      B2S_CUDA_TRY(cudaMalloc(&t->d_found, cap * 4));
      t->cap_rows = cap;
    }
    if (n > t->enr_rows || out_cols > t->enr_out_cols) {
      if (t->d_votes) { cudaFree(t->d_votes); cudaFree(t->d_status); cudaFreeHost(t->h_pin); t->d_votes = nullptr; }
      t->enr_rows = 0;
      const int64_t cap = std::max<int64_t>(n, 4096);
      const int32_t oc = std::max(out_cols, t->enr_out_cols);
      B2S_CUDA_TRY(cudaMalloc(&t->d_votes, (size_t)cap * oc * 4));
      B2S_CUDA_TRY(cudaMalloc(&t->d_status, cap * 4));
      B2S_CUDA_TRY(cudaMallocHost(&t->h_pin, (size_t)cap * (8 + (size_t)oc * 4 + 4)));
      t->enr_rows = cap;
      t->enr_out_cols = oc;
    }
    cudaStream_t st = b2s_int_stream();
    int64_t* h_keys = (int64_t*)t->h_pin;
    char* h_votes = t->h_pin + (size_t)t->enr_rows * 8;
    int32_t* h_status = (int32_t*)(h_votes + (size_t)t->enr_rows * t->enr_out_cols * 4);
    const size_t votes_sz = (size_t)n * out_cols * 4;
    // pinned caller buffers are used as they are; pageable ones go through the pinned block (one host memcpy each way)
    const void* k_src = keys;
    if (!host_pinned(keys)) {
      memcpy(h_keys, keys, (size_t)n * 8);
      k_src = h_keys;
    }
    void* v_dst = host_pinned(out) ? out : (void*)h_votes;
    int32_t* s_dst = row_status ? (host_pinned(row_status) ? row_status : h_status) : nullptr;
    B2S_CUDA_TRY(cudaEventRecord(t->ev[0], st));
    B2S_CUDA_TRY(cudaMemcpyAsync(t->d_keys, k_src, (size_t)n * 8, cudaMemcpyHostToDevice, st));
    B2S_CUDA_TRY(cudaEventRecord(t->ev[1], st));
    int n_kernels = 1;
    int rc = launch_fused(t, plan, t->d_keys, n, t->d_votes, t->d_status, st);  // gather inside the scoring kernel
    if (rc == B2S_ERR_UNSUPPORTED) {  // plans the gather loader does not cover: gather, score, fold the flags
      n_kernels = 2 + b2s_int_plan_kernels(plan);
      if ((rc = launch_lookup(t, t->d_keys, n, t->d_out, stride, t->d_found, st))) return rc;
      if ((rc = b2s_run_device(plan, t->d_out, n, stride, t->d_votes, t->d_status, st))) return rc;
      const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(4 * b2s_int_sm_count(), (n + 255) / 256));
      b2s_int_count_launches(1);
      mark_unknown_kernel<<<grid, 256, 0, st>>>(t->d_found, t->d_status, n);
      cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) return b2s_int_fail(B2S_ERR_CUDA, "mark_unknown launch failed: %s", cudaGetErrorString(e));
    } else if (rc) {
      return rc;
    }
    B2S_CUDA_TRY(cudaEventRecord(t->ev[2], st));
    B2S_CUDA_TRY(cudaMemcpyAsync(v_dst, t->d_votes, votes_sz, cudaMemcpyDeviceToHost, st));
    if (s_dst) B2S_CUDA_TRY(cudaMemcpyAsync(s_dst, t->d_status, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    B2S_CUDA_TRY(cudaEventRecord(t->ev[3], st));
    B2S_CUDA_TRY(cudaStreamSynchronize(st));
    if (v_dst != out) memcpy(out, h_votes, votes_sz);
    if (s_dst && s_dst != row_status) memcpy(row_status, h_status, (size_t)n * 4);
    if (stats) {
      memset(stats, 0, sizeof(*stats));
      stats->rows = n;
      cudaEventElapsedTime(&stats->h2d_ms, t->ev[0], t->ev[1]);
      cudaEventElapsedTime(&stats->kernel_ms, t->ev[1], t->ev[2]);
      cudaEventElapsedTime(&stats->d2h_ms, t->ev[2], t->ev[3]);
      stats->kernels = n_kernels;  // 1: gather fused into the scoring kernel; else gather + the plan's launches + mark_unknown
      if (row_status)
        for (int64_t r = 0; r < n; ++r) stats->nonfinite_rows += (row_status[r] & B2S_ROW_NONFINITE_INPUT) ? 1 : 0;
    }
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_table_time_device(b2s_table_t t, const int64_t* const* d_keys, int32_t n_bufs, int64_t n, float* d_rows,
                                     int64_t row_stride_bytes, int32_t* d_found, int32_t n_iters, float* total_ms) {
  try {  // no C++ exception crosses the C boundary
    if (!t || !d_keys || n_bufs <= 0 || n_iters <= 0 || !total_ms) return b2s_int_fail(B2S_ERR_INVALID, "bad arguments");
    B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
    cudaStream_t st = b2s_int_stream();
    std::lock_guard<std::mutex> lk(t->mu);
    B2S_CUDA_TRY(cudaEventRecord(t->ev[0], st));
    for (int i = 0; i < n_iters; ++i)
      if (int rc = launch_lookup(t, d_keys[i % n_bufs], n, d_rows, row_stride_bytes, d_found, st)) return rc;
    B2S_CUDA_TRY(cudaEventRecord(t->ev[1], st));
    B2S_CUDA_TRY(cudaStreamSynchronize(st));
    B2S_CUDA_TRY(cudaEventElapsedTime(total_ms, t->ev[0], t->ev[1]));
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_table_info(b2s_table_t t, int64_t* n_keys, int32_t* n_features, int64_t* capacity) {
  try {  // no C++ exception crosses the C boundary
    if (!t) return b2s_int_fail(B2S_ERR_INVALID, "null table");
    if (n_keys) *n_keys = t->n_keys;
    if (n_features) *n_features = t->n_feat;
    if (capacity) *capacity = (int64_t)t->cap;
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_table_destroy(b2s_table_t t) {
  try {  // no C++ exception crosses the C boundary
    if (!t) return B2S_OK;
    if (t->d_slots) cudaFree(t->d_slots);
    if (t->d_values) cudaFree(t->d_values);
    if (t->d_impute) cudaFree(t->d_impute);
    if (t->d_keys) cudaFree(t->d_keys);
    if (t->d_out) cudaFree(t->d_out);
    if (t->d_found) cudaFree(t->d_found);
    if (t->d_votes) cudaFree(t->d_votes);
    if (t->d_status) cudaFree(t->d_status);
    if (t->h_pin) cudaFreeHost(t->h_pin);
    for (auto& e : t->ev)
      if (e) cudaEventDestroy(e);
    delete t;
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

// FNV-1a over each string of a packed buffer: the 64-bit entity key of a string-valued entity (host code)
extern "C" int b2s_hash_strings(const char* bytes, const int64_t* offsets, int64_t n, int64_t* keys_out) {
  try {  // no C++ exception crosses the C boundary
    if (!bytes || !offsets || !keys_out || n < 0) return b2s_int_fail(B2S_ERR_INVALID, "bad arguments");
    for (int64_t i = 0; i < n; ++i) {
      uint64_t h = 1469598103934665603ULL;
      for (int64_t j = offsets[i]; j < offsets[i + 1]; ++j) {
        h ^= (unsigned char)bytes[j];
        h *= 1099511628211ULL;
      }
      keys_out[i] = (int64_t)h;
    }
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

// ---- the online table built from device columns --------------------------------------------------------------------------
// A vector's online rows that already live in HBM (CUDA columns, a device ingest's result) become a table without a host
// round trip: table_pack_kernel writes the row-major float32 values, table_insert_kernel claims one slot per key,
// table_check_kernel finds repeated keys; the statistics of the impute policy and the keys of truthy labels are reduced and
// compacted where the columns are.
namespace {

struct TCol {
  const void* src;
  int32_t bytes;
  int32_t kind;
};

constexpr int kTableThreads = 256;
constexpr unsigned kNaN32 = 0x7fc00000u;  // the NaN numpy writes

// the value of row i as numpy's astype(float32) gives it (round to nearest even, overflow to +-inf, bool to 0 / 1; a
// float64 NaN keeps its sign and the top of its payload, quieted, as x86's conversion keeps them)
__device__ __forceinline__ float col_f32(const TCol& c, int64_t i) {
  switch (c.kind) {
    case B2S_TCOL_FLOAT:
      if (c.bytes == 4) return static_cast<const float*>(c.src)[i];
      {
        const double d = static_cast<const double*>(c.src)[i];
        if (d != d) {
          const unsigned long long b = (unsigned long long)__double_as_longlong(d);
          return __uint_as_float((unsigned)(b >> 32 & 0x80000000u) | kNaN32 | (unsigned)(b >> 29 & 0x3fffffu));
        }
        return __double2float_rn(d);
      }
    case B2S_TCOL_INT:
      switch (c.bytes) {
        case 1: return (float)static_cast<const int8_t*>(c.src)[i];
        case 2: return (float)static_cast<const int16_t*>(c.src)[i];
        case 4: return __int2float_rn(static_cast<const int32_t*>(c.src)[i]);
        default: return __ll2float_rn(static_cast<const long long*>(c.src)[i]);
      }
    case B2S_TCOL_UINT:
      switch (c.bytes) {
        case 1: return (float)static_cast<const uint8_t*>(c.src)[i];
        case 2: return (float)static_cast<const uint16_t*>(c.src)[i];
        case 4: return __uint2float_rn(static_cast<const uint32_t*>(c.src)[i]);
        default: return __ull2float_rn(static_cast<const unsigned long long*>(c.src)[i]);
      }
    default: return static_cast<const uint8_t*>(c.src)[i] ? 1.f : 0.f;
  }
}

// values[r][c] = column c at row r, through a 32 x 32 shared tile: loads run down each column, stores along each row.
// blockIdx.y is the tile of 32 columns; the blocks of x = 0 also write row n, all NaN (the unknown key's row).
__global__ void __launch_bounds__(kTableThreads) table_pack_kernel(const TCol* __restrict__ cols, int32_t n_feat, int64_t n,
                                                                    float* __restrict__ values) {
  __shared__ float tile[32][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c0 = blockIdx.y * 32;
  const int cw = min(32, n_feat - c0);
  if (blockIdx.x == 0 && (int)threadIdx.x < cw) values[n * n_feat + c0 + threadIdx.x] = __uint_as_float(kNaN32);
  for (int64_t r0 = (int64_t)blockIdx.x * 32; r0 < n; r0 += (int64_t)gridDim.x * 32) {
    for (int c = warp; c < cw; c += kTableThreads / 32) {
      const TCol col = cols[c0 + c];
      if (r0 + lane < n) tile[c][lane] = col_f32(col, r0 + lane);
    }
    __syncthreads();
    for (int r = warp; r < 32 && r0 + r < n; r += kTableThreads / 32)
      if (lane < cw) values[(r0 + r) * n_feat + c0 + lane] = tile[lane][r];
    __syncthreads();
  }
}

// one range of b2s_run_columns_device: rows[r][c] = column c at row first + r for r < n, the same tile transpose and
// conversion as table_pack_kernel without its NaN row (kept apart so that table_pack_kernel's code stays as it is)
__global__ void __launch_bounds__(kTableThreads) rows_pack_kernel(const TCol* __restrict__ cols, int32_t n_feat, int64_t first,
                                                                   int64_t n, float* __restrict__ rows) {
  __shared__ float tile[32][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c0 = blockIdx.y * 32;
  const int cw = min(32, n_feat - c0);
  for (int64_t r0 = (int64_t)blockIdx.x * 32; r0 < n; r0 += (int64_t)gridDim.x * 32) {
    for (int c = warp; c < cw; c += kTableThreads / 32) {
      const TCol col = cols[c0 + c];
      if (r0 + lane < n) tile[c][lane] = col_f32(col, first + r0 + lane);
    }
    __syncthreads();
    for (int r = warp; r < 32 && r0 + r < n; r += kTableThreads / 32)
      if (lane < cw) rows[(r0 + r) * n_feat + c0 + lane] = tile[lane][r];
    __syncthreads();
  }
}

// one thread per key claims the first free slot of its walk (the row word goes from -1 to the row, then the key is
// stored): a repeated key takes a slot of its own, which table_check_kernel finds
__global__ void __launch_bounds__(kTableThreads) table_insert_kernel(const int64_t* __restrict__ keys, int64_t n, Slot* slots, uint64_t mask) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const long long k = keys[i];
    uint64_t h = mix64((uint64_t)k) & mask;
    for (;;) {
      unsigned long long* rw = reinterpret_cast<unsigned long long*>(&slots[h].row);
      if (atomicCAS(rw, ~0ull, (unsigned long long)i) == ~0ull) {
        slots[h].key = k;
        break;
      }
      h = (h + 1) & mask;
    }
  }
}

// Every row of a key lies on that key's walk, before its first empty slot.  Row i repeats an earlier row when the walk
// shows the key at a smaller row; *dup = min over such i of (i << 32 | the key's first row): b2s_table_create stops at
// the first row that repeats a key and names the row it repeats, the key's first.
__global__ void __launch_bounds__(kTableThreads) table_check_kernel(const int64_t* __restrict__ keys, int64_t n, const Slot* __restrict__ slots,
                                                                     uint64_t mask, unsigned long long* __restrict__ dup) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const long long k = keys[i];
    uint64_t h = mix64((uint64_t)k) & mask;
    long long first = i;
    for (;;) {
      const longlong2 s = __ldg(reinterpret_cast<const longlong2*>(slots) + h);
      if (s.y < 0) break;
      if (s.x == k && s.y < first) first = s.y;
      h = (h + 1) & mask;
    }
    if (first < i) atomicMin(dup, ((unsigned long long)i << 32) | (unsigned long long)first);
  }
}

struct StatPart {
  double sum;
  long long count;
  float min, max;
};

// the block's sum of v (fixed order: lanes by shuffle, then warps by thread 0); valid in thread 0
template <class T, class Op>
__device__ __forceinline__ T block_reduce(T v, Op op, T* smem) {
  for (int o = 16; o; o >>= 1) v = op(v, __shfl_down_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < kTableThreads / 32; ++w) v = op(v, smem[w]);
  __syncthreads();
  return v;
}

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }

// pass 1, blockIdx.y the column: count, sum (float64), min and max of the finite values, one partial per block
__global__ void __launch_bounds__(kTableThreads) table_stats_sum_kernel(const TCol* __restrict__ cols, int64_t n, StatPart* __restrict__ part) {
  __shared__ double s_d[kTableThreads / 32];
  __shared__ long long s_c[kTableThreads / 32];
  __shared__ float s_f[kTableThreads / 32];
  const TCol col = cols[blockIdx.y];
  double sum = 0.0;
  long long count = 0;
  float mn = INFINITY, mx = -INFINITY;
  for (int64_t i = (int64_t)blockIdx.x * kTableThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kTableThreads) {
    const float v = col_f32(col, i);
    if (fabsf(v) <= 3.402823466e38f) {
      sum = __dadd_rn(sum, (double)v);
      ++count;
      mn = fminf(mn, v);
      mx = fmaxf(mx, v);
    }
  }
  sum = block_reduce(sum, dadd, s_d);
  count = block_reduce(count, [](long long a, long long b) { return a + b; }, s_c);
  mn = block_reduce(mn, [](float a, float b) { return fminf(a, b); }, s_f);
  mx = block_reduce(mx, [](float a, float b) { return fmaxf(a, b); }, s_f);
  if (threadIdx.x == 0) part[(int64_t)blockIdx.y * gridDim.x + blockIdx.x] = StatPart{sum, count, mn, mx};
}

// the column's mean from its pass-1 partials, summed in block order (every caller gets the same bits)
__device__ __forceinline__ double column_mean(const StatPart* part, int nb, int c) {
  double sum = 0.0;
  long long count = 0;
  for (int b = 0; b < nb; ++b) {
    sum = __dadd_rn(sum, part[(int64_t)c * nb + b].sum);
    count += part[(int64_t)c * nb + b].count;
  }
  return __ddiv_rn(sum, (double)count);
}

// pass 2: the sum of squared deviations from the mean, one partial per block (numpy's nanvar: subtract, multiply, sum)
__global__ void __launch_bounds__(kTableThreads) table_stats_sq_kernel(const TCol* __restrict__ cols, int64_t n, const StatPart* __restrict__ part,
                                                                        double* __restrict__ sq) {
  __shared__ double s_d[kTableThreads / 32];
  __shared__ double s_mean;
  if (threadIdx.x == 0) s_mean = column_mean(part, gridDim.x, blockIdx.y);
  __syncthreads();
  const double mean = s_mean;
  const TCol col = cols[blockIdx.y];
  double ss = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * kTableThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kTableThreads) {
    const float v = col_f32(col, i);
    if (fabsf(v) <= 3.402823466e38f) {
      const double d = __dsub_rn((double)v, mean);
      ss = __dadd_rn(ss, __dmul_rn(d, d));
    }
  }
  ss = block_reduce(ss, dadd, s_d);
  if (threadIdx.x == 0) sq[(int64_t)blockIdx.y * gridDim.x + blockIdx.x] = ss;
}

// one thread per column: out[5][n_feat] = mean, min, max, std (ddof 1), count, rounded to float32
__global__ void table_stats_finish_kernel(const StatPart* __restrict__ part, const double* __restrict__ sq, int nb, int32_t n_feat,
                                          float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_feat) return;
  long long count = 0;
  float mn = INFINITY, mx = -INFINITY;
  double ss = 0.0;
  for (int b = 0; b < nb; ++b) {
    const StatPart p = part[(int64_t)c * nb + b];
    count += p.count;
    mn = fminf(mn, p.min);
    mx = fmaxf(mx, p.max);
    ss = __dadd_rn(ss, sq[(int64_t)c * nb + b]);
  }
  const float nan = __uint_as_float(kNaN32);
  out[c] = count ? __double2float_rn(column_mean(part, nb, c)) : nan;
  out[n_feat + c] = count ? mn : nan;
  out[2 * n_feat + c] = count ? mx : nan;
  out[3 * n_feat + c] = count > 1 ? __double2float_rn(__dsqrt_rn(__ddiv_rn(ss, (double)(count - 1)))) : nan;
  out[4 * n_feat + c] = (float)count;
}

// `notna(label) & bool(label)`
__device__ __forceinline__ bool truthy(const TCol& c, int64_t i) {
  if (c.kind == B2S_TCOL_FLOAT) {
    const double v = c.bytes == 4 ? (double)static_cast<const float*>(c.src)[i] : static_cast<const double*>(c.src)[i];
    return v == v && v != 0.0;
  }
  switch (c.bytes) {
    case 1: return static_cast<const uint8_t*>(c.src)[i] != 0;
    case 2: return static_cast<const uint16_t*>(c.src)[i] != 0;
    case 4: return static_cast<const uint32_t*>(c.src)[i] != 0;
    default: return static_cast<const unsigned long long*>(c.src)[i] != 0;
  }
}

// keys of the truthy rows, appended warp by warp (one atomicAdd per warp)
__global__ void __launch_bounds__(kTableThreads) table_label_keys_kernel(const int64_t* __restrict__ keys, int64_t n, const TCol label,
                                                                          int64_t* __restrict__ out, unsigned long long* __restrict__ count) {
  const int lane = threadIdx.x & 31;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i - lane < n; i += (int64_t)gridDim.x * blockDim.x) {
    const bool t = i < n && truthy(label, i);
    const unsigned m = __ballot_sync(0xffffffffu, t);
    unsigned long long base = 0;
    if (lane == 0 && m) base = atomicAdd(count, (unsigned long long)__popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (t) out[base + __popc(m & ((1u << lane) - 1u))] = keys[i];
  }
}

int check_tcols(const b2s_table_col* cols, int32_t n_cols, int64_t n, std::vector<TCol>& dev) {
  dev.resize(n_cols);
  for (int c = 0; c < n_cols; ++c) {
    const b2s_table_col& k = cols[c];
    const bool ok = k.kind == B2S_TCOL_FLOAT ? (k.bytes == 4 || k.bytes == 8)
                    : k.kind == B2S_TCOL_BOOL ? k.bytes == 1
                    : (k.kind == B2S_TCOL_INT || k.kind == B2S_TCOL_UINT) && (k.bytes == 1 || k.bytes == 2 || k.bytes == 4 || k.bytes == 8);
    if (!ok) return b2s_int_fail(B2S_ERR_INVALID, "column %d: kind %d of %d bytes is not a column kind", c, k.kind, k.bytes);
    if (n && !k.src) return b2s_int_fail(B2S_ERR_INVALID, "column %d: null", c);
    dev[c] = TCol{k.src, k.bytes, k.kind};
  }
  return B2S_OK;
}

int check_tcols_on_device(const std::vector<TCol>& cols) {
  for (size_t c = 0; c < cols.size(); ++c)
    if (int rc = check_on_device(cols[c].src, cols[c].bytes, "column", (int)c)) return rc;
  return B2S_OK;
}

int table_device_ready() {
  if (!b2s_int_inited()) return b2s_int_fail(B2S_ERR_STATE, "b2s_init was not called (no CUDA device: there is no CPU fallback)");
  B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
  return B2S_OK;
}

int launched(const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return b2s_int_fail(B2S_ERR_CUDA, "%s launch failed: %s", what, cudaGetErrorString(e));
  return B2S_OK;
}

// the pack, insert and check launches into t (slots and values allocated here), then the host build's refusal of a repeat
int table_build_device(b2s_table_s* t, const int64_t* d_keys, const std::vector<TCol>& cols, cudaStream_t st) {
  const int64_t n = t->n_keys;
  const int32_t F = t->n_feat;
  SyncOnExit done{st};
  DeviceBlock blk(st);
  const TCol* d_cols = nullptr;
  unsigned long long* d_dup = nullptr;
  blk.input(d_cols, cols.data(), sizeof(TCol) * cols.size());
  blk.scratch(d_dup, 8);
  if (int rc = blk.alloc()) return rc;
  if (int rc = blk.upload()) return rc;
  B2S_CUDA_TRY(cudaMalloc(&t->d_slots, t->cap * sizeof(Slot)));
  B2S_CUDA_TRY(cudaMalloc(&t->d_values, ((size_t)n + 1) * F * 4));
  B2S_CUDA_TRY(cudaMemsetAsync(t->d_slots, 0xff, t->cap * sizeof(Slot), st));  // row -1: empty
  B2S_CUDA_TRY(cudaMemsetAsync(d_dup, 0xff, 8, st));
  Launches launches;
  const int gy = (F + 31) / 32;
  const int gx = (int)std::max<int64_t>(1, std::min<int64_t>((n + 31) / 32, ((int64_t)b2s_int_sm_count() * 8 + gy - 1) / gy));
  table_pack_kernel<<<dim3(gx, gy), kTableThreads, 0, st>>>(d_cols, F, n, t->d_values);
  launches.add(1);
  if (int rc = launched("table pack")) return rc;
  const int g = grid_for(n, kTableThreads);
  table_insert_kernel<<<g, kTableThreads, 0, st>>>(d_keys, n, t->d_slots, t->cap - 1);
  launches.add(1);
  if (int rc = launched("table insert")) return rc;
  table_check_kernel<<<g, kTableThreads, 0, st>>>(d_keys, n, t->d_slots, t->cap - 1, d_dup);
  launches.add(1);
  if (int rc = launched("table check")) return rc;
  unsigned long long dup = 0;
  B2S_CUDA_TRY(cudaMemcpyAsync(&dup, d_dup, 8, cudaMemcpyDeviceToHost, st));
  B2S_CUDA_TRY(cudaStreamSynchronize(st));
  if (dup != ~0ull) {
    const long long row = (long long)(dup >> 32), first = (long long)(dup & 0xffffffffull);
    long long key = 0;
    B2S_CUDA_TRY(cudaMemcpy(&key, d_keys + row, 8, cudaMemcpyDeviceToHost));
    return b2s_int_fail(B2S_ERR_INVALID, "duplicate entity key %lld (rows %lld and %lld)", key, first, row);
  }
  return B2S_OK;
}

}  // namespace

extern "C" int b2s_table_create_device(const int64_t* d_keys, int64_t n_keys, const b2s_table_col* cols, int32_t n_features,
                                       const float* impute, b2s_table_t* out) {
  try {  // no C++ exception crosses the C boundary
    if (!d_keys || !cols || !out || n_keys <= 0 || n_keys > 0x7fffffffll || n_features <= 0 || n_features > 65535 * 32)
      return b2s_int_fail(B2S_ERR_INVALID, "bad arguments");
    std::vector<TCol> dev;
    if (int rc = check_tcols(cols, n_features, n_keys, dev)) return rc;
    if (int rc = table_device_ready()) return rc;
    if (int rc = check_on_device(d_keys, 8, "keys", 0)) return rc;
    if (int rc = check_tcols_on_device(dev)) return rc;
    uint64_t cap = 16;
    while (cap < (uint64_t)n_keys * 2) cap <<= 1;  // b2s_table_create's capacity: load factor <= 0.5
    auto* t = new b2s_table_s();
    t->n_keys = n_keys;
    t->n_feat = n_features;
    t->cap = cap;
    int rc = table_build_device(t, d_keys, dev, b2s_int_stream());
    if (!rc) rc = table_finish(t, impute);
    if (rc) {
      b2s_table_destroy(t);
      return rc;
    }
    *out = t;
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_table_stats_device(const b2s_table_col* cols, int32_t n_features, int64_t n, float* stats_out, void* stream) {
  try {  // no C++ exception crosses the C boundary
    if (!cols || !stats_out || n < 0 || n_features <= 0 || n_features > 65535) return b2s_int_fail(B2S_ERR_INVALID, "bad arguments");
    std::vector<TCol> dev;
    if (int rc = check_tcols(cols, n_features, n, dev)) return rc;
    if (int rc = table_device_ready()) return rc;
    if (n)
      if (int rc = check_tcols_on_device(dev)) return rc;
    cudaStream_t st = stream ? (cudaStream_t)stream : b2s_int_stream();
    const int nb = (int)std::max<int64_t>(1, std::min<int64_t>((n + kTableThreads - 1) / kTableThreads,
                                                               ((int64_t)b2s_int_sm_count() * 8 + n_features - 1) / n_features));
    SyncOnExit done{st};
    DeviceBlock blk(st);
    const TCol* d_cols = nullptr;
    StatPart* d_part = nullptr;
    double* d_sq = nullptr;
    float* d_out = nullptr;
    blk.input(d_cols, dev.data(), sizeof(TCol) * dev.size());
    blk.scratch(d_part, sizeof(StatPart) * (size_t)nb * n_features);
    blk.scratch(d_sq, sizeof(double) * (size_t)nb * n_features);
    blk.output(d_out, stats_out, sizeof(float) * 5, n_features);
    if (int rc = blk.alloc()) return rc;
    if (int rc = blk.upload()) return rc;
    Launches launches;
    table_stats_sum_kernel<<<dim3(nb, n_features), kTableThreads, 0, st>>>(d_cols, n, d_part);
    launches.add(1);
    if (int rc = launched("table stats")) return rc;
    table_stats_sq_kernel<<<dim3(nb, n_features), kTableThreads, 0, st>>>(d_cols, n, d_part, d_sq);
    launches.add(1);
    if (int rc = launched("table stats")) return rc;
    table_stats_finish_kernel<<<(n_features + 127) / 128, 128, 0, st>>>(d_part, d_sq, nb, n_features, d_out);
    launches.add(1);
    if (int rc = launched("table stats")) return rc;
    B2S_CUDA_TRY(cudaMemcpyAsync(stats_out, d_out, sizeof(float) * 5 * n_features, cudaMemcpyDeviceToHost, st));
    B2S_CUDA_TRY(cudaStreamSynchronize(st));
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_table_label_keys_device(const int64_t* d_keys, int64_t n, const b2s_table_col* label, int64_t* keys_out, int64_t* n_out,
                                           void* stream) {
  try {  // no C++ exception crosses the C boundary
    if (!label || !n_out || n < 0 || (n && (!d_keys || !keys_out))) return b2s_int_fail(B2S_ERR_INVALID, "bad arguments");
    std::vector<TCol> dev;
    if (int rc = check_tcols(label, 1, n, dev)) return rc;
    *n_out = 0;
    if (n == 0) return B2S_OK;
    if (int rc = table_device_ready()) return rc;
    if (int rc = check_on_device(d_keys, 8, "keys", 0)) return rc;
    if (int rc = check_tcols_on_device(dev)) return rc;
    cudaStream_t st = stream ? (cudaStream_t)stream : b2s_int_stream();
    SyncOnExit done{st};
    DeviceBlock blk(st);
    unsigned long long* d_count = nullptr;
    int64_t* d_out = nullptr;
    blk.scratch(d_count, 8);
    blk.scratch(d_out, (size_t)n * 8);
    if (int rc = blk.alloc()) return rc;
    B2S_CUDA_TRY(cudaMemsetAsync(d_count, 0, 8, st));
    Launches launches;
    table_label_keys_kernel<<<grid_for(n, kTableThreads), kTableThreads, 0, st>>>(d_keys, n, dev[0], d_out, d_count);
    launches.add(1);
    if (int rc = launched("label keys")) return rc;
    unsigned long long count = 0;
    B2S_CUDA_TRY(cudaMemcpyAsync(&count, d_count, 8, cudaMemcpyDeviceToHost, st));
    B2S_CUDA_TRY(cudaStreamSynchronize(st));
    if (count) B2S_CUDA_TRY(cudaMemcpyAsync(keys_out, d_out, count * 8, cudaMemcpyDeviceToHost, st));
    B2S_CUDA_TRY(cudaStreamSynchronize(st));
    *n_out = (int64_t)count;
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_table_mark_unknown_device(const int32_t* d_found, int32_t* d_status, int64_t n, void* stream) {
  try {  // no C++ exception crosses the C boundary
    if (n < 0 || (n && (!d_found || !d_status))) return b2s_int_fail(B2S_ERR_INVALID, "bad arguments");
    if (n == 0) return B2S_OK;
    if (int rc = table_device_ready()) return rc;
    if (int rc = check_on_device(d_found, 4, "found", 0)) return rc;
    if (int rc = check_on_device(d_status, 4, "status", 0)) return rc;
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(4 * b2s_int_sm_count(), (n + 255) / 256));
    b2s_int_count_launches(1);
    mark_unknown_kernel<<<grid, 256, 0, stream ? (cudaStream_t)stream : b2s_int_stream()>>>(d_found, d_status, n);
    return launched("mark_unknown");
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

// ---- scoring rows held as device columns ---------------------------------------------------------------------------------
// Columns in HBM (a device ingest's result, a mapping of CUDA columns) are packed into float32 rows at the stride a
// contiguous host matrix has, so the plan picks the kernel it picks for b2s_run_host rows of that width, then scored by the
// plan's own launches.  Ranges of kColumnRangeRows rows share one scratch buffer (stream order keeps a range's pack behind
// the previous range's scoring), so a batch of any size needs at most 4 * n_in MiB of staging.
namespace {
constexpr int64_t kColumnRangeRows = 1 << 20;
}

extern "C" int b2s_run_columns_device(b2s_plan_t plan, const b2s_table_col* cols, int32_t n_cols, int64_t n_rows, void* d_out,
                                      int32_t* d_status, b2s_stats* stats, void* stream) {
  try {  // no C++ exception crosses the C boundary
    if (stats) memset(stats, 0, sizeof(*stats));
    if (!plan || !cols || n_rows < 0 || (n_rows && !d_out)) return b2s_int_fail(B2S_ERR_INVALID, "bad arguments");
    int n_in = 0, out_cols = 0;
    if (b2s_int_plan_shape(plan, &n_in, &out_cols)) return b2s_int_fail(B2S_ERR_INVALID, "plan not finalized");
    if (n_cols != n_in) return b2s_int_fail(B2S_ERR_INVALID, "%d columns, the plan takes %d", n_cols, n_in);
    std::vector<TCol> dev;
    if (int rc = check_tcols(cols, n_cols, n_rows, dev)) return rc;
    if (misaligned(d_out, 4) || misaligned(d_status, 4)) return b2s_int_fail(B2S_ERR_INVALID, "out and status must be 4-byte aligned");
    if (int rc = refuse_merging(plan)) return rc;  // a range per communicator step would split one call into several
    if (n_rows == 0) return B2S_OK;
    if (int rc = table_device_ready()) return rc;
    if (int rc = check_tcols_on_device(dev)) return rc;
    cudaStream_t st = stream ? (cudaStream_t)stream : b2s_int_stream();
    const int64_t row_bytes = (int64_t)n_in * 4, out_bytes = (int64_t)out_cols * 4;
    DeviceBlock blk(st);  // freed in stream order on every return
    const TCol* d_cols = nullptr;
    float* d_rows = nullptr;
    blk.input(d_cols, dev.data(), sizeof(TCol) * dev.size());
    blk.scratch(d_rows, (size_t)std::min(n_rows, kColumnRangeRows) * row_bytes);
    if (int rc = blk.alloc()) return rc;
    if (int rc = blk.upload()) return rc;
    Launches launches;
    const int gy = (n_in + 31) / 32;
    for (int64_t r0 = 0; r0 < n_rows; r0 += kColumnRangeRows) {
      const int64_t n = std::min(kColumnRangeRows, n_rows - r0);
      const int gx = (int)std::max<int64_t>(1, std::min<int64_t>((n + 31) / 32, ((int64_t)b2s_int_sm_count() * 8 + gy - 1) / gy));
      rows_pack_kernel<<<dim3(gx, gy), kTableThreads, 0, st>>>(d_cols, n_in, r0, n, d_rows);
      launches.add(1);
      if (int rc = launched("rows pack")) return rc;
      if (int rc = b2s_run_device(plan, d_rows, n, row_bytes, static_cast<char*>(d_out) + r0 * out_bytes,
                                  d_status ? d_status + r0 : nullptr, st))
        return rc;
      launches.n += b2s_int_plan_kernels(plan);  // b2s_run_device adds them to the library's count itself
    }
    if (stats) {
      stats->rows = n_rows;
      stats->kernels = launches.n;
    }
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}
