// b2s_pit.cu -- point-in-time correct training sets on the device, sm_90a.
//
// Replaces the local engine's get_offline_features (mlrun/feature_store/retrieval/base.py:412-468 BaseMerger.merge,
// local_merger.py:29-81 _asof_join): for each feature set, pandas.merge_asof of the entity frame onto the set's rows by
// key, taking the set's last row whose timestamp is <= the entity row's.  Here a feature set is indexed once: its rows are
// radix-sorted by (key, timestamp) on the device, their timestamps and feature words laid out in that order, and each key's
// run (start, length) recorded in an open-addressing slot array (b2s_hash.cuh).  A query sorts the entity rows by timestamp
// (stable: ties keep input order), then one launch per feature set resolves every entity row -- probe the key's run,
// binary-search it for the last timestamp <= t, gather the selected feature words into columnar outputs at the row's sorted
// position -- and permutes the entity frame's own columns into the same order.
// Bound: HBM, random row reads (one 4 * row_words-byte row per hit) plus sequential column writes.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cstring>
#include <exception>
#include <vector>

#include "../../include/b200serve.h"
#include "b2s_internal.h"
#include "b2s_pit.cuh"
#include "b2s_sort.cuh"
#include "b2s_stage.h"

using namespace b2s_pit;
using b2s::TableSlot;

namespace {

// ---- index build ----------------------------------------------------------------------------------------------------------
__global__ void gather_keys_kernel(const int64_t* __restrict__ src, const uint32_t* __restrict__ perm, uint64_t* __restrict__ dst, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = (uint64_t)src[perm[i]];
}

// rows[i] = the words of input row perm[i]: column c is (bytes[c] / 4) words from word woff[c]
struct LayoutParams {
  const void* cols[kMaxOuts];
  int32_t words[kMaxOuts];
  int32_t n_cols, row_words;
};

__global__ void layout_rows_kernel(const __grid_constant__ LayoutParams p, const uint32_t* __restrict__ perm, uint32_t* __restrict__ rows,
                                   int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = perm[i];
    uint32_t* dst = rows + i * p.row_words;
    int w = 0;
    for (int c = 0; c < p.n_cols; ++c) {
      const uint32_t* src = static_cast<const uint32_t*>(p.cols[c]) + r * p.words[c];
      for (int k = 0; k < p.words[c]; ++k) dst[w++] = src[k];
    }
  }
}

__global__ void count_runs_kernel(const uint64_t* __restrict__ keys, int64_t n, unsigned long long* __restrict__ n_runs) {
  unsigned long long c = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    c += (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
  for (int off = 16; off; off >>= 1) c += __shfl_down_sync(0xffffffffu, c, off);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(n_runs, c);
}

// every run head finds its run's end by binary search and claims a slot (keys are distinct: only the row word is contended)
__global__ void insert_runs_kernel(const uint64_t* __restrict__ keys, int64_t n, TableSlot* slots, uint64_t mask,
                                   unsigned long long* __restrict__ longest) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t k = keys[i];
    if (i > 0 && keys[i - 1] == k) continue;
    int64_t lo = i + 1, hi = n;  // first position past the run
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (keys[mid] == k) lo = mid + 1; else hi = mid;
    }
    const unsigned long long len = (unsigned long long)(lo - i);
    const unsigned long long row = ((unsigned long long)i << 32) | len;
    uint64_t h = b2s::mix64(k) & mask;
    for (;;) {
      unsigned long long* rw = reinterpret_cast<unsigned long long*>(&slots[h].row);
      if (atomicCAS(rw, ~0ull, row) == ~0ull) {
        slots[h].key = (long long)k;
        break;
      }
      h = (h + 1) & mask;
    }
    atomicMax(longest, len);
  }
}

// ---- join ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void copy_elem(const EntCol& c, int64_t dst, int64_t src) {
  switch (c.bytes) {
    case 1: static_cast<uint8_t*>(c.dst)[dst] = static_cast<const uint8_t*>(c.src)[src]; break;
    case 2: static_cast<uint16_t*>(c.dst)[dst] = static_cast<const uint16_t*>(c.src)[src]; break;
    case 4: static_cast<uint32_t*>(c.dst)[dst] = static_cast<const uint32_t*>(c.src)[src]; break;
    default: static_cast<uint64_t*>(c.dst)[dst] = static_cast<const uint64_t*>(c.src)[src]; break;
  }
}

__global__ void __launch_bounds__(256) pit_join_kernel(const __grid_constant__ JoinParams p) {
  __shared__ unsigned long long s_miss[kMaxSets];
  if (threadIdx.x < kMaxSets) s_miss[threadIdx.x] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t q = p.q0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < p.q1; q += stride) {
    const int64_t r = p.order ? (int64_t)p.order[q] : q;
    if (p.order_out) p.order_out[q] = r;
    const int64_t t = p.sorted_ts ? p.sorted_ts[q] : 0;
    for (int c = 0; c < p.n_cols; ++c) copy_elem(p.cols[c], q, r);
    const unsigned active = __activemask();
    for (int s = 0; s < p.n_sets; ++s) {
      const SetDesc& d = p.sets[s];
      const long long slot = b2s::table_find(d.slots, d.mask, d.keys[r]);
      int64_t pos = -1;
      if (slot >= 0) {
        const int64_t start = slot >> 32, len = slot & 0xffffffffll;
        if (d.asof) {  // merge_asof(direction="backward", allow_exact_matches=True): last ts <= t
          int64_t lo = start, hi = start + len;
          while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (__ldg(d.ts + mid) <= t) lo = mid + 1; else hi = mid;
          }
          pos = lo > start ? lo - 1 : -1;
        } else {
          pos = start;  // exact-key join: the index has one row per key
        }
      }
      if (d.found) d.found[q] = pos >= 0 ? 1 : 0;
      if (d.ts_out) d.ts_out[q] = pos >= 0 ? __ldg(d.ts + pos) : INT64_MIN;
      const uint32_t* row = d.rows + (pos >= 0 ? pos : 0) * d.row_words;
      for (int j = d.out0; j < d.out0 + d.n_out; ++j) {
        const OutCol& o = p.outs[j];
        if (o.bytes == 4) {
          static_cast<uint32_t*>(o.out)[q] = pos >= 0 ? row[o.src_word] : (uint32_t)o.miss;
        } else {
          const uint64_t v = pos >= 0 ? ((uint64_t)row[o.src_word] | ((uint64_t)row[o.src_word + 1] << 32)) : o.miss;
          static_cast<uint64_t*>(o.out)[q] = v;
        }
      }
      const unsigned missed = __ballot_sync(active, pos < 0);
      if (missed && lane == __ffs(active) - 1) atomicAdd(&s_miss[s], (unsigned long long)__popc(missed));
    }
  }
  __syncthreads();
  if (threadIdx.x < p.n_sets && s_miss[threadIdx.x]) atomicAdd(&p.miss[threadIdx.x], s_miss[threadIdx.x]);
}

}  // namespace

struct b2s_pit_s {
  int64_t n_rows = 0;
  int64_t n_keys = 0;
  int64_t longest_run = 0;
  int32_t row_words = 0;
  uint64_t cap = 0;
  TableSlot* d_slots = nullptr;
  int64_t* d_ts = nullptr;
  uint32_t* d_rows = nullptr;
};

extern "C" int b2s_pit_index_destroy(b2s_pit_t ix) {
  try {  // no C++ exception crosses the C boundary
    if (!ix) return B2S_OK;
    if (ix->d_slots) cudaFree(ix->d_slots);
    if (ix->d_ts) cudaFree(ix->d_ts);
    if (ix->d_rows) cudaFree(ix->d_rows);
    delete ix;
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

// Builds the index from device arrays of n rows: keys, timestamps and the feature columns (4 or 8 bytes wide).  Both
// entry points end here; the host one stages its arrays first.
static int index_build(b2s_pit_s* ix, const int64_t* d_keys, const int64_t* d_ts_in, int64_t n, const void* const* d_cols,
                       const int32_t* col_bytes, int32_t n_cols, cudaStream_t st) {
  LayoutParams lp{};
  lp.n_cols = n_cols;
  for (int c = 0; c < n_cols; ++c) {
    lp.cols[c] = d_cols[c];
    lp.words[c] = col_bytes[c] / 4;
    lp.row_words += lp.words[c];
  }
  ix->row_words = lp.row_words;
  SyncOnExit done{st};
  DeviceBlock blk(st);
  unsigned long long* d_stat = nullptr;  // [0] runs, [1] longest run
  blk.scratch(d_stat, 16);
  SortBufs sb(st);
  if (int rc = sb.alloc(n)) return rc;
  if (int rc = blk.alloc()) return rc;
  B2S_CUDA_TRY(cudaMemsetAsync(d_stat, 0, 16, st));
  B2S_CUDA_TRY(cudaMemcpyAsync(sb.k[0], d_ts_in, n * 8, cudaMemcpyDeviceToDevice, st));
  // by timestamp, then (stably) by key: rows ordered by (key, timestamp), equal pairs in input order
  Launches launches;
  if (int rc = radix_sort(sb, false, n, launches)) return rc;
  const int g = grid_for(n, 256);
  gather_keys_kernel<<<g, 256, 0, st>>>(d_keys, sb.v[0], sb.k[0], n);
  if (int rc = radix_sort(sb, true, n, launches)) return rc;
  B2S_CUDA_TRY(cudaMalloc(&ix->d_ts, n * 8));
  B2S_CUDA_TRY(cudaMalloc(&ix->d_rows, (size_t)n * std::max(lp.row_words, 1) * 4));
  gather_keys_kernel<<<g, 256, 0, st>>>(d_ts_in, sb.v[0], reinterpret_cast<uint64_t*>(ix->d_ts), n);
  layout_rows_kernel<<<g, 256, 0, st>>>(lp, sb.v[0], ix->d_rows, n);
  count_runs_kernel<<<g, 256, 0, st>>>(sb.k[0], n, d_stat);
  launches.add(4);
  unsigned long long runs = 0;
  B2S_CUDA_TRY(cudaMemcpyAsync(&runs, d_stat, 8, cudaMemcpyDeviceToHost, st));
  B2S_CUDA_TRY(cudaStreamSynchronize(st));
  uint64_t cap = 16;
  while (cap < runs * 2) cap <<= 1;  // load factor <= 0.5: table_find's walk always meets an empty slot
  ix->cap = cap;
  ix->n_keys = (int64_t)runs;
  B2S_CUDA_TRY(cudaMalloc(&ix->d_slots, cap * sizeof(TableSlot)));
  B2S_CUDA_TRY(cudaMemsetAsync(ix->d_slots, 0xff, cap * sizeof(TableSlot), st));  // row -1: empty
  insert_runs_kernel<<<g, 256, 0, st>>>(sb.k[0], n, ix->d_slots, cap - 1, d_stat + 1);
  launches.add(1);
  unsigned long long longest = 0;
  B2S_CUDA_TRY(cudaMemcpyAsync(&longest, d_stat + 1, 8, cudaMemcpyDeviceToHost, st));
  B2S_CUDA_TRY(cudaStreamSynchronize(st));
  ix->longest_run = (int64_t)longest;
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return b2s_int_fail(B2S_ERR_CUDA, "index build failed: %s", cudaGetErrorString(e));
  return B2S_OK;
}

// the host entry's first step: keys, timestamps and columns uploaded into one block, then the shared build
static int index_build_host(b2s_pit_s* ix, const int64_t* keys, const int64_t* ts, int64_t n, const void* const* cols,
                            const int32_t* col_bytes, int32_t n_cols, cudaStream_t st) {
  SyncOnExit done{st};
  DeviceBlock blk(st);
  const int64_t* d_keys = nullptr;
  const int64_t* d_ts = nullptr;
  const void* d_cols[kMaxOuts] = {};
  blk.input(d_keys, keys, (size_t)n * 8);
  blk.input(d_ts, ts, (size_t)n * 8);
  for (int c = 0; c < n_cols; ++c) blk.input(d_cols[c], cols[c], (size_t)n * col_bytes[c]);
  if (int rc = blk.alloc()) return rc;
  if (int rc = blk.upload()) return rc;
  return index_build(ix, d_keys, d_ts, n, d_cols, col_bytes, n_cols, st);
}

static int check_index_args(const int64_t* keys, const int64_t* ts_ns, int64_t n_rows, const void* const* cols, const int32_t* col_bytes,
                            int32_t n_cols, b2s_pit_t* out) {
  if (!keys || !ts_ns || !out || n_rows <= 0 || n_rows > 0x7fffffffll || n_cols < 0 || n_cols > kMaxOuts || (n_cols && (!cols || !col_bytes)))
    return b2s_int_fail(B2S_ERR_INVALID, "bad arguments");
  for (int c = 0; c < n_cols; ++c)
    if (!cols[c] || (col_bytes[c] != 4 && col_bytes[c] != 8)) return b2s_int_fail(B2S_ERR_INVALID, "column %d: null or not 4 / 8 bytes wide", c);
  if (!b2s_int_inited()) return b2s_int_fail(B2S_ERR_STATE, "b2s_init was not called (no CUDA device: there is no CPU fallback)");
  return B2S_OK;
}

using IndexBuild = int (*)(b2s_pit_s*, const int64_t*, const int64_t*, int64_t, const void* const*, const int32_t*, int32_t, cudaStream_t);

static int index_create(IndexBuild build, const int64_t* keys, const int64_t* ts_ns, int64_t n_rows, const void* const* cols,
                        const int32_t* col_bytes, int32_t n_cols, b2s_pit_t* out) {
  B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
  auto* ix = new b2s_pit_s();
  ix->n_rows = n_rows;
  if (int rc = build(ix, keys, ts_ns, n_rows, cols, col_bytes, n_cols, b2s_int_stream())) {
    b2s_pit_index_destroy(ix);
    return rc;
  }
  *out = ix;
  return B2S_OK;
}

extern "C" int b2s_pit_index_create(const int64_t* keys, const int64_t* ts_ns, int64_t n_rows, const void* const* cols,
                                    const int32_t* col_bytes, int32_t n_cols, b2s_pit_t* out) {
  try {  // no C++ exception crosses the C boundary
    if (int rc = check_index_args(keys, ts_ns, n_rows, cols, col_bytes, n_cols, out)) return rc;
    return index_create(index_build_host, keys, ts_ns, n_rows, cols, col_bytes, n_cols, out);
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_pit_index_create_device(const int64_t* d_keys, const int64_t* d_ts, int64_t n_rows, const void* const* d_cols,
                                           const int32_t* col_bytes, int32_t n_cols, b2s_pit_t* out) {
  try {  // no C++ exception crosses the C boundary
    if (int rc = check_index_args(d_keys, d_ts, n_rows, d_cols, col_bytes, n_cols, out)) return rc;
    if (int rc = check_on_device(d_keys, 8, "keys", 0)) return rc;
    if (int rc = check_on_device(d_ts, 8, "timestamps", 0)) return rc;
    for (int c = 0; c < n_cols; ++c)
      if (int rc = check_on_device(d_cols[c], col_bytes[c], "column", c)) return rc;
    return index_create(index_build, d_keys, d_ts, n_rows, d_cols, col_bytes, n_cols, out);
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_pit_index_info(b2s_pit_t ix, int64_t* n_rows, int64_t* n_keys, int64_t* longest_run, int32_t* row_words, int64_t* capacity) {
  try {  // no C++ exception crosses the C boundary
    if (!ix) return b2s_int_fail(B2S_ERR_INVALID, "null index");
    if (n_rows) *n_rows = ix->n_rows;
    if (n_keys) *n_keys = ix->n_keys;
    if (longest_run) *longest_run = ix->longest_run;
    if (row_words) *row_words = ix->row_words;
    if (capacity) *capacity = (int64_t)ix->cap;
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

static int check_sets(const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols, int32_t n_cols, const int64_t* ts, int64_t n) {
  if (n < 0 || n > 0x7fffffffll || n_sets < 0 || n_cols < 0 || (n_sets && !sets) || (n_cols && !cols))
    return b2s_int_fail(B2S_ERR_INVALID, "bad arguments");
  if (misaligned(ts, 8)) return b2s_int_fail(B2S_ERR_INVALID, "timestamps must be 8-byte aligned");
  for (int s = 0; s < n_sets; ++s) {
    const b2s_pit_set& d = sets[s];
    if (!d.index || (n && !d.keys) || d.n_out < 0 || d.n_out > kMaxOuts || (d.n_out && !d.outs))
      return b2s_int_fail(B2S_ERR_INVALID, "set %d: null index / keys / outputs", s);
    if (d.asof && !ts) return b2s_int_fail(B2S_ERR_INVALID, "set %d is an as-of join: entity timestamps are required", s);
    if (!d.asof && d.index->longest_run > 1)
      return b2s_int_fail(B2S_ERR_INVALID, "set %d: an exact-key join needs one row per key (a key has %lld)", s, (long long)d.index->longest_run);
    if (misaligned(d.keys, 8) || misaligned(d.ts_out, 8)) return b2s_int_fail(B2S_ERR_INVALID, "set %d: keys / ts_out must be 8-byte aligned", s);
    for (int j = 0; j < d.n_out; ++j) {
      const b2s_pit_out& o = d.outs[j];
      if ((o.bytes != 4 && o.bytes != 8) || o.src_word < 0 || o.src_word + o.bytes / 4 > d.index->row_words || (n && !o.out) ||
          misaligned(o.out, o.bytes))
        return b2s_int_fail(B2S_ERR_INVALID, "set %d output %d: bad width / word / pointer", s, j);
    }
  }
  for (int c = 0; c < n_cols; ++c) {
    const int b = cols[c].bytes;
    if ((b != 1 && b != 2 && b != 4 && b != 8) || (n && (!cols[c].src || !cols[c].dst)) || misaligned(cols[c].src, b) || misaligned(cols[c].dst, b))
      return b2s_int_fail(B2S_ERR_INVALID, "entity column %d: bad width / pointer", c);
  }
  return B2S_OK;
}

// sort (when ts is given) and launch the join over sorted positions [q0, q1); sets / cols hold device pointers.  Sets and
// columns beyond one launch's parameter block go to further launches over the same range.
static int launch_join(const int64_t* d_sorted_ts, const uint32_t* d_order, int64_t* d_order_out, int64_t q0, int64_t q1,
                       const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols, int32_t n_cols, unsigned long long* d_miss,
                       cudaStream_t st, Launches& launches) {
  int s = 0, c = 0;
  bool first = true;
  while (first || s < n_sets || c < n_cols) {
    JoinParams p{};
    p.sorted_ts = d_sorted_ts;
    p.order = d_order;
    p.order_out = first ? d_order_out : nullptr;
    p.q0 = q0;
    p.q1 = q1;
    p.miss = d_miss + s;
    int outs = 0;
    while (s < n_sets && p.n_sets < kMaxSets && outs + sets[s].n_out <= kMaxOuts) {
      const b2s_pit_set& d = sets[s];
      SetDesc& sd = p.sets[p.n_sets++];
      sd.slots = d.index->d_slots;
      sd.mask = d.index->cap - 1;
      sd.ts = d.index->d_ts;
      sd.rows = d.index->d_rows;
      sd.row_words = d.index->row_words;
      sd.asof = d.asof;
      sd.keys = d.keys;
      sd.ts_out = d.ts_out;
      sd.found = d.found;
      sd.out0 = outs;
      sd.n_out = d.n_out;
      for (int j = 0; j < d.n_out; ++j) p.outs[outs++] = OutCol{d.outs[j].src_word, d.outs[j].bytes, d.outs[j].miss, d.outs[j].out};
      ++s;
    }
    while (c < n_cols && p.n_cols < kMaxCols) {
      p.cols[p.n_cols++] = EntCol{cols[c].src, cols[c].dst, cols[c].bytes};
      ++c;
    }
    first = false;
    if (q1 > q0) {
      pit_join_kernel<<<grid_for(q1 - q0, 256), 256, 0, st>>>(p);
      launches.add(1);
    }
  }
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return b2s_int_fail(B2S_ERR_CUDA, "join launch failed: %s", cudaGetErrorString(e));
  return B2S_OK;
}

// Device copies of a call's descriptors over n entity rows.  Every output (each set's outputs, ts_out and found, each
// entity column's destination, the order) and, when `inputs`, every input (the timestamps, each set's keys, each entity
// column's source) gets a region of blk; blk.outputs() lists the outputs with the pointers their regions replace as
// destinations.  So do the join's miss counters.  The copies point at the regions once blk is allocated.
namespace {
struct DeviceDescs {
  DeviceDescs(DeviceBlock& blk, int64_t n, bool inputs, const int64_t* ts, const b2s_pit_set* sets, int32_t n_sets,
              const b2s_pit_col* cols, int32_t n_cols, int64_t* order)
      : ts(ts), sets(sets, sets + n_sets), outs(n_sets), cols(cols, cols + n_cols), order(order) {
    if (inputs && ts) blk.input(this->ts, ts, (size_t)n * 8);
    for (int s = 0; s < n_sets; ++s) {
      b2s_pit_set& d = this->sets[s];
      if (inputs) blk.input(d.keys, d.keys, (size_t)n * 8);
      outs[s].assign(d.outs, d.outs + d.n_out);
      d.outs = outs[s].data();
      for (b2s_pit_out& o : outs[s]) blk.output(o.out, o.out, o.bytes, n);
      if (d.ts_out) blk.output(d.ts_out, d.ts_out, 8, n);
      if (d.found) blk.output(d.found, d.found, 1, n);
    }
    for (b2s_pit_col& c : this->cols) {
      if (inputs) blk.input(c.src, c.src, (size_t)n * c.bytes);
      blk.output(c.dst, c.dst, c.bytes, n);
    }
    if (order) blk.output(this->order, order, 8, n);
    blk.scratch(miss, 8 * (size_t)std::max(n_sets, 1));
  }
  DeviceDescs(const DeviceDescs&) = delete;
  DeviceDescs& operator=(const DeviceDescs&) = delete;

  const int64_t* ts;
  std::vector<b2s_pit_set> sets;
  std::vector<std::vector<b2s_pit_out>> outs;
  std::vector<b2s_pit_col> cols;
  int64_t* order;
  unsigned long long* miss = nullptr;  // [max(n_sets, 1)]
};
}  // namespace

extern "C" int b2s_pit_join_device(const int64_t* d_ts, int64_t n, const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols,
                                   int32_t n_cols, int64_t* d_order, uint64_t* d_miss, void* stream) {
  try {  // no C++ exception crosses the C boundary
    if (int rc = check_sets(sets, n_sets, cols, n_cols, d_ts, n)) return rc;
    if (n_sets && !d_miss) return b2s_int_fail(B2S_ERR_INVALID, "null miss counters");
    if (misaligned(d_order, 8) || misaligned(d_miss, 8)) return b2s_int_fail(B2S_ERR_INVALID, "order / miss must be 8-byte aligned");
    if (n == 0) return B2S_OK;
    B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
    cudaStream_t st = stream ? (cudaStream_t)stream : b2s_int_stream();
    SortBufs sb(st);  // stays empty without timestamps: the join then reads no sorted order
    Launches launches;
    if (int rc = d_ts ? sort_keys(sb, d_ts, n, launches) : B2S_OK) return rc;
    return launch_join(reinterpret_cast<const int64_t*>(sb.k[0]), sb.v[0], d_order, 0, n, sets, n_sets, cols, n_cols,
                       reinterpret_cast<unsigned long long*>(d_miss), st, launches);
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_pit_join_host(const int64_t* ts, int64_t n, const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols,
                                 int32_t n_cols, int64_t* order, uint64_t* miss, b2s_stats* stats) {
  try {  // no C++ exception crosses the C boundary
    if (int rc = check_sets(sets, n_sets, cols, n_cols, ts, n)) return rc;
    if (n_sets && !miss) return b2s_int_fail(B2S_ERR_INVALID, "null miss counters");
    if (n == 0) {
      for (int s = 0; s < n_sets; ++s) miss[s] = 0;
      return B2S_OK;
    }
    B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
    cudaStream_t st = b2s_int_stream(), cs = b2s_int_copy_stream();
    // row ranges of sorted positions: range k's results go back on the copy stream while range k + 1 is joined
    const int64_t kRange = 1 << 20;
    const int n_ranges = (int)((n + kRange - 1) / kRange);
    Events ev, range_ev;
    if (int rc = ev.create(3)) return rc;
    if (int rc = range_ev.create(n_ranges, cudaEventDisableTiming)) return rc;
    // device mirrors of every input and output in one block, freed after the copy stream is synchronised
    SyncOnExit st_done{st};
    DeviceBlock blk(st);
    SyncOnExit cs_done{cs};  // after a failure, copies back queued on cs may still read the block
    DeviceDescs d(blk, n, true, ts, sets, n_sets, cols, n_cols, order);
    if (int rc = blk.alloc()) return rc;
    B2S_CUDA_TRY(cudaMemsetAsync(d.miss, 0, 8 * (size_t)std::max(n_sets, 1), st));
    B2S_CUDA_TRY(cudaEventRecord(ev[0], st));
    if (int rc = blk.upload()) return rc;
    B2S_CUDA_TRY(cudaEventRecord(ev[1], st));
    SortBufs sb(st);
    Launches launches;
    if (int rc = d.ts ? sort_keys(sb, d.ts, n, launches) : B2S_OK) return rc;
    for (int k = 0; k < n_ranges; ++k) {
      const int64_t q0 = (int64_t)k * kRange, q1 = std::min<int64_t>(n, q0 + kRange);
      if (int rc = launch_join(reinterpret_cast<const int64_t*>(sb.k[0]), sb.v[0], d.order, q0, q1, d.sets.data(), n_sets, d.cols.data(),
                               n_cols, d.miss, st, launches))
        return rc;
      B2S_CUDA_TRY(cudaEventRecord(range_ev[k], st));
      B2S_CUDA_TRY(cudaStreamWaitEvent(cs, range_ev[k], 0));
      if (int rc = blk.download(q0, q1, cs)) return rc;
    }
    B2S_CUDA_TRY(cudaEventRecord(ev[2], st));
    if (n_sets) B2S_CUDA_TRY(cudaMemcpyAsync(miss, d.miss, 8 * (size_t)n_sets, cudaMemcpyDeviceToHost, cs));
    B2S_CUDA_TRY(cudaStreamSynchronize(cs));
    B2S_CUDA_TRY(cudaStreamSynchronize(st));
    if (stats) {
      memset(stats, 0, sizeof(*stats));
      stats->rows = n;
      cudaEventElapsedTime(&stats->h2d_ms, ev[0], ev[1]);
      cudaEventElapsedTime(&stats->kernel_ms, ev[1], ev[2]);  // sort + join (the copies back overlap the join)
      stats->kernels = launches.n;
    }
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

// ---- training sets: the join, then the rows the reference's merge and label dropna keep, compacted in order --------------
namespace {

constexpr int kTrainSets = 64;     // sets one training-set call may join (the keep kernel reads every set's found flags)
constexpr int kTile = 1024;        // rows per block of the keep and scatter kernels: one row per thread
constexpr int kScatterCols = 64;   // arrays one scatter launch moves

struct KeepParams {
  const uint8_t* found[kTrainSets];
  int32_t exact[kTrainSets];       // 1: an inner (exact-key) join drops the rows this set misses
  int32_t n_sets;
  const uint8_t* label_found;      // the label set's found flags; null: the label is an entity column (or there is none)
  const void* label;               // the label values; null: no value test
  int32_t label_bytes, label_kind;
  int64_t n;
};

// keep[q] = the row survives every inner join and has a label; tile_count[tile] = its kept rows.  miss[s] counts the rows
// set s misses among those every earlier inner join kept (the rows of the merged frame at the set's place in the merge).
__global__ void __launch_bounds__(kTile) keep_kernel(const __grid_constant__ KeepParams p, uint8_t* __restrict__ keep,
                                                     int64_t* __restrict__ tile_count, unsigned long long* __restrict__ miss) {
  __shared__ unsigned long long s_miss[kTrainSets];
  if (threadIdx.x < kTrainSets) s_miss[threadIdx.x] = 0;
  __syncthreads();
  const int64_t q = (int64_t)blockIdx.x * kTile + threadIdx.x;
  const bool in = q < p.n;
  bool alive = in;
  for (int s = 0; s < p.n_sets; ++s) {
    const bool f = in && p.found[s][q];
    const unsigned missed = __ballot_sync(0xffffffffu, alive && !f);
    if (missed && (threadIdx.x & 31) == 0) atomicAdd(&s_miss[s], (unsigned long long)__popc(missed));
    if (p.exact[s]) alive = alive && f;
  }
  bool k = alive && (!p.label_found || p.label_found[q]);
  if (k && p.label) {
    if (p.label_kind == B2S_PIT_LABEL_NAN) {
      k = p.label_bytes == 4 ? !isnan(static_cast<const float*>(p.label)[q]) : !isnan(static_cast<const double*>(p.label)[q]);
    } else if (p.label_kind == B2S_PIT_LABEL_NAT) {
      k = static_cast<const int64_t*>(p.label)[q] != INT64_MIN;
    }
  }
  if (in) keep[q] = k ? 1 : 0;
  const int kept = __syncthreads_count(k);
  if (threadIdx.x == 0) tile_count[blockIdx.x] = kept;
  if (threadIdx.x < p.n_sets && s_miss[threadIdx.x]) atomicAdd(&miss[threadIdx.x], s_miss[threadIdx.x]);
}

// one block: tile counts -> exclusive offsets (in place), *total = the kept rows
__global__ void __launch_bounds__(1024) scan_tiles_kernel(int64_t* __restrict__ counts, int64_t n_tiles, int64_t* __restrict__ total) {
  __shared__ int64_t s_sum[1024];
  const int64_t per = (n_tiles + 1023) / 1024;
  const int64_t lo = threadIdx.x * per < n_tiles ? threadIdx.x * per : n_tiles, hi = lo + per < n_tiles ? lo + per : n_tiles;
  int64_t sum = 0;
  for (int64_t i = lo; i < hi; ++i) sum += counts[i];
  s_sum[threadIdx.x] = sum;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {  // inclusive Hillis-Steele scan of the chunk sums
    const int64_t v = threadIdx.x >= off ? s_sum[threadIdx.x - off] : 0;
    __syncthreads();
    s_sum[threadIdx.x] += v;
    __syncthreads();
  }
  int64_t run = s_sum[threadIdx.x] - sum;
  for (int64_t i = lo; i < hi; ++i) {
    const int64_t c = counts[i];
    counts[i] = run;
    run += c;
  }
  if (threadIdx.x == 1023) *total = s_sum[1023];
}

struct ScatterParams {
  const void* src[kScatterCols];
  void* dst[kScatterCols];
  int32_t bytes[kScatterCols];
  int32_t n_cols;
  int64_t n;
};

// the kept rows of every array, in order: row q goes to tile_off[tile] + its rank among the tile's kept rows
__global__ void __launch_bounds__(kTile) scatter_kernel(const __grid_constant__ ScatterParams p, const uint8_t* __restrict__ keep,
                                                        const int64_t* __restrict__ tile_off) {
  __shared__ int s_warp[kTile / 32];
  const int64_t q = (int64_t)blockIdx.x * kTile + threadIdx.x;
  const bool k = q < p.n && keep[q];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, k);
  if (lane == 0) s_warp[warp] = __popc(bal);
  __syncthreads();
  if (warp == 0) {  // exclusive scan of the 32 warp counts
    const int c = s_warp[lane];
    int v = c;
    for (int off = 1; off < 32; off <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, v, off);
      if (lane >= off) v += u;
    }
    s_warp[lane] = v - c;
  }
  __syncthreads();
  if (!k) return;
  const int64_t d = tile_off[blockIdx.x] + s_warp[warp] + __popc(bal & ((1u << lane) - 1u));
  for (int c = 0; c < p.n_cols; ++c) {
    switch (p.bytes[c]) {
      case 1: static_cast<uint8_t*>(p.dst[c])[d] = static_cast<const uint8_t*>(p.src[c])[q]; break;
      case 2: static_cast<uint16_t*>(p.dst[c])[d] = static_cast<const uint16_t*>(p.src[c])[q]; break;
      case 4: static_cast<uint32_t*>(p.dst[c])[d] = static_cast<const uint32_t*>(p.src[c])[q]; break;
      default: static_cast<uint64_t*>(p.dst[c])[d] = static_cast<const uint64_t*>(p.src[c])[q]; break;
    }
  }
}

// ---- training sets as device tensors: the kept rows of the selected columns, packed into one row-major matrix -----------
constexpr int kPackCols = 32;  // matrix columns one pack block writes: a 128-byte (float32) / 256-byte (float64) row segment

struct PackCol {
  const void* src;       // [n] the join's column, in sorted order
  const uint8_t* found;  // [n] its set's found flags (NaN where 0); null: an entity column
  int32_t bytes, kind;   // B2S_PIT_FEAT_*
};

struct PackParams {
  const PackCol* cols;  // [n_feats] device memory
  int32_t n_feats;
  void* x;              // [kept][n_feats] float / double
  PackCol label;
  void* y;              // [kept] the label (FLOAT: its width, INT / UINT: int64, BOOL: one byte); null: none
  const int64_t* order_src;
  int64_t* order;       // [kept]
  int64_t n;
};

template <class T>
__device__ __forceinline__ T nan_of();
template <>
__device__ __forceinline__ float nan_of<float>() { return __int_as_float(0x7fc00000); }
template <>
__device__ __forceinline__ double nan_of<double>() { return __longlong_as_double(0x7ff8000000000000ll); }

// element q of a column as T: C conversions, which round to nearest
template <class T>
__device__ __forceinline__ T convert(const void* src, int64_t q, int bytes, int kind) {
  switch (kind) {
    case B2S_PIT_FEAT_FLOAT:
      return bytes == 4 ? (T)static_cast<const float*>(src)[q] : (T)static_cast<const double*>(src)[q];
    case B2S_PIT_FEAT_INT:
      switch (bytes) {
        case 1: return (T)static_cast<const int8_t*>(src)[q];
        case 2: return (T)static_cast<const int16_t*>(src)[q];
        case 4: return (T)static_cast<const int32_t*>(src)[q];
        default: return (T)static_cast<const int64_t*>(src)[q];
      }
    case B2S_PIT_FEAT_UINT:
      switch (bytes) {
        case 1: return (T)static_cast<const uint8_t*>(src)[q];
        case 2: return (T)static_cast<const uint16_t*>(src)[q];
        case 4: return (T)static_cast<const uint32_t*>(src)[q];
        default: return (T)static_cast<const uint64_t*>(src)[q];
      }
    default: {  // BOOL
      bool nz;
      switch (bytes) {
        case 1: nz = static_cast<const uint8_t*>(src)[q] != 0; break;
        case 2: nz = static_cast<const uint16_t*>(src)[q] != 0; break;
        case 4: nz = static_cast<const uint32_t*>(src)[q] != 0; break;
        default: nz = static_cast<const uint64_t*>(src)[q] != 0; break;
      }
      return nz ? T(1) : T(0);
    }
  }
}

template <class T>
__device__ __forceinline__ T pack_value(const PackCol& c, int64_t q) {
  return c.found && !c.found[q] ? nan_of<T>() : convert<T>(c.src, q, c.bytes, c.kind);
}

// Block (tile, chunk): the tile's kept rows of matrix columns [32 * chunk, + 32), at tile_off[tile] onward.  Each step
// gathers rows x columns of the chunk into shared memory, a warp reading consecutive kept rows of one column, and writes
// them out along the matrix rows, so that consecutive threads write consecutive addresses (one contiguous run of the
// matrix when the chunk is the whole row).  The chunk-0 blocks also compact order and the label.
template <class T>
__global__ void __launch_bounds__(kTile) pack_kernel(const __grid_constant__ PackParams p, const uint8_t* __restrict__ keep,
                                                     const int64_t* __restrict__ tile_off) {
  __shared__ int s_warp[kTile / 32];
  __shared__ int s_row[kTile];           // the tile's kept rows in order, as offsets in the tile
  __shared__ PackCol s_col[kPackCols];
  __shared__ T s_tile[kTile + kTile / 2];  // rows x (columns | 1) with rows = kTile / columns: at most 1.5 kTile
  const int64_t q0 = (int64_t)blockIdx.x * kTile;
  const bool k = q0 + threadIdx.x < p.n && keep[q0 + threadIdx.x];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, k);
  if (lane == 0) s_warp[warp] = __popc(bal);
  const int c0 = blockIdx.y * kPackCols, cw = min(kPackCols, p.n_feats - c0);
  if ((int)threadIdx.x < cw) s_col[threadIdx.x] = p.cols[c0 + threadIdx.x];
  const int count = __syncthreads_count(k);
  if (warp == 0) {  // exclusive scan of the 32 warp counts
    const int c = s_warp[lane];
    int v = c;
    for (int off = 1; off < 32; off <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, v, off);
      if (lane >= off) v += u;
    }
    s_warp[lane] = v - c;
  }
  __syncthreads();
  if (k) s_row[s_warp[warp] + __popc(bal & ((1u << lane) - 1u))] = threadIdx.x;
  __syncthreads();
  const int64_t base = tile_off[blockIdx.x];
  if (blockIdx.y == 0 && (int)threadIdx.x < count) {
    const int64_t q = q0 + s_row[threadIdx.x], d = base + threadIdx.x;
    p.order[d] = p.order_src[q];
    if (p.y) {
      const PackCol& l = p.label;
      switch (l.kind) {
        case B2S_PIT_FEAT_FLOAT:
          if (l.bytes == 4) static_cast<float*>(p.y)[d] = static_cast<const float*>(l.src)[q];
          else static_cast<double*>(p.y)[d] = static_cast<const double*>(l.src)[q];
          break;
        case B2S_PIT_FEAT_BOOL: static_cast<uint8_t*>(p.y)[d] = convert<int>(l.src, q, l.bytes, l.kind); break;
        case B2S_PIT_FEAT_UINT: static_cast<int64_t*>(p.y)[d] = (int64_t)convert<uint64_t>(l.src, q, l.bytes, l.kind); break;
        default: static_cast<int64_t*>(p.y)[d] = convert<int64_t>(l.src, q, l.bytes, l.kind); break;
      }
    }
  }
  if (cw <= 0) return;  // no feature columns: this launch only compacts order and the label
  const int rows = kTile / cw, stride = cw | 1;  // an odd row stride: a warp's column reads hit distinct banks
  const int gr = threadIdx.x % rows, gc = threadIdx.x / rows;  // gather: lanes run down the kept rows of column gc
  const int wr = threadIdx.x / cw, wc = threadIdx.x % cw;      // write: lanes run along matrix row wr
  T* x = static_cast<T*>(p.x);
  for (int r0 = 0; r0 < count; r0 += rows) {
    const int nr = min(rows, count - r0);
    if (gc < cw && gr < nr) s_tile[gr * stride + gc] = pack_value<T>(s_col[gc], q0 + s_row[r0 + gr]);
    __syncthreads();
    if (wr < nr) x[(base + r0 + wr) * p.n_feats + c0 + wc] = s_tile[wr * stride + wc];
    __syncthreads();
  }
}

int check_train(const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols, int32_t n_cols, const int64_t* ts, int64_t n,
                const b2s_pit_label* label, const void* miss, const void* kept) {
  if (int rc = check_sets(sets, n_sets, cols, n_cols, ts, n)) return rc;
  if (n_sets > kTrainSets) return b2s_int_fail(B2S_ERR_INVALID, "%d feature sets: a training set joins at most %d", n_sets, kTrainSets);
  if ((n_sets && !miss) || !kept) return b2s_int_fail(B2S_ERR_INVALID, "null miss / kept counters");
  if (misaligned(miss, 8) || misaligned(kept, 8)) return b2s_int_fail(B2S_ERR_INVALID, "miss / kept must be 8-byte aligned");
  for (int s = 0; s < n_sets; ++s)
    if (n && !sets[s].found) return b2s_int_fail(B2S_ERR_INVALID, "set %d: a training set needs every set's found flags", s);
  if (label) {
    int bytes = 0;
    if (label->set >= 0 && label->set < n_sets && label->out >= 0 && label->out < sets[label->set].n_out)
      bytes = sets[label->set].outs[label->out].bytes;
    else if (label->set == -1 && label->out >= 0 && label->out < n_cols)
      bytes = cols[label->out].bytes;
    if (!bytes) return b2s_int_fail(B2S_ERR_INVALID, "label (set %d, output %d): no such output or entity column", label->set, label->out);
    const int k = label->kind;
    if (k != B2S_PIT_LABEL_FOUND && !(k == B2S_PIT_LABEL_NAN && (bytes == 4 || bytes == 8)) && !(k == B2S_PIT_LABEL_NAT && bytes == 8))
      return b2s_int_fail(B2S_ERR_INVALID, "label kind %d does not fit a %d-byte column", k, bytes);
  }
  return B2S_OK;
}

// What b2s_pit_train_pack asks of train_run: the matrix columns, the label vector and x_bytes; the results go to *out.
// ev: two events recorded around the pack launch (may be null).
struct Pack {
  const b2s_pit_feat* feats;
  int32_t n_feats;
  const b2s_pit_feat* label;
  int32_t x_bytes;
  b2s_pit_tensors* out;
  const cudaEvent_t* ev;
};

// The join of n rows into scratch copies of every output, then the kept rows of each into the caller's arrays (device
// memory: sets[s].outs[j].out, ts_out, found, cols[c].dst, d_order).  d_miss and *d_kept are written.  ev (may be null):
// four events recorded before the sort, after it, after the join and after the compaction.
// With `pack`, the kept rows are packed into the matrix it describes instead (pack_rows), and ev[3] is recorded before that.
int pack_rows(const Pack& pk, const DeviceDescs& d, const uint8_t* d_keep, const int64_t* d_off, const int64_t* d_kept, PackCol* d_cols,
              int64_t n, cudaStream_t st, Launches& launches);

int train_run(const int64_t* d_ts, int64_t n, const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols, int32_t n_cols,
              const b2s_pit_label* label, int64_t* d_order, unsigned long long* d_miss, int64_t* d_kept, cudaStream_t st,
              const cudaEvent_t* ev, Launches& launches, const Pack* pack = nullptr) {
  const int64_t n_tiles = (n + kTile - 1) / kTile;
  // scratch: one n-row copy of every output, the join's own miss counters, the keep flags and the tile counts
  DeviceBlock blk(st);
  DeviceDescs d(blk, n, false, d_ts, sets, n_sets, cols, n_cols, d_order);
  uint8_t* d_keep = nullptr;
  int64_t* d_count = nullptr;
  blk.scratch(d_keep, (size_t)n);
  blk.scratch(d_count, (size_t)n_tiles * 8);
  PackCol* d_pack_cols = nullptr;
  if (pack) blk.scratch(d_pack_cols, sizeof(PackCol) * (size_t)std::max(pack->n_feats, 1));
  if (int rc = blk.alloc()) return rc;
  B2S_CUDA_TRY(cudaMemsetAsync(d.miss, 0, 8 * (size_t)std::max(n_sets, 1), st));
  if (n_sets) B2S_CUDA_TRY(cudaMemsetAsync(d_miss, 0, 8 * (size_t)n_sets, st));
  if (ev) B2S_CUDA_TRY(cudaEventRecord(ev[0], st));
  SortBufs sb(st);
  if (int rc = d_ts ? sort_keys(sb, d_ts, n, launches) : B2S_OK) return rc;
  if (ev) B2S_CUDA_TRY(cudaEventRecord(ev[1], st));
  if (int rc = launch_join(reinterpret_cast<const int64_t*>(sb.k[0]), sb.v[0], d.order, 0, n, d.sets.data(), n_sets, d.cols.data(), n_cols,
                           d.miss, st, launches))
    return rc;
  if (ev) B2S_CUDA_TRY(cudaEventRecord(ev[2], st));
  KeepParams kp{};
  kp.n_sets = n_sets;
  kp.n = n;
  for (int s = 0; s < n_sets; ++s) {
    kp.found[s] = d.sets[s].found;
    kp.exact[s] = sets[s].asof ? 0 : 1;
  }
  if (label) {
    kp.label_kind = label->kind;
    if (label->set >= 0) {
      kp.label_found = d.sets[label->set].found;
      kp.label = d.outs[label->set][label->out].out;
      kp.label_bytes = d.outs[label->set][label->out].bytes;
    } else {
      kp.label = d.cols[label->out].dst;
      kp.label_bytes = d.cols[label->out].bytes;
    }
    if (kp.label_kind == B2S_PIT_LABEL_FOUND) kp.label = nullptr;
  }
  keep_kernel<<<(unsigned)n_tiles, kTile, 0, st>>>(kp, d_keep, d_count, d_miss);
  scan_tiles_kernel<<<1, 1024, 0, st>>>(d_count, n_tiles, d_kept);
  launches.add(2);
  if (pack) {
    if (ev) B2S_CUDA_TRY(cudaEventRecord(ev[3], st));
    return pack_rows(*pack, d, d_keep, d_count, d_kept, d_pack_cols, n, st, launches);
  }
  // each scratch copy's kept rows go to the array it stands for
  const std::vector<DeviceBlock::Out>& moves = blk.outputs();
  for (size_t i = 0; i < moves.size(); i += kScatterCols) {
    ScatterParams sp{};
    sp.n = n;
    for (size_t j = i; j < moves.size() && sp.n_cols < kScatterCols; ++j, ++sp.n_cols) {
      sp.src[sp.n_cols] = blk.at(moves[j].off);
      sp.dst[sp.n_cols] = moves[j].dst;
      sp.bytes[sp.n_cols] = (int32_t)moves[j].elem;
    }
    scatter_kernel<<<(unsigned)n_tiles, kTile, 0, st>>>(sp, d_keep, d_count);
    launches.add(1);
  }
  if (ev) B2S_CUDA_TRY(cudaEventRecord(ev[3], st));
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return b2s_int_fail(B2S_ERR_CUDA, "training-set launch failed: %s", cudaGetErrorString(e));
  return B2S_OK;
}

}  // namespace

extern "C" int b2s_pit_train_device(const int64_t* d_ts, int64_t n, const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols,
                                    int32_t n_cols, const b2s_pit_label* label, int64_t* d_order, uint64_t* d_miss, int64_t* d_kept,
                                    void* stream) {
  try {  // no C++ exception crosses the C boundary
    if (int rc = check_train(sets, n_sets, cols, n_cols, d_ts, n, label, d_miss, d_kept)) return rc;
    if (misaligned(d_order, 8)) return b2s_int_fail(B2S_ERR_INVALID, "order must be 8-byte aligned");
    B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
    cudaStream_t st = stream ? (cudaStream_t)stream : b2s_int_stream();
    if (n == 0) {
      B2S_CUDA_TRY(cudaMemsetAsync(d_kept, 0, 8, st));
      if (n_sets) B2S_CUDA_TRY(cudaMemsetAsync(d_miss, 0, 8 * (size_t)n_sets, st));
      return B2S_OK;
    }
    Launches launches;
    return train_run(d_ts, n, sets, n_sets, cols, n_cols, label, d_order, reinterpret_cast<unsigned long long*>(d_miss), d_kept, st,
                     nullptr, launches);
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_pit_train_host(const int64_t* ts, int64_t n, const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols,
                                  int32_t n_cols, const b2s_pit_label* label, int64_t* order, uint64_t* miss, int64_t* kept,
                                  float* phase_ms, b2s_stats* stats) {
  try {  // no C++ exception crosses the C boundary
    if (int rc = check_train(sets, n_sets, cols, n_cols, ts, n, label, miss, kept)) return rc;
    if (n == 0) {
      *kept = 0;
      for (int s = 0; s < n_sets; ++s) miss[s] = 0;
      if (phase_ms) phase_ms[0] = phase_ms[1] = phase_ms[2] = 0.f;
      if (stats) memset(stats, 0, sizeof(*stats));
      return B2S_OK;
    }
    B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
    cudaStream_t st = b2s_int_stream();
    Events ev;
    if (int rc = ev.create(6)) return rc;
    // one device block: every input, then every output's kept rows (n rows reserved), the counters
    SyncOnExit done{st};
    DeviceBlock blk(st);
    DeviceDescs d(blk, n, true, ts, sets, n_sets, cols, n_cols, order);
    int64_t* d_kept = nullptr;
    blk.scratch(d_kept, 8);
    if (int rc = blk.alloc()) return rc;
    B2S_CUDA_TRY(cudaEventRecord(ev[0], st));
    if (int rc = blk.upload()) return rc;
    Launches launches;
    if (int rc = train_run(d.ts, n, d.sets.data(), n_sets, d.cols.data(), n_cols, label, d.order, d.miss, d_kept, st, ev.data() + 1, launches))
      return rc;
    B2S_CUDA_TRY(cudaMemcpyAsync(kept, d_kept, 8, cudaMemcpyDeviceToHost, st));
    if (n_sets) B2S_CUDA_TRY(cudaMemcpyAsync(miss, d.miss, 8 * (size_t)n_sets, cudaMemcpyDeviceToHost, st));
    B2S_CUDA_TRY(cudaStreamSynchronize(st));
    // only the kept rows come back, in ranges of 1 Mi rows
    const int64_t kRange = 1 << 20;
    for (int64_t q0 = 0; q0 < *kept; q0 += kRange)
      if (int rc = blk.download(q0, std::min<int64_t>(*kept, q0 + kRange), st)) return rc;
    B2S_CUDA_TRY(cudaEventRecord(ev[5], st));
    B2S_CUDA_TRY(cudaStreamSynchronize(st));
    if (phase_ms) {
      cudaEventElapsedTime(&phase_ms[0], ev[1], ev[2]);  // sort
      cudaEventElapsedTime(&phase_ms[1], ev[2], ev[3]);  // join
      cudaEventElapsedTime(&phase_ms[2], ev[3], ev[4]);  // compaction
    }
    if (stats) {
      memset(stats, 0, sizeof(*stats));
      stats->rows = n;
      cudaEventElapsedTime(&stats->h2d_ms, ev[0], ev[1]);
      cudaEventElapsedTime(&stats->kernel_ms, ev[1], ev[4]);
      cudaEventElapsedTime(&stats->d2h_ms, ev[4], ev[5]);
      stats->kernels = launches.n;
    }
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

// ---- training sets as device tensors ---------------------------------------------------------------------------------
struct b2s_darray_s {
  void* ptr;
  int64_t bytes;
  std::atomic<int> refs{1};
  b2s_darray_s* base = nullptr;  // a view holds one reference on the array that owns its memory
};

namespace {

std::atomic<int64_t> g_darrays{0};  // arrays not yet freed (b2s_darray_live)
// the destination of every output b2s_pit_train_pack joins: train_run gives each a scratch region and never writes here
alignas(8) char g_stand_in[8];

int darray_new(b2s_darray_t& a, int64_t bytes) {
  void* p = nullptr;
  B2S_CUDA_TRY(cudaMalloc(&p, (size_t)std::max<int64_t>(bytes, 1)));  // never null: an empty array still has an address
  a = new b2s_darray_s();
  a->ptr = p;
  a->bytes = bytes;
  ++g_darrays;
  return B2S_OK;
}

void darray_unref(b2s_darray_t a) {
  if (a && a->refs.fetch_sub(1) == 1) {
    if (a->base) darray_unref(a->base);
    else cudaFree(a->ptr);
    delete a;
    --g_darrays;
  }
}

// the DLPack ABI (dlpack.h, unversioned DLManagedTensor)
struct DLDevice {
  int32_t device_type;  // kDLCUDA = 2
  int32_t device_id;
};
struct DLDataType {
  uint8_t code;  // kDLInt 0, kDLUInt 1, kDLFloat 2, kDLBool 6
  uint8_t bits;
  uint16_t lanes;
};
struct DLTensor {
  void* data;
  DLDevice device;
  int32_t ndim;
  DLDataType dtype;
  int64_t* shape;
  int64_t* strides;  // null: compact row-major
  uint64_t byte_offset;
};
struct DLManagedTensor {
  DLTensor dl_tensor;
  void* manager_ctx;
  void (*deleter)(DLManagedTensor* self);
};
struct Managed {
  DLManagedTensor m;
  b2s_darray_t array;
  int64_t shape[8];
};

void dlpack_deleter(DLManagedTensor* self) {
  Managed* h = static_cast<Managed*>(self->manager_ctx);
  darray_unref(h->array);
  delete h;
}

void release_tensors(b2s_pit_tensors& t) {
  darray_unref(t.features);
  darray_unref(t.label);
  darray_unref(t.order);
  t = b2s_pit_tensors{};
}

int label_vec_bytes(const b2s_pit_feat& f) {
  return f.kind == B2S_PIT_FEAT_FLOAT ? f.bytes : f.kind == B2S_PIT_FEAT_BOOL ? 1 : 8;
}

PackCol pack_source(const DeviceDescs& d, const b2s_pit_feat& f) {
  if (f.set >= 0) return PackCol{d.outs[f.set][f.out].out, d.sets[f.set].found, f.bytes, f.kind};
  return PackCol{d.cols[f.out].dst, nullptr, f.bytes, f.kind};
}

}  // namespace

namespace {

// the matrix, order and label of the kept rows: allocated once *d_kept is known, then one pack launch
int pack_rows(const Pack& pk, const DeviceDescs& d, const uint8_t* d_keep, const int64_t* d_off, const int64_t* d_kept, PackCol* d_cols,
              int64_t n, cudaStream_t st, Launches& launches) {
  int64_t kept = 0;
  B2S_CUDA_TRY(cudaMemcpyAsync(&kept, d_kept, 8, cudaMemcpyDeviceToHost, st));
  B2S_CUDA_TRY(cudaStreamSynchronize(st));
  b2s_pit_tensors& o = *pk.out;
  o.kept = kept;
  if (int rc = darray_new(o.features, kept * pk.n_feats * pk.x_bytes)) return rc;
  if (int rc = darray_new(o.order, kept * 8)) return rc;
  if (pk.label)
    if (int rc = darray_new(o.label, kept * label_vec_bytes(*pk.label))) return rc;
  std::vector<PackCol> cols(pk.n_feats);
  for (int i = 0; i < pk.n_feats; ++i) cols[i] = pack_source(d, pk.feats[i]);
  if (pk.n_feats) B2S_CUDA_TRY(cudaMemcpyAsync(d_cols, cols.data(), sizeof(PackCol) * cols.size(), cudaMemcpyHostToDevice, st));
  PackParams p{};
  p.cols = d_cols;
  p.n_feats = pk.n_feats;
  p.x = o.features->ptr;
  if (pk.label) {
    p.label = pack_source(d, *pk.label);
    p.y = o.label->ptr;
  }
  p.order_src = d.order;
  p.order = static_cast<int64_t*>(o.order->ptr);
  p.n = n;
  const dim3 grid((unsigned)((n + kTile - 1) / kTile), (unsigned)std::max(1, (pk.n_feats + kPackCols - 1) / kPackCols));
  if (pk.ev) B2S_CUDA_TRY(cudaEventRecord(pk.ev[0], st));
  if (pk.x_bytes == 4) pack_kernel<float><<<grid, kTile, 0, st>>>(p, d_keep, d_off);
  else pack_kernel<double><<<grid, kTile, 0, st>>>(p, d_keep, d_off);
  launches.add(1);
  if (pk.ev) B2S_CUDA_TRY(cudaEventRecord(pk.ev[1], st));
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return b2s_int_fail(B2S_ERR_CUDA, "pack launch failed: %s", cudaGetErrorString(e));
  return B2S_OK;
}

int check_feat(const b2s_pit_feat& f, const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols, int32_t n_cols, const char* what,
               int i) {
  int width = 0;
  if (f.set >= 0 && f.set < n_sets && f.out >= 0 && f.out < sets[f.set].n_out)
    width = sets[f.set].outs[f.out].bytes;
  else if (f.set == -1 && f.out >= 0 && f.out < n_cols)
    width = cols[f.out].bytes;
  if (!width) return b2s_int_fail(B2S_ERR_INVALID, "%s %d (set %d, output %d): no such output or entity column", what, i, f.set, f.out);
  const bool fits = f.kind == B2S_PIT_FEAT_FLOAT ? (f.bytes == 4 || f.bytes == 8)
                                                  : (f.kind == B2S_PIT_FEAT_INT || f.kind == B2S_PIT_FEAT_UINT || f.kind == B2S_PIT_FEAT_BOOL);
  if (f.bytes != width || !fits)
    return b2s_int_fail(B2S_ERR_INVALID, "%s %d: kind %d of %d bytes does not fit a %d-byte source", what, i, f.kind, f.bytes, width);
  return B2S_OK;
}

}  // namespace

namespace {

// n = 0: empty arrays, no launch
int pack_empty(b2s_pit_tensors& out, bool label) {
  if (int rc = darray_new(out.features, 0)) return rc;
  if (int rc = darray_new(out.order, 0)) return rc;
  return label ? darray_new(out.label, 0) : B2S_OK;
}

// b2s_pit_train_pack over n > 0 rows: sets / cols are checked descriptors whose destinations are stand-ins and whose
// inputs (d_ts, each set's keys, each column's source) are device memory.  Both entry points end here; the host one
// stages its inputs first.
int pack_call(const int64_t* d_ts, int64_t n, b2s_pit_set* sets, int32_t n_sets, b2s_pit_col* cols, int32_t n_cols,
              const b2s_pit_label* label, Pack pk, float* phase_ms, b2s_stats* stats) {
  cudaStream_t st = b2s_int_stream();
  Events ev;
  if (int rc = ev.create(6)) return rc;
  pk.ev = ev.data() + 4;
  Launches launches;
  {
    // the counters: the outputs are train_run's scratch
    SyncOnExit done{st};
    DeviceBlock blk(st);
    unsigned long long* d_miss = nullptr;
    int64_t* d_kept = nullptr;
    blk.scratch(d_miss, 8 * (size_t)std::max(n_sets, 1));
    blk.scratch(d_kept, 8);
    if (int rc = blk.alloc()) return rc;
    if (int rc = train_run(d_ts, n, sets, n_sets, cols, n_cols, label, reinterpret_cast<int64_t*>(g_stand_in),
                           d_miss, d_kept, st, ev.data(), launches, &pk))
      return rc;
  }
  B2S_CUDA_TRY(cudaStreamSynchronize(st));
  float keep_ms = 0.f, pack_ms = 0.f;
  cudaEventElapsedTime(&keep_ms, ev[2], ev[3]);  // keep + scan
  cudaEventElapsedTime(&pack_ms, ev[4], ev[5]);
  if (phase_ms) {
    cudaEventElapsedTime(&phase_ms[0], ev[0], ev[1]);  // sort
    cudaEventElapsedTime(&phase_ms[1], ev[1], ev[2]);  // join
    phase_ms[2] = keep_ms + pack_ms;                   // compaction (the host reads kept between the two)
    phase_ms[3] = pack_ms;
  }
  if (stats) {
    stats->rows = n;
    cudaEventElapsedTime(&stats->kernel_ms, ev[0], ev[3]);
    stats->kernel_ms += pack_ms;
    stats->kernels = launches.n;
  }
  return B2S_OK;
}

// the host entry's first step: the timestamps, keys and entity columns uploaded into one block, then pack_call
int pack_call_host(const int64_t* ts, int64_t n, b2s_pit_set* sets, int32_t n_sets, b2s_pit_col* cols, int32_t n_cols,
                   const b2s_pit_label* label, Pack pk, float* phase_ms, b2s_stats* stats) {
  cudaStream_t st = b2s_int_stream();
  Events ev;
  if (int rc = ev.create(2)) return rc;
  SyncOnExit done{st};
  DeviceBlock blk(st);
  const int64_t* d_ts = nullptr;
  if (ts) blk.input(d_ts, ts, (size_t)n * 8);
  for (int s = 0; s < n_sets; ++s) blk.input(sets[s].keys, sets[s].keys, (size_t)n * 8);
  for (int c = 0; c < n_cols; ++c) blk.input(cols[c].src, cols[c].src, (size_t)n * cols[c].bytes);
  if (int rc = blk.alloc()) return rc;
  B2S_CUDA_TRY(cudaEventRecord(ev[0], st));
  if (int rc = blk.upload()) return rc;
  B2S_CUDA_TRY(cudaEventRecord(ev[1], st));
  if (int rc = pack_call(d_ts, n, sets, n_sets, cols, n_cols, label, pk, phase_ms, stats)) return rc;
  if (stats) cudaEventElapsedTime(&stats->h2d_ms, ev[0], ev[1]);  // pack_call has synchronised the stream
  return B2S_OK;
}

using PackRun = int (*)(const int64_t*, int64_t, b2s_pit_set*, int32_t, b2s_pit_col*, int32_t, const b2s_pit_label*, Pack, float*,
                        b2s_stats*);

// Both b2s_pit_train_pack entries: the checks, then `run` over n > 0 rows (on_device: ts, keys and sources must be memory
// of the library's device).
int train_pack(PackRun run, bool on_device, const int64_t* ts, int64_t n, const b2s_pit_set* sets, int32_t n_sets,
               const b2s_pit_col* cols, int32_t n_cols, const b2s_pit_label* label, const b2s_pit_feat* feats, int32_t n_feats,
               const b2s_pit_feat* label_vec, int32_t x_bytes, b2s_pit_tensors* out, float* phase_ms, b2s_stats* stats) {
  if (!out || n_sets < 0 || n_cols < 0 || n_feats < 0 || (n_sets && !sets) || (n_cols && !cols) || (n_feats && !feats))
    return b2s_int_fail(B2S_ERR_INVALID, "bad arguments");
  if (x_bytes != 4 && x_bytes != 8) return b2s_int_fail(B2S_ERR_INVALID, "x_bytes %d: the matrix is float32 (4) or float64 (8)", x_bytes);
  *out = b2s_pit_tensors{};
  // every output, found flag and entity destination lives in scratch: the checks of b2s_pit_train_host run on copies
  // whose destinations stand in for those regions
  std::vector<b2s_pit_set> s2(sets, sets + n_sets);
  std::vector<std::vector<b2s_pit_out>> o2(n_sets);
  for (int s = 0; s < n_sets; ++s) {
    if (s2[s].n_out < 0 || s2[s].n_out > kMaxOuts || (s2[s].n_out && !s2[s].outs))
      return b2s_int_fail(B2S_ERR_INVALID, "set %d: null index / keys / outputs", s);
    o2[s].assign(s2[s].outs, s2[s].outs + s2[s].n_out);
    for (b2s_pit_out& o : o2[s]) o.out = g_stand_in;
    s2[s].outs = o2[s].data();
    s2[s].found = reinterpret_cast<uint8_t*>(g_stand_in);
    s2[s].ts_out = nullptr;
  }
  std::vector<b2s_pit_col> c2(cols, cols + n_cols);
  for (b2s_pit_col& c : c2) c.dst = g_stand_in;
  int64_t counters[2];
  if (int rc = check_train(s2.data(), n_sets, c2.data(), n_cols, ts, n, label, counters, counters + 1)) return rc;
  for (int i = 0; i < n_feats; ++i)
    if (int rc = check_feat(feats[i], s2.data(), n_sets, c2.data(), n_cols, "feature", i)) return rc;
  if (label_vec)
    if (int rc = check_feat(*label_vec, s2.data(), n_sets, c2.data(), n_cols, "label", 0)) return rc;
  if (phase_ms) phase_ms[0] = phase_ms[1] = phase_ms[2] = phase_ms[3] = 0.f;
  if (stats) memset(stats, 0, sizeof(*stats));
  if (!b2s_int_inited()) return b2s_int_fail(B2S_ERR_STATE, "b2s_init was not called (no CUDA device: there is no CPU fallback)");
  if (on_device && n) {
    if (ts)
      if (int rc = check_on_device(ts, 8, "timestamps", 0)) return rc;
    for (int s = 0; s < n_sets; ++s)
      if (int rc = check_on_device(s2[s].keys, 8, "keys of set", s)) return rc;
    for (int c = 0; c < n_cols; ++c)
      if (int rc = check_on_device(c2[c].src, c2[c].bytes, "entity column", c)) return rc;
  }
  B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
  const int rc = n ? run(ts, n, s2.data(), n_sets, c2.data(), n_cols, label, Pack{feats, n_feats, label_vec, x_bytes, out, nullptr},
                         phase_ms, stats)
                   : pack_empty(*out, label_vec != nullptr);
  if (rc) release_tensors(*out);
  return rc;
}

}  // namespace

extern "C" int b2s_darray_info(b2s_darray_t a, void** ptr, int64_t* bytes) {
  if (!a) return b2s_int_fail(B2S_ERR_INVALID, "null array");
  if (ptr) *ptr = a->ptr;
  if (bytes) *bytes = a->bytes;
  return B2S_OK;
}

extern "C" int b2s_darray_release(b2s_darray_t a) {
  darray_unref(a);
  return B2S_OK;
}

extern "C" void* b2s_darray_dlpack(b2s_darray_t a, int32_t ndim, const int64_t* shape, int32_t code, int32_t bits) {
  try {  // no C++ exception crosses the C boundary
    if (!a || ndim < 0 || ndim > 8 || (ndim && !shape) || code < 0 || code > 255 || bits <= 0 || bits % 8) {
      b2s_int_fail(B2S_ERR_INVALID, "bad arguments");
      return nullptr;
    }
    int64_t elems = 1;
    for (int i = 0; i < ndim; ++i) elems = shape[i] < 0 ? -1 : elems * shape[i];
    if (elems < 0 || elems * (bits / 8) > a->bytes) {
      b2s_int_fail(B2S_ERR_INVALID, "the shape does not fit the array's %lld bytes", (long long)a->bytes);
      return nullptr;
    }
    Managed* h = new Managed();
    for (int i = 0; i < ndim; ++i) h->shape[i] = shape[i];
    h->array = a;
    a->refs.fetch_add(1);
    DLTensor& t = h->m.dl_tensor;
    t.data = a->ptr;
    t.device = DLDevice{2, b2s_int_device()};
    t.ndim = ndim;
    t.dtype = DLDataType{(uint8_t)code, (uint8_t)bits, 1};
    t.shape = h->shape;
    h->m.manager_ctx = h;
    h->m.deleter = dlpack_deleter;
    return &h->m;
  } catch (const std::exception& e) {
    b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
    return nullptr;
  }
}

extern "C" int b2s_dlpack_delete(void* managed) {
  DLManagedTensor* m = static_cast<DLManagedTensor*>(managed);
  if (m && m->deleter) m->deleter(m);
  return B2S_OK;
}

extern "C" int64_t b2s_darray_live(void) { return g_darrays.load(); }

extern "C" int b2s_darray_alloc(int64_t bytes, int32_t zero, b2s_darray_t* out) {
  try {  // no C++ exception crosses the C boundary
    if (!out || bytes < 0) return b2s_int_fail(B2S_ERR_INVALID, "null out or negative size");
    *out = nullptr;
    if (!b2s_int_inited()) return b2s_int_fail(B2S_ERR_STATE, "b2s_init was not called (no CUDA device: there is no CPU fallback)");
    B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
    b2s_darray_t a = nullptr;
    if (int rc = darray_new(a, bytes)) return rc;
    if (zero && bytes) {
      const cudaError_t e = cudaMemsetAsync(a->ptr, 0, (size_t)bytes, b2s_int_stream());
      if (e != cudaSuccess) {
        darray_unref(a);
        return b2s_int_fail(B2S_ERR_CUDA, "cudaMemsetAsync failed: %s", cudaGetErrorString(e));
      }
    }
    *out = a;
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_darray_view(b2s_darray_t base, int64_t offset, int64_t bytes, b2s_darray_t* out) {
  try {  // no C++ exception crosses the C boundary
    if (!out) return b2s_int_fail(B2S_ERR_INVALID, "null out");
    *out = nullptr;
    if (!base || offset < 0 || bytes < 0 || offset % 8 || offset > base->bytes || bytes > base->bytes - offset)
      return b2s_int_fail(B2S_ERR_INVALID, "view [%lld, +%lld) of a %lld-byte array: outside it, or not 8-byte aligned", (long long)offset,
                          (long long)bytes, base ? (long long)base->bytes : 0ll);
    b2s_darray_t v = new b2s_darray_s();
    v->ptr = static_cast<char*>(base->ptr) + offset;
    v->bytes = bytes;
    v->base = base;
    base->refs.fetch_add(1);
    ++g_darrays;
    *out = v;
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_pit_train_pack(const int64_t* ts, int64_t n, const b2s_pit_set* sets, int32_t n_sets, const b2s_pit_col* cols,
                                  int32_t n_cols, const b2s_pit_label* label, const b2s_pit_feat* feats, int32_t n_feats,
                                  const b2s_pit_feat* label_vec, int32_t x_bytes, b2s_pit_tensors* out, float* phase_ms,
                                  b2s_stats* stats) {
  try {  // no C++ exception crosses the C boundary
    return train_pack(pack_call_host, false, ts, n, sets, n_sets, cols, n_cols, label, feats, n_feats, label_vec, x_bytes, out, phase_ms,
                      stats);
  } catch (const std::exception& e) {
    if (out) release_tensors(*out);
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_pit_train_pack_device(const int64_t* d_ts, int64_t n, const b2s_pit_set* sets, int32_t n_sets,
                                         const b2s_pit_col* cols, int32_t n_cols, const b2s_pit_label* label, const b2s_pit_feat* feats,
                                         int32_t n_feats, const b2s_pit_feat* label_vec, int32_t x_bytes, b2s_pit_tensors* out,
                                         float* phase_ms, b2s_stats* stats) {
  try {  // no C++ exception crosses the C boundary
    return train_pack(pack_call, true, d_ts, n, sets, n_sets, cols, n_cols, label, feats, n_feats, label_vec, x_bytes, out, phase_ms,
                      stats);
  } catch (const std::exception& e) {
    if (out) release_tensors(*out);
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}
