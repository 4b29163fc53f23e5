// b2s_columns.cuh -- columnar feature-set transforms (sm_90a): the device side of the ingest path.
//
// Replaces, for DataFrame-shaped input, the reference's row-at-a-time walk of the feature-set graph
// (feature_store/ingestion.py:38-127: DataFrame -> storey.DataframeSource -> one dict per row -> Imputer /
// MapValues / OneHotEncoder / DateExtractor / DropFeatures / FeaturesetValidator -> ReduceToDataFrame).
// Data stays COLUMNAR end to end, as a DataFrame already is: an input "slot" is n_rows 4-byte words (float32 or
// int32; an int64 column is two adjacent slots), an output slot likewise.  The lowered graph is a list of
// column ops, each reading one input column and writing 0..n output columns; a work item is (op, chunk of
// rows); persistent CTAs take items round-robin, so neighbouring CTAs stream different columns of the same
// row range.  Every access is a fully coalesced 16-byte-per-lane load/store (4-byte on ragged tails): each input word is
// read once, each output word written once -- the kernel is a pure HBM stream.
// Compares run in fp64 against fp64 tables: float32/int32 values convert exactly, so range edges and category
// matches agree bit for bit with the reference's Python comparisons.  Violations / unmatched values are counted
// per op with one atomic per CTA-item (the reference only prints them).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "b2s_dates.cuh"

namespace b2s {

enum ColKind : int32_t {
  CK_COPY32 = 0,  // 4-byte word, no interpretation (int32 counters, codes)
  CK_COPY64 = 1,  // 8-byte word (timestamps kept in the output)
  CK_F32 = 2,     // float32 with Imputer fill
  CK_RANGE = 3,   // MapValues ranges: first lo <= v < hi -> val, else v passes through (counted)
  CK_VALUE = 4,   // MapValues dict: v == key -> val, else v passes through (counted)
  CK_ONEHOT = 5,  // OneHotEncoder: n int32 0/1 columns
  CK_DATE = 6,    // DateExtractor part of an int64 nanosecond timestamp -> int32
  CK_CHECK = 7,   // validator only (column dropped from the output but still checked)
};

struct ColOp {
  int32_t kind;
  int32_t src;       // input slot
  int32_t dst;       // first output slot (-1: none)
  int32_t n;         // table entries / categories
  int32_t src_int;   // source words are int32 (never missing)
  int32_t has_fill;  // Imputer value for a missing (NaN) float source, applied before anything else
  float fill;
  union {            // (a union keeps ColOp at 64 bytes: four 16-byte loads per item)
    int32_t part;     // CK_DATE
    int32_t int_out;  // CK_RANGE / CK_VALUE: int32 output words (int32 source, every value an int32 integer), else float32
  };
  int32_t tab;       // offset (doubles) into the table array: RANGE lo[n] hi[n] val[n]; VALUE key[n] val[n]; ONEHOT cat[n]
  int32_t check;     // bit 0: min, bit 1: max  (MinMaxValidator.check, mlrun/features.py:292-321)
  int32_t counter;   // counters[counter] += rows violating the check
  int32_t miss;      // counters[miss] += rows that matched no range / key (RANGE, VALUE) or were NaT (DATE); -1: none
  double cmin, cmax;
};

static_assert(sizeof(ColOp) == 64, "ColOp is loaded as four 16-byte words");

struct ColParams {
  const char* in;   // input slots: slot s starts at in + s * in_stride
  int64_t in_stride;
  char* out;
  int64_t out_stride;
  int64_t n_rows;     // rows of this launch: [row_begin, row_begin + n_rows) of the slots
  const ColOp* ops;
  int32_t n_ops;
  const double* tab;
  unsigned long long* counters;
  int64_t row_begin;  // a multiple of kColChunk (the host path pipelines a frame in row ranges)
};

#ifndef B2S_COL_THREADS
#define B2S_COL_THREADS 256
#endif
#ifndef B2S_COL_UNROLL
#define B2S_COL_UNROLL 4
#endif
constexpr int kColThreads = B2S_COL_THREADS;
constexpr int kColVec = 4;                                  // rows per 16-byte access
constexpr int kColUnroll = B2S_COL_UNROLL;                  // independent 16-byte loads in flight per thread
constexpr int kColChunk = kColThreads * kColUnroll * kColVec;  // rows per work item (4096)

// one 4-byte source word -> the op's outputs (shared by the vector and the tail paths)
__device__ __forceinline__ uint32_t col_word(const ColOp& op, const double* __restrict__ tab, uint32_t bits, double& x, bool& hit) {
  hit = true;
  if (op.src_int) {
    x = (double)(int32_t)bits;
  } else {
    float f = __uint_as_float(bits);
    if (op.has_fill && f != f) f = op.fill;  // Imputer._impute (steps.py:397-406)
    bits = __float_as_uint(f);
    x = (double)f;
  }
  if (op.kind == CK_RANGE) {  // MapValues._map_value (steps.py:189-201): first match in mapping order wins
    double val = x;
    hit = false;
    for (int q = op.n - 1; q >= 0; --q) {
      const bool in = x >= tab[q] && x < tab[op.n + q];
      val = in ? tab[2 * op.n + q] : val;
      hit |= in;
    }
    x = val;
    bits = op.int_out ? (uint32_t)(int32_t)val : __float_as_uint((float)val);
  } else if (op.kind == CK_VALUE) {
    double val = x;
    hit = false;
    for (int q = op.n - 1; q >= 0; --q) {
      const bool in = x == tab[q];
      val = in ? tab[op.n + q] : val;
      hit |= in;
    }
    x = val;
    bits = op.int_out ? (uint32_t)(int32_t)val : __float_as_uint((float)val);
  }
  return bits;
}

__device__ __forceinline__ unsigned int col_check(const ColOp& op, double x) {
  const bool lo_bad = (op.check & 1) && x < op.cmin;
  const bool hi_bad = (op.check & 2) && x > op.cmax;
  return (lo_bad || hi_bad) ? 1u : 0u;
}

// ---- per-kind item bodies.  They are separate (non-inlined) functions so that the instruction footprint a CTA touches
// is the body of the op it is working on (plain copies and imputed floats are ~85 % of a typical plan), not the union.

// CK_COPY32 without a check: a 16-byte stream copy
__device__ __noinline__ void item_copy32(const uint32_t* __restrict__ s, uint32_t* __restrict__ d, int rows, int quads, int tid) {
  for (int base = tid; base < quads; base += kColThreads * kColUnroll) {
    uint4 w[kColUnroll];
#pragma unroll
    for (int u = 0; u < kColUnroll; ++u) {
      const int i = base + u * kColThreads;
      w[u] = i < quads ? reinterpret_cast<const uint4*>(s)[i] : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < kColUnroll; ++u) {
      const int i = base + u * kColThreads;
      if (i < quads) reinterpret_cast<uint4*>(d)[i] = w[u];
    }
  }
  for (int i = quads * kColVec + tid; i < rows; i += kColThreads) d[i] = s[i];
}

// CK_F32 / checked CK_COPY32 / CK_CHECK: Imputer fill + MinMaxValidator count, no tables
__device__ __noinline__ unsigned int item_plain(const ColOp& op, const uint32_t* __restrict__ s, uint32_t* __restrict__ d, int rows,
                                                int quads, int tid) {
  unsigned int bad = 0;
  auto one = [&](uint32_t bits) {
    double x;
    if (op.src_int) {
      x = (double)(int32_t)bits;
    } else {
      float f = __uint_as_float(bits);
      if (op.has_fill && f != f) f = op.fill;  // Imputer._impute (steps.py:397-406)
      bits = __float_as_uint(f);
      x = (double)f;
    }
    if (op.check) bad += col_check(op, x);
    return bits;
  };
  for (int base = tid; base < quads; base += kColThreads * kColUnroll) {
    uint4 w[kColUnroll];
#pragma unroll
    for (int u = 0; u < kColUnroll; ++u) {
      const int i = base + u * kColThreads;
      w[u] = i < quads ? reinterpret_cast<const uint4*>(s)[i] : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < kColUnroll; ++u) {
      const int i = base + u * kColThreads;
      if (i >= quads) continue;
      uint4 o;
      o.x = one(w[u].x);
      o.y = one(w[u].y);
      o.z = one(w[u].z);
      o.w = one(w[u].w);
      if (d) reinterpret_cast<uint4*>(d)[i] = o;
    }
  }
  for (int i = quads * kColVec + tid; i < rows; i += kColThreads) {
    const uint32_t o = one(s[i]);
    if (d) d[i] = o;
  }
  return bad;
}

// CK_RANGE / CK_VALUE / CK_ONEHOT: table ops (rare: kept compact, one element at a time inside a 16-byte access)
__device__ __noinline__ void item_table(const ColOp& op, const double* __restrict__ tab, const uint32_t* __restrict__ s, char* dst,
                                        int64_t out_stride, int64_t row0, int rows, int quads, int tid, unsigned int& bad,
                                        unsigned int& miss) {
  auto one = [&](uint32_t bits, int64_t row, uint32_t* oh /* n outputs for one-hot, else 1 */) {
    double x;
    bool hit;
    const uint32_t o = col_word(op, tab, bits, x, hit);
    miss += hit ? 0u : 1u;
    if (op.check) bad += col_check(op, x);
    (void)row;
    (void)oh;
    return o;
  };
  if (op.kind == CK_ONEHOT) {  // OneHotEncoder._encode (steps.py:453-470): unknown -> all zeros
    for (int i = tid; i < quads; i += kColThreads) {
      const uint4 w = reinterpret_cast<const uint4*>(s)[i];
      double x[4];
      bool hit;
      col_word(op, tab, w.x, x[0], hit);
      col_word(op, tab, w.y, x[1], hit);
      col_word(op, tab, w.z, x[2], hit);
      col_word(op, tab, w.w, x[3], hit);
      int any0 = 0, any1 = 0, any2 = 0, any3 = 0;
      for (int q = 0; q < op.n; ++q) {
        const double c = tab[q];
        int4 oh;
        oh.x = x[0] == c;
        oh.y = x[1] == c;
        oh.z = x[2] == c;
        oh.w = x[3] == c;
        any0 |= oh.x;
        any1 |= oh.y;
        any2 |= oh.z;
        any3 |= oh.w;
        reinterpret_cast<int4*>(reinterpret_cast<int32_t*>(dst + (int64_t)q * out_stride) + row0)[i] = oh;
      }
      miss += 4u - (unsigned)(any0 + any1 + any2 + any3);
    }
    for (int i = quads * kColVec + tid; i < rows; i += kColThreads) {
      double x;
      bool hit;
      col_word(op, tab, s[i], x, hit);
      bool any = false;
      for (int q = 0; q < op.n; ++q) {
        const bool is = x == tab[q];
        any |= is;
        reinterpret_cast<int32_t*>(dst + (int64_t)q * out_stride)[row0 + i] = is ? 1 : 0;
      }
      miss += any ? 0u : 1u;
    }
    return;
  }
  uint32_t* d = reinterpret_cast<uint32_t*>(dst) + row0;
  for (int i = tid; i < quads; i += kColThreads) {
    const uint4 w = reinterpret_cast<const uint4*>(s)[i];
    uint4 o;
    o.x = one(w.x, 0, nullptr);
    o.y = one(w.y, 0, nullptr);
    o.z = one(w.z, 0, nullptr);
    o.w = one(w.w, 0, nullptr);
    reinterpret_cast<uint4*>(d)[i] = o;
  }
  for (int i = quads * kColVec + tid; i < rows; i += kColThreads) d[i] = one(s[i], 0, nullptr);
}

// CK_COPY64 / CK_DATE: 8-byte sources, two rows per 16-byte load
__device__ __noinline__ unsigned int item_wide(const ColOp& op, const int64_t* __restrict__ s, char* dst, int64_t row0, int rows,
                                               bool vec_ok, int tid) {
  unsigned int miss = 0;
  const int pairs = vec_ok ? rows / 2 : 0;
  for (int i = tid; i < pairs; i += kColThreads) {
    const longlong2 v = reinterpret_cast<const longlong2*>(s)[i];
    if (op.kind == CK_COPY64) {
      reinterpret_cast<longlong2*>(reinterpret_cast<int64_t*>(dst) + row0)[i] = v;
    } else {
      const bool n0 = v.x == INT64_MIN, n1 = v.y == INT64_MIN;  // NaT
      miss += (n0 ? 1u : 0u) + (n1 ? 1u : 0u);
      int2 o;
      o.x = n0 ? -1 : date_part(v.x, op.part);
      o.y = n1 ? -1 : date_part(v.y, op.part);
      reinterpret_cast<int2*>(reinterpret_cast<int32_t*>(dst) + row0)[i] = o;
    }
  }
  for (int i = pairs * 2 + tid; i < rows; i += kColThreads) {  // tail / unaligned
    const int64_t v = s[i];
    if (op.kind == CK_COPY64) {
      reinterpret_cast<int64_t*>(dst)[row0 + i] = v;
    } else {
      const bool nat = v == INT64_MIN;
      miss += nat ? 1u : 0u;
      reinterpret_cast<int32_t*>(dst)[row0 + i] = nat ? -1 : date_part(v, op.part);
    }
  }
  return miss;
}

__global__ void __launch_bounds__(kColThreads) columns_kernel(const __grid_constant__ ColParams p) {
  __shared__ unsigned int s_cnt[2];
  const int tid = threadIdx.x;
  const int64_t n_chunks = (p.n_rows + kColChunk - 1) / kColChunk;
  const int64_t n_items = n_chunks * p.n_ops;
  // 16-byte accesses need 16-byte aligned slots (the strides the host path uses are multiples of 256)
  const bool vec_ok = ((p.in_stride | p.out_stride) & 15) == 0 && ((reinterpret_cast<uintptr_t>(p.in) | reinterpret_cast<uintptr_t>(p.out)) & 15) == 0;
  for (int64_t item = blockIdx.x; item < n_items; item += gridDim.x) {
#ifdef B2S_COL_CHUNK_MAJOR
    const int64_t chunk = item / p.n_ops;
    const ColOp op = p.ops[item - chunk * p.n_ops];
#else
    // column-major item order: neighbouring CTAs stream neighbouring chunks of the SAME column, so the GPU works on a
    // handful of long sequential streams at a time (DRAM row locality) instead of one short stream per CTA
    const int64_t opi = item / n_chunks;
    const int64_t chunk = item - opi * n_chunks;
    const ColOp op = p.ops[opi];
#endif
    const int64_t row0 = p.row_begin + chunk * kColChunk;
    const int64_t row_end = p.row_begin + p.n_rows;
    const int rows = (int)((row_end - row0 < kColChunk) ? (row_end - row0) : kColChunk);
    const char* src = p.in + (int64_t)op.src * p.in_stride;
    char* dst = op.dst >= 0 ? p.out + (int64_t)op.dst * p.out_stride : nullptr;
    unsigned int bad = 0, miss = 0;
    const bool counts = op.check || op.miss >= 0;
    if (counts) {
      if (tid < 2) s_cnt[tid] = 0;
      __syncthreads();
    }
    const int quads = vec_ok ? rows / kColVec : 0;
    const uint32_t* s32 = reinterpret_cast<const uint32_t*>(src) + row0;
    uint32_t* d32 = dst ? reinterpret_cast<uint32_t*>(dst) + row0 : nullptr;
    switch (op.kind) {
      case CK_COPY64:
      case CK_DATE:
        miss = item_wide(op, reinterpret_cast<const int64_t*>(src) + row0, dst, row0, rows, vec_ok, tid);
        break;
      case CK_RANGE:
      case CK_VALUE:
      case CK_ONEHOT:
        item_table(op, p.tab + op.tab, s32, dst, p.out_stride, row0, rows, quads, tid, bad, miss);
        break;
      case CK_COPY32:
        if (!op.check) {
          item_copy32(s32, d32, rows, quads, tid);
          break;
        }
        [[fallthrough]];
      default:  // CK_F32, checked CK_COPY32, CK_CHECK
        bad = item_plain(op, s32, d32, rows, quads, tid);
        break;
    }
    if (counts) {
      // one shared-memory atomic per warp, one global atomic per item
      for (int o = 16; o > 0; o >>= 1) {
        bad += __shfl_xor_sync(0xffffffffu, bad, o);
        miss += __shfl_xor_sync(0xffffffffu, miss, o);
      }
      if ((tid & 31) == 0) {
        if (bad) atomicAdd(&s_cnt[0], bad);
        if (miss) atomicAdd(&s_cnt[1], miss);
      }
      __syncthreads();
      if (tid == 0) {
        if (op.check && s_cnt[0]) atomicAdd(&p.counters[op.counter], (unsigned long long)s_cnt[0]);
        if (op.miss >= 0 && s_cnt[1]) atomicAdd(&p.counters[op.miss], (unsigned long long)s_cnt[1]);
      }
      __syncthreads();
    }
  }
}

}  // namespace b2s
