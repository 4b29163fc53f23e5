// b2s_devcols.cu -- device-resident feature-set ingest: what the host path does around the columns and aggregation kernels,
// done on the device for columns that already live in HBM.  convert_kernel stages the caller's columns into the slot block
// b2s_cols_run_device reads (copies, and widening of 1- and 2-byte ints), counts int32 values a float32 map output would
// round, and gives result columns the dtypes the host path gives them; keys_kernel encodes entity keys as keys.py does;
// ts_profile_kernel counts what registration and the as-of join ask of a timestamp column (NaT, and its coarsest unit).
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <vector>

#include "../../include/b200serve.h"
#include "b2s_internal.h"
#include "b2s_stage.h"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxOps = 65535;  // gridDim.y

struct ConvOp {
  const void* src;
  void* dst;
  int kind;
  int counter;
};

__global__ void __launch_bounds__(kThreads) convert_kernel(const ConvOp* __restrict__ ops, int64_t n, unsigned long long* counters) {
  const ConvOp op = ops[blockIdx.y];
  unsigned long long hits = 0;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    switch (op.kind) {
      case B2S_CONV_COPY4: static_cast<uint32_t*>(op.dst)[i] = static_cast<const uint32_t*>(op.src)[i]; break;
      case B2S_CONV_COPY8: static_cast<uint64_t*>(op.dst)[i] = static_cast<const uint64_t*>(op.src)[i]; break;
      case B2S_CONV_I8_I32: static_cast<int32_t*>(op.dst)[i] = static_cast<const int8_t*>(op.src)[i]; break;
      case B2S_CONV_U8_I32: static_cast<int32_t*>(op.dst)[i] = static_cast<const uint8_t*>(op.src)[i]; break;
      case B2S_CONV_I16_I32: static_cast<int32_t*>(op.dst)[i] = static_cast<const int16_t*>(op.src)[i]; break;
      case B2S_CONV_U16_I32: static_cast<int32_t*>(op.dst)[i] = static_cast<const uint16_t*>(op.src)[i]; break;
      case B2S_CONV_I32_F64: static_cast<double*>(op.dst)[i] = static_cast<const int32_t*>(op.src)[i]; break;
      case B2S_CONV_F32_I32: {  // numpy's astype on x86: out of range and NaN give INT32_MIN
        const float v = static_cast<const float*>(op.src)[i];
        static_cast<int32_t*>(op.dst)[i] = (v >= -2147483648.0f && v < 2147483648.0f) ? (int32_t)v : INT32_MIN;
        break;
      }
      case B2S_CONV_DATE_F64: {
        const int32_t v = static_cast<const int32_t*>(op.src)[i];
        static_cast<double*>(op.dst)[i] = v < 0 ? (double)NAN : (double)v;
        break;
      }
      case B2S_CONV_I32_BOOL: static_cast<uint8_t*>(op.dst)[i] = static_cast<const int32_t*>(op.src)[i] != 0; break;
      case B2S_CONV_CHECK_F32: {
        const int32_t v = static_cast<const int32_t*>(op.src)[i];
        hits += (int64_t)__int2float_rn(v) != (int64_t)v;
        break;
      }
    }
  }
  if (op.kind == B2S_CONV_CHECK_F32) {
    for (int o = 16; o; o >>= 1) hits += __shfl_xor_sync(0xffffffffu, hits, o);
    if ((threadIdx.x & 31) == 0 && hits) atomicAdd(counters + op.counter, hits);
  }
}

struct KeyCol {
  const void* src;
  int bytes;
  int is_signed;
};

__device__ __forceinline__ int64_t key_word(const KeyCol& c, int64_t i) {
  switch (c.bytes) {
    case 1: return c.is_signed ? (int64_t) static_cast<const int8_t*>(c.src)[i] : (int64_t) static_cast<const uint8_t*>(c.src)[i];
    case 2: return c.is_signed ? (int64_t) static_cast<const int16_t*>(c.src)[i] : (int64_t) static_cast<const uint16_t*>(c.src)[i];
    case 4: return c.is_signed ? (int64_t) static_cast<const int32_t*>(c.src)[i] : (int64_t) static_cast<const uint32_t*>(c.src)[i];
    default: return static_cast<const int64_t*>(c.src)[i];
  }
}

// keys.py _encode_keys: one int column widened to int64; two int32 columns as hi << 32 | (lo & 0xFFFFFFFF)
__global__ void __launch_bounds__(kThreads) keys_kernel(KeyCol hi, KeyCol lo, int pair, int64_t n, int64_t* __restrict__ keys) {
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    const int64_t h = key_word(hi, i);
    keys[i] = pair ? (int64_t)(((uint64_t)h << 32) | ((uint64_t)key_word(lo, i) & 0xFFFFFFFFull)) : h;
  }
}

constexpr int kMaxDecimalCols = 16;

struct DecimalCols {
  KeyCol c[kMaxDecimalCols];
  int n;
};

__device__ __forceinline__ uint64_t fnv_byte(uint64_t h, unsigned b) { return (h ^ b) * 1099511628211ULL; }

// FNV-1a folded over the decimal text of v, most significant digit first.  The magnitude is taken in uint64 (2^63 for
// INT64_MIN, which has no int64 negation); it has at most 19 digits, so p never passes 10^18.
__device__ __forceinline__ uint64_t fnv_decimal(uint64_t h, int64_t v) {
  uint64_t u = (uint64_t)v;
  if (v < 0) {
    h = fnv_byte(h, '-');
    u = 0ull - u;
  }
  uint64_t p = 1;
  while (u / p >= 10) p *= 10;
  for (;;) {
    const uint64_t d = u / p;
    h = fnv_byte(h, (unsigned)('0' + d));
    u -= d * p;
    if (p == 1) return h;
    p /= 10;
  }
}

// online.py _encode_keys of a composite key: FNV-1a of ".".join(str(v) for v in row)
__global__ void __launch_bounds__(kThreads) keys_decimal_kernel(const __grid_constant__ DecimalCols cols, int64_t n, int64_t* __restrict__ keys) {
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    uint64_t h = 1469598103934665603ULL;
    for (int c = 0; c < cols.n; ++c) {
      if (c) h = fnv_byte(h, '.');
      h = fnv_decimal(h, key_word(cols.c[c], i));
    }
    keys[i] = (int64_t)h;
  }
}

// counts[0]: NaT (INT64_MIN) values; counts[1..3]: the other values that are not whole multiples of 10^3, 10^6, 10^9 ns.
// A zero remainder means the same in C (truncated) and numpy (floored) division, so negative timestamps count alike.
__global__ void __launch_bounds__(kThreads) ts_profile_kernel(const int64_t* __restrict__ ts, int64_t n, unsigned long long* __restrict__ counts) {
  unsigned long long c[4] = {0, 0, 0, 0};
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    const int64_t t = ts[i];
    if (t == INT64_MIN) {
      ++c[0];
    } else {
      c[1] += t % 1000ll != 0;
      c[2] += t % 1000000ll != 0;
      c[3] += t % 1000000000ll != 0;
    }
  }
  for (int k = 0; k < 4; ++k) {
    unsigned long long v = c[k];
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(counts + k, v);
  }
}

int src_bytes(int kind) {
  switch (kind) {
    case B2S_CONV_COPY8: return 8;
    case B2S_CONV_I8_I32: case B2S_CONV_U8_I32: return 1;
    case B2S_CONV_I16_I32: case B2S_CONV_U16_I32: return 2;
    default: return 4;
  }
}

int dst_bytes(int kind) {
  switch (kind) {
    case B2S_CONV_COPY8: case B2S_CONV_I32_F64: case B2S_CONV_DATE_F64: return 8;
    case B2S_CONV_I32_BOOL: return 1;
    case B2S_CONV_CHECK_F32: return 0;
    default: return 4;
  }
}

int device_ready() {
  if (!b2s_int_inited()) return b2s_int_fail(B2S_ERR_STATE, "b2s_init was not called (no CUDA device: there is no CPU fallback)");
  B2S_CUDA_TRY(cudaSetDevice(b2s_int_device()));
  return B2S_OK;
}

}  // namespace

extern "C" void* b2s_stream(void) { return b2s_int_inited() ? (void*)b2s_int_stream() : nullptr; }

extern "C" int b2s_stream_wait(void* producer) {
  try {  // no C++ exception crosses the C boundary
    if (int rc = device_ready()) return rc;
    cudaEvent_t ev = nullptr;
    B2S_CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    cudaError_t e = cudaEventRecord(ev, (cudaStream_t)producer);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(b2s_int_stream(), ev, 0);
    cudaEventDestroy(ev);  // released once the wait is satisfied
    B2S_CUDA_TRY(e);
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_pointer_device(const void* p, int32_t* device) {
  try {  // no C++ exception crosses the C boundary
    if (!p || !device) return b2s_int_fail(B2S_ERR_INVALID, "null pointer");
    cudaPointerAttributes a{};
    const cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) {
      cudaGetLastError();
      *device = -1;
      return B2S_OK;
    }
    *device = (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) ? a.device : -1;
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_cols_convert_device(const b2s_convert* ops, int32_t n_ops, int64_t n, uint64_t* d_counters, int32_t n_counters,
                                       void* stream) {
  try {  // no C++ exception crosses the C boundary
    if (n < 0 || n_ops < 1 || n_ops > kMaxOps || !ops || n_counters < 0)
      return b2s_int_fail(B2S_ERR_INVALID, "n >= 0, 1 .. %d operations and n_counters >= 0", kMaxOps);
    if (misaligned(d_counters, 8)) return b2s_int_fail(B2S_ERR_INVALID, "d_counters must be 8-byte aligned");
    std::vector<ConvOp> dev(n_ops);
    for (int i = 0; i < n_ops; ++i) {
      const b2s_convert& o = ops[i];
      if (o.kind < B2S_CONV_COPY4 || o.kind > B2S_CONV_CHECK_F32) return b2s_int_fail(B2S_ERR_INVALID, "operation %d: unknown kind %d", i, o.kind);
      const int sb = src_bytes(o.kind), db = dst_bytes(o.kind);
      if ((n && !o.src) || misaligned(o.src, sb)) return b2s_int_fail(B2S_ERR_INVALID, "operation %d: source null or not %d-byte aligned", i, sb);
      if (db && ((n && !o.dst) || misaligned(o.dst, db)))
        return b2s_int_fail(B2S_ERR_INVALID, "operation %d: destination null or not %d-byte aligned", i, db);
      if (o.kind == B2S_CONV_CHECK_F32 && (!d_counters || o.counter < 0 || o.counter >= n_counters))
        return b2s_int_fail(B2S_ERR_INVALID, "operation %d: counter %d outside the %d counters", i, o.counter, n_counters);
      dev[i] = ConvOp{o.src, o.dst, o.kind, o.counter};
    }
    if (n == 0) return B2S_OK;
    if (int rc = device_ready()) return rc;
    cudaStream_t st = stream ? (cudaStream_t)stream : b2s_int_stream();
    Launches launches;
    DeviceBlock blk(st);
    const ConvOp* d_ops = nullptr;
    blk.input(d_ops, dev.data(), sizeof(ConvOp) * dev.size());
    if (int rc = blk.alloc()) return rc;
    if (int rc = blk.upload()) return rc;
    const int gx = (int)std::max<int64_t>(1, std::min<int64_t>((n + kThreads - 1) / kThreads, ((int64_t)b2s_int_sm_count() * 8 + n_ops - 1) / n_ops));
    convert_kernel<<<dim3(gx, n_ops), kThreads, 0, st>>>(d_ops, n, reinterpret_cast<unsigned long long*>(d_counters));
    launches.add(1);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return b2s_int_fail(B2S_ERR_CUDA, "convert launch failed: %s", cudaGetErrorString(e));
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_keys_encode_device(const b2s_key_col* cols, int32_t n_cols, int64_t n, int64_t* d_keys, void* stream) {
  try {  // no C++ exception crosses the C boundary
    if (n < 0 || !cols || (n_cols != 1 && n_cols != 2)) return b2s_int_fail(B2S_ERR_INVALID, "n >= 0 and one or two key columns");
    for (int c = 0; c < n_cols; ++c) {
      const b2s_key_col& k = cols[c];
      const bool width = n_cols == 2 ? (k.bytes == 4 && k.is_signed) : (k.bytes == 1 || k.bytes == 2 || k.bytes == 4 || (k.bytes == 8 && k.is_signed));
      if (!width) return b2s_int_fail(B2S_ERR_INVALID, "key column %d: %d bytes %s is not a key (one int column, or two int32)", c, k.bytes,
                                      k.is_signed ? "signed" : "unsigned");
      if ((n && !k.src) || misaligned(k.src, k.bytes)) return b2s_int_fail(B2S_ERR_INVALID, "key column %d: null or misaligned", c);
    }
    if ((n && !d_keys) || misaligned(d_keys, 8)) return b2s_int_fail(B2S_ERR_INVALID, "d_keys: null or not 8-byte aligned");
    if (n == 0) return B2S_OK;
    if (int rc = device_ready()) return rc;
    cudaStream_t st = stream ? (cudaStream_t)stream : b2s_int_stream();
    Launches launches;
    const KeyCol hi{cols[0].src, cols[0].bytes, cols[0].is_signed};
    const KeyCol lo = n_cols == 2 ? KeyCol{cols[1].src, cols[1].bytes, cols[1].is_signed} : hi;
    keys_kernel<<<grid_for(n, kThreads), kThreads, 0, st>>>(hi, lo, n_cols == 2, n, d_keys);
    launches.add(1);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return b2s_int_fail(B2S_ERR_CUDA, "keys launch failed: %s", cudaGetErrorString(e));
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_keys_hash_decimal_device(const b2s_key_col* cols, int32_t n_cols, int64_t n, int64_t* d_keys, void* stream) {
  try {  // no C++ exception crosses the C boundary
    if (n < 0 || !cols || n_cols < 1 || n_cols > kMaxDecimalCols)
      return b2s_int_fail(B2S_ERR_INVALID, "n >= 0 and 1 .. %d key columns", kMaxDecimalCols);
    DecimalCols dc{};
    dc.n = n_cols;
    for (int c = 0; c < n_cols; ++c) {
      const b2s_key_col& k = cols[c];
      if (!k.is_signed || (k.bytes != 1 && k.bytes != 2 && k.bytes != 4 && k.bytes != 8))
        return b2s_int_fail(B2S_ERR_INVALID, "key column %d: %d bytes %s is not a signed int column", c, k.bytes, k.is_signed ? "signed" : "unsigned");
      if (n && !k.src) return b2s_int_fail(B2S_ERR_INVALID, "key column %d: null", c);
      dc.c[c] = KeyCol{k.src, k.bytes, 1};
    }
    if (n && !d_keys) return b2s_int_fail(B2S_ERR_INVALID, "d_keys: null");
    if (n == 0) return B2S_OK;
    if (int rc = device_ready()) return rc;
    for (int c = 0; c < n_cols; ++c)
      if (int rc = check_on_device(cols[c].src, cols[c].bytes, "key column", c)) return rc;
    if (int rc = check_on_device(d_keys, 8, "d_keys", 0)) return rc;
    cudaStream_t st = stream ? (cudaStream_t)stream : b2s_int_stream();
    Launches launches;
    keys_decimal_kernel<<<grid_for(n, kThreads), kThreads, 0, st>>>(dc, n, d_keys);
    launches.add(1);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return b2s_int_fail(B2S_ERR_CUDA, "decimal keys launch failed: %s", cudaGetErrorString(e));
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}

extern "C" int b2s_ts_profile_device(const int64_t* d_ts, int64_t n, int64_t* counts, void* stream) {
  try {  // no C++ exception crosses the C boundary
    if (n < 0 || !counts || (n && !d_ts)) return b2s_int_fail(B2S_ERR_INVALID, "n >= 0, non-null counts and (n > 0) timestamps");
    if (misaligned(d_ts, 8)) return b2s_int_fail(B2S_ERR_INVALID, "d_ts must be 8-byte aligned");
    for (int k = 0; k < 4; ++k) counts[k] = 0;
    if (n == 0) return B2S_OK;
    if (int rc = device_ready()) return rc;
    int32_t dev = -1;
    if (int rc = b2s_pointer_device(d_ts, &dev)) return rc;
    if (dev != b2s_int_device()) return b2s_int_fail(B2S_ERR_INVALID, "d_ts is not memory of the library's device %d", b2s_int_device());
    cudaStream_t st = stream ? (cudaStream_t)stream : b2s_int_stream();
    Launches launches;
    SyncOnExit done{st};
    DeviceBlock blk(st);
    unsigned long long* d_counts = nullptr;
    blk.scratch(d_counts, 32);
    if (int rc = blk.alloc()) return rc;
    B2S_CUDA_TRY(cudaMemsetAsync(d_counts, 0, 32, st));
    const int gx = (int)std::max<int64_t>(1, std::min<int64_t>((n + kThreads - 1) / kThreads, (int64_t)b2s_int_sm_count() * 8));
    ts_profile_kernel<<<gx, kThreads, 0, st>>>(d_ts, n, d_counts);
    launches.add(1);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return b2s_int_fail(B2S_ERR_CUDA, "ts profile launch failed: %s", cudaGetErrorString(e));
    B2S_CUDA_TRY(cudaMemcpyAsync(counts, d_counts, 32, cudaMemcpyDeviceToHost, st));
    B2S_CUDA_TRY(cudaStreamSynchronize(st));
    return B2S_OK;
  } catch (const std::exception& e) {
    return b2s_int_fail(B2S_ERR_INVALID, "%s: %s", __func__, e.what());
  }
}
