// b2s_internal.h -- what the translation units of libb200serve.so share (not part of the C-ABI).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#define B2S_HIDDEN __attribute__((visibility("hidden")))

B2S_HIDDEN int b2s_int_fail(int code, const char* fmt, ...);  // sets b2s_last_error(), returns code
B2S_HIDDEN bool b2s_int_inited();
B2S_HIDDEN int b2s_int_device();
B2S_HIDDEN int b2s_int_sm_count();
B2S_HIDDEN cudaStream_t b2s_int_stream();                      // the library stream
B2S_HIDDEN cudaStream_t b2s_int_copy_stream();                 // the library's copy stream (pipelined host runs)
B2S_HIDDEN void b2s_int_count_launches(int n);

// return B2S_ERR_CUDA (with the failed call, the CUDA error and the source line in b2s_last_error()) when expr fails
#define B2S_CUDA_TRY(expr)                                                                                             \
  do {                                                                                                                 \
    cudaError_t _e = (expr);                                                                                           \
    if (_e != cudaSuccess)                                                                                             \
      return b2s_int_fail(B2S_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

static inline bool misaligned(const void* ptr, uintptr_t bytes) { return ((uintptr_t)ptr & (bytes - 1)) != 0; }

// blocks of a grid-stride launch over n items: enough to fill the device (8 per SM), no more than the items need
static inline int grid_for(int64_t n, int threads) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)b2s_int_sm_count() * 8, (n + threads - 1) / threads));
}

struct b2s_plan_s;
B2S_HIDDEN int b2s_int_plan_shape(b2s_plan_s* plan, int* n_in, int* out_cols);  // B2S_ERR_STATE unless finalized
B2S_HIDDEN int b2s_int_plan_kernels(const b2s_plan_s* plan);  // launches of one batch of a finalized plan (trees3: 3)
// the plan's kernels store their votes to merge targets or an attached communicator, not into the caller's output
B2S_HIDDEN bool b2s_int_plan_merges(const b2s_plan_s* plan);

// the online table as the scoring kernel's gather loader sees it (b2s_table.cu fills it in)
struct B2SGather {
  const long long* d_keys;   // [n]
  const void* d_slots;       // b2s::TableSlot[mask + 1]
  unsigned long long mask;
  const float* d_values;     // [n_keys + 1][n_feat], last row NaN
  long long missing_row;     // n_keys
  const float* h_impute;     // [n_feat] host copy; NaN = keep the stored value
  int any_impute;
  int n_feat;
};
// keys -> (gather inside the scoring kernel) -> outputs + status (B2S_ROW_UNKNOWN_KEY included), one launch.
// B2S_ERR_UNSUPPORTED when this plan / table pair cannot be fused (the caller then gathers first).
B2S_HIDDEN int b2s_int_launch_gathered(b2s_plan_s* plan, const B2SGather& g, long long n, void* d_out, int* d_status, cudaStream_t st);
