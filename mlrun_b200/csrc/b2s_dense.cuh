// b2s_dense.cuh -- dense linear head on the wgmma tensor cores (kernel in b2s_dense.cu): parameters and launcher.
#pragma once
#include <cuda.h>

#include "b2s_device.cuh"

namespace b2s {

constexpr int kDenseTileRows = 128;  // rows per tile == two warpgroups of wgmma M = 64
constexpr int kDenseMaxIn = 128;     // input columns (a multiple of 32: whole TMA boxes / swizzle atoms)

struct DenseParams {
  int64_t n_rows;
  const float* wh;     // [n_pad][n_in] W^T as three tf32 terms: the float64 coefficient w = wh + wm + wl to 33 bits
  const float* wm;     //   (each the leading 11 significant bits of what the previous ones left; rows past n_scores are zero)
  const float* wl;
  const float* fill;   // [n_in] Imputer values (NaN: not imputed)
  const double* bias;  // [n_scores] intercepts
  int32_t n_in, n_scores, n_pad, any_fill;
  int32_t exact;       // 1: inputs split into three tf32 terms (exact); 0: two terms, the second rounded to nearest (2^-23 |x|)
  // epilogue: the common shapes run in float32 registers (fp64 conversions and local-memory arrays are what the generic
  // epilogue spends its time on); everything else takes the generic link + vote functions
  int32_t epi;         // 0 generic | 1 every model one identity score, all emitted | 2 the same under a mean vote | 3 one argmax classifier
  float biasf[32];     // intercepts (float32)
  float votewf[32];    // epi 2: vote weights
  int32_t labels[32];  // epi 3: class labels
};

enum { DENSE_EPI_GENERIC = 0, DENSE_EPI_SCORES = 1, DENSE_EPI_MEAN = 2, DENSE_EPI_ARGMAX = 3 };

cudaError_t dense_launch(const DenseParams& p, const KParams& kp, const CUtensorMap& tmap, int grid, int smem, int smem_optin,
                         cudaStream_t st);
int dense_smem_bytes(int n_in, int n_pad);

}  // namespace b2s
