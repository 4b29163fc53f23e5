// b2s_rowmma.cuh -- linear path, round 2: the dot products on the FP64 tensor-core instruction (DMMA m8n8k4).
//
// Why: `rowthread_kernel` can be issue bound on the metric workload: 8 DFMA + 7.6 LDCU warp-instructions per event for 64 columns x 4 scores, one
// constant-bank fetch per DFMA.  One `mma.sync.m8n8k4.f64` does 8 events x 4 columns x 8 scores (256 exact fp64 FMAs),
// with the weights resident in registers as B fragments: 2 warp-instructions per event instead of 15.6, same IEEE fp64
// arithmetic (every product and sum is a fused fp64 multiply-add; only the order of the additions differs).
//
//   * every WARP owns a private ring of S stages of 32-row tiles (TMA tensor-map boxes of 32 floats x 32 rows, 128-byte
//     swizzle) with its own mbarriers: no CTA-wide barrier anywhere; tiles are claimed from a per-CTA counter (the CTA's
//     tiles are blockIdx + i * grid), so the warps of an SM stay balanced to within one tile;
//   * phase A (lane = row): one-hot gathers + intercepts -> the row's initial accumulators (shared-memory scratch);
//   * phase B (lane = A/C fragment element): per 8-row group 4 x LDS.128, per value compare/select (Imputer) + F2F, 16 DMMAs
//     (NCH k-steps); two groups in flight for ILP; MMA row m reads tile row pi(m) = (m >> 1) | ((m & 1) << 2) so that the two
//     rows of a quarter-warp sit in different halves of the 128-byte swizzle atom (conflict-free LDS.128);
//     k index (lane & 3) of k-step (j, u) is column 16 j + 4 (lane & 3) + u: the 16-byte chunk a lane loads feeds 4 k-steps;
//   * phase C (lane = row): status, links / vote, coalesced stores -- the epilogues of rowthread_kernel.
// Per-lane operands (B fragments, Imputer fills and limits of the lane's 16 columns) live in registers for the whole kernel.
#pragma once
#include "b2s_rowthread.cuh"

namespace b2s {

constexpr int kRMMaxWarps = 16;
constexpr int kRMMaxStages = 4;

__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

template <int NCH, int NS>
__global__ void __launch_bounds__(kRMMaxWarps * 32, 1)
    rowmma_kernel(const __grid_constant__ RTParams<NCH, NS> p, const __grid_constant__ CUtensorMap tmap) {
  static_assert(NCH % 8 == 0 && NCH <= 16, "whole 32-float boxes; the per-lane operands must fit the register file");
  static_assert(NS <= 8, "one n = 8 fragment");
  constexpr int NSP = NS < 2 ? 2 : NS;      // scratch doubles per row (C fragments are pairs)
  constexpr int NJ = NCH / 4;               // 16-byte chunks per lane and row
  constexpr int TILE_BYTES = NCH * 512;     // 32 rows x NCH x 16 bytes
  extern __shared__ __align__(16) unsigned char smem[];
  const int W = (int)blockDim.x >> 5, S = p.stages;
  const int warp = (int)threadIdx.x >> 5, lane = (int)threadIdx.x & 31;
  // [W*S mbarriers | next-tile counter][W*S claimed tiles][one-hot weight rows][W x 32 x NSP scratch][tiles, 1024-aligned]
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(smem);
  int* s_next = reinterpret_cast<int*>(smem + kRMMaxWarps * kRMMaxStages * 8);
  long long* s_tileq = reinterpret_cast<long long*>(smem + kRMMaxWarps * kRMMaxStages * 8 + 16);
  double* s_wcat = reinterpret_cast<double*>(smem + kRMMaxWarps * kRMMaxStages * 16 + 16);
  const size_t wcat_bytes = (((size_t)(p.n_cat + 1) * NS * 8 + 15) / 16) * 16;
  double* s_scr = reinterpret_cast<double*>(reinterpret_cast<unsigned char*>(s_wcat) + wcat_bytes) + (size_t)warp * 32 * NSP;
  unsigned char* s_tiles = reinterpret_cast<unsigned char*>(s_wcat) + wcat_bytes + (size_t)W * 32 * NSP * 8;
  {
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(s_tiles);
    s_tiles += (1024u - (a & 1023u)) & 1023u;
  }
  s_tiles += (size_t)warp * S * TILE_BYTES;
  uint64_t* bar = s_bar + warp * kRMMaxStages;
  long long* tileq = s_tileq + warp * kRMMaxStages;

  const int64_t n_tiles = (p.n_rows + 31) >> 5;
  if (threadIdx.x == 0) *s_next = 0;
  if (lane == 0) {
    for (int s = 0; s < S; ++s) mbar_init(&bar[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < p.n_cat * NS; i += blockDim.x) s_wcat[i] = p.wcat[i];
  for (int i = threadIdx.x; i < NS; i += blockDim.x) s_wcat[p.n_cat * NS + i] = 0.0;
  __syncthreads();  // the only CTA-wide barrier: counter, weight rows

  auto claim_and_issue = [&](int st) {  // lane 0
    const int64_t t = (int64_t)blockIdx.x + (int64_t)atomicAdd(s_next, 1) * gridDim.x;
    tileq[st] = t;
    if (t < n_tiles) {
      mbar_expect_tx(&bar[st], (uint32_t)TILE_BYTES);
#pragma unroll
      for (int b = 0; b < NCH / 8; ++b) tensor_load_2d(s_tiles + st * TILE_BYTES + b * 4096, &tmap, b * 32, (int)(t << 5), &bar[st]);
    }
  };
  if (lane == 0)
    for (int s = 0; s < S; ++s) claim_and_issue(s);

  // ---- per-lane operands of phase B
  const int kq = lane & 3, nq = lane >> 2;
  const int pr = (nq >> 1) | ((nq & 1) << 2);  // tile row (mod 8) of this lane's MMA row
  double bw[NCH];                               // B fragments: w[column of (j, u, kq)][score nq]
  float fillr[NCH], limr[NCH];
#pragma unroll
  for (int j = 0; j < NJ; ++j)
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int c = 16 * j + 4 * kq + u;
      bw[j * 4 + u] = nq < NS ? p.w[c][nq < NS ? nq : 0] : 0.0;
      fillr[j * 4 + u] = p.fill[c];
      limr[j * 4 + u] = p.lim[c];
    }
  const uint32_t off_even = (uint32_t)pr * 128u + (uint32_t)((kq ^ pr) << 4);  // chunk 4j + kq of row pr, j even / odd
  const uint32_t off_odd = off_even ^ 64u;
  const bool c_lane = 2 * kq < NSP;  // this lane's C pair holds real scores
  __syncwarp();

  int stage = 0;
  uint32_t phase_bits = 0;
  for (;;) {
    const int64_t t = *reinterpret_cast<volatile long long*>(&tileq[stage]);
    if (t >= n_tiles) break;  // claims grow monotonically: every later claim of this warp is past the end as well
    mbar_wait(&bar[stage], (phase_bits >> stage) & 1u);
    phase_bits ^= 1u << stage;
    const unsigned char* tile = s_tiles + stage * TILE_BYTES;
    const int64_t row = (t << 5) + lane;

    {  // ---- phase A: lane = row
      RowSwizzled xr[1];
      xr[0].box0 = reinterpret_cast<const float*>(tile) + lane * 32;
      xr[0].box_words = 32 * 32;
      xr[0].r7s = (lane & 7) << 2;
      double acc[1][NS];
#pragma unroll
      for (int k = 0; k < NS; ++k) acc[0][k] = 0.0;
      rt_cats<NCH, NS, 0, 1>(p, xr, s_wcat, acc);
#pragma unroll
      for (int k = 0; k < NS; ++k) acc[0][k] += p.bias[k];
      double* mine = s_scr + lane * NSP;
      if constexpr (NS == 1) {
        *reinterpret_cast<double2*>(mine) = make_double2(acc[0][0], 0.0);
      } else {
#pragma unroll
        for (int k = 0; k < NS; k += 2) *reinterpret_cast<double2*>(mine + k) = make_double2(acc[0][k], acc[0][k + 1]);
      }
    }
    __syncwarp();

    // ---- phase B: two 8-row groups at a time
#pragma unroll 1
    for (int g = 0; g < 4; g += 2) {
      double c[2][2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        c[h][0] = 0.0;
        c[h][1] = 0.0;
        if (c_lane) {
          const double2 v = *reinterpret_cast<const double2*>(s_scr + ((g + h) * 8 + pr) * NSP + 2 * kq);
          c[h][0] = v.x;
          c[h][1] = v.y;
        }
      }
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        float4 v[2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
          v[h] = *reinterpret_cast<const float4*>(tile + (j >> 1) * 4096 + (g + h) * 1024 + ((j & 1) ? off_odd : off_even));
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float x = u == 0 ? v[h].x : (u == 1 ? v[h].y : (u == 2 ? v[h].z : v[h].w));
            x = !(fabsf(x) <= limr[j * 4 + u]) ? fillr[j * 4 + u] : x;  // Imputer / non-input -> +0 (see RTParams)
            dmma884(c[h][0], c[h][1], (double)x, bw[j * 4 + u]);
          }
      }
      if (c_lane) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
          *reinterpret_cast<double2*>(s_scr + ((g + h) * 8 + pr) * NSP + 2 * kq) = make_double2(c[h][0], c[h][1]);
      }
    }
    __syncwarp();

    // ---- phase C: lane = row (the epilogues of rowthread_kernel)
    if (row < p.n_rows) {
      double sc[NS];
      const double* mine = s_scr + lane * NSP;
      if constexpr (NS == 1) {
        sc[0] = mine[0];
      } else {
#pragma unroll
        for (int k = 0; k < NS; k += 2) {
          const double2 v = *reinterpret_cast<const double2*>(mine + k);
          sc[k] = v.x;
          sc[k + 1] = v.y;
        }
      }
      uint32_t st = 0;
#pragma unroll
      for (int k = 0; k < NS; ++k) st |= (fabs(sc[k]) <= 1.7976931348623157e308) ? 0u : 1u;
      if (p.fast_epilogue) {
        if (p.vote_kind == 1) {  // VotingEnsemble._mean_vote: sum_m w[m] * pred[m], model order
          double s = 0.0;
#pragma unroll
          for (int k = 0; k < NS; ++k) s = __dadd_rn(s, __dmul_rn(sc[k], p.vote_w[k]));
          store_word(p, row, 0, __float_as_uint((float)s));
        } else {
#pragma unroll
          for (int k = 0; k < NS; ++k)
            if (k < p.n_models) store_word(p, row, k, __float_as_uint((float)sc[k]));
        }
        if (p.status) p.status[row] = (int32_t)st;
      } else {
        rt_generic_epilogue(p, sc, row, st);
      }
    }
    __syncwarp();  // every lane is done with the tile and the scratch rows
    if (lane == 0) claim_and_issue(stage);
    __syncwarp();
    ++stage;
    if (stage == S) stage = 0;
  }
  merge_signal(p.sig);
}

// host side (b2s_rowmma.cu): shared memory the kernel needs for `warps` warps and `stages` stages
size_t rowmma_smem_bytes(int nch, int ns, int n_cat, int warps, int stages);
// launches the instantiation for (nch, ns); `params` is the RTParams<nch, ns> blob.  cudaErrorInvalidValue: no such variant
cudaError_t rowmma_launch(int nch, int ns, const void* params, const CUtensorMap* tmap, int grid, int warps, size_t smem, cudaStream_t st);
cudaError_t rowmma_prepare(int nch, int ns, int max_smem);  // opt-in shared-memory attribute

}  // namespace b2s
