// b2s_dense.cu -- dense linear head on the Hopper tensor cores (sm_90a: wgmma.mma_async kind tf32, TMA, mbarriers).
//
// north_star: "tensor cores only on the dense linear-predict path".  A linear / logistic scorer (or an ensemble of them)
// with many scores per event -- a 16-class LogisticRegression is scores = X (B x K) . W^T (K x 16) + b, then argmax
// (sklearn decision_function + predict behind PickleModelServer.predict, frameworks/_ml_common/pkl_model_server.py:52-60)
// -- is a GEMM with a skinny N.  The fp64 FMA path of the row kernels does K x N DFMAs per event; here the products run on
// the tensor cores.  One persistent CTA per SM, a producer warp and two math warpgroups connected by mbarriers:
//
//   producer   (1 thread)   TMA boxes (32 floats x 128 rows, 128-byte swizzle: already the wgmma K-major operand layout) into
//                           a ring of 3 raw stages
//   math       (2 warpgroups, rows 0-63 | 64-127 of every tile) per box:
//                           split -- every value x (after the Imputer) becomes xh + xm + xl, three tf32 numbers that add up
//                           to x EXACTLY (11 + 11 + 2 significant bits, by masking and exact subtraction), written to one of
//                           two operand stages of the warpgroup; non-finite values flag their row.  Warp w owns the 16-byte
//                           chunks w and w + 4 of every box row, lanes take consecutive rows: LDS.128 / STS.128 without bank
//                           conflicts.
//                           mma -- per k-step of 8 columns five or six wgmma.m64nNk8.f32.tf32 (N = 16 | 32):
//                             main [box]  += xh.wh                                  one accumulator per 32-column box
//                             small       += xh.wm + xm.wh + xm.wm + xh.wl + xl.wh   (two accumulators) per box group
//                           weights are split on the host into wh + wm + wl (33 bits of the float64 coefficient); the dropped
//                           products are < 2^-33 |x w|.  Every product is exact in fp32; what rounds is the accumulation
//                           (the tensor core truncates), so large terms get one accumulator per box and the small ones
//                           (2^-11 of the large) their own: the error is a few ulp of a 32-column partial sum, ~1e-6
//                           absolute for unit-scale data, where a single accumulator loses 1e-5.
//                           Every warp ends a box with wait_group 0: a warp's wait covers only its own part of a
//                           warpgroup MMA, while every warp rewrites all 64 rows of an operand stage, so stage b & 1 is
//                           free for box b + 2 only once every warp has passed the barrier of box b + 1.  The other
//                           warpgroup's split overlaps this one's MMAs.
//                           epilogue -- the accumulators (registers) are summed, staged through shared memory so that one
//                           thread owns one row, then the intercepts, the links and the VotingEnsemble reduce are applied and
//                           votes + status stored (to every merge target when sharded) -- float32 fast paths for the common
//                           shapes, the generic epilogue functions of the other kernels (fp64) for the rest.
// Evidence to look for: SASS HGMMA + UTMALDG.
#include <cuda.h>
#include <cuda_runtime.h>

#include <atomic>

#include "b2s_rowthread.cuh"  // mbarrier / TMA helpers, KParams, epilogue functions
#include "b2s_dense.cuh"

namespace b2s {

constexpr int kDM = kDenseTileRows;  // rows per tile: two warpgroups of wgmma M = 64
constexpr int kWgRows = 64;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// K-major, 128-byte swizzle shared-memory matrix descriptor (sm90 GMMA): start address >> 4 in bits [0,14), leading byte
// offset (unused: one swizzle atom along K) [16,30), stride byte offset = 8 rows x 128 B >> 4 in [32,46), layout type
// SWIZZLE_128B (1) in [62,64)
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3fffu) | (1ull << 16) | ((uint64_t)(1024u >> 4) << 32) | (1ull << 62);
}

// d (64 x N, fp32, registers of the warpgroup) += A (64 x 8 tf32, smem) . B (N x 8 tf32, smem)^T
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc);

template <>
__device__ __forceinline__ void wgmma_tf32<16>(float (&d)[8], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(1));
}

template <>
__device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(1));
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int K>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(K) : "memory"); }
// registers in flight in an asynchronous wgmma must not be moved by the compiler across the wait
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
  for (int k = 0; k < N; ++k) asm volatile("" : "+f"(d[k])::"memory");
}
__device__ __forceinline__ void wg_sync(int wg) {  // named barrier of one warpgroup (id 0 is __syncthreads)
  asm volatile("bar.sync %0, %1;" ::"r"(wg + 1), "r"(128) : "memory");
}
__device__ __forceinline__ uint32_t tf32_hi(float x) { return __float_as_uint(x) & 0xffffe000u; }

constexpr int kRawStages = 3;                  // TMA landing boxes of 16 KB
constexpr int kMathWGs = 2;
constexpr int kDenseThreads = (kMathWGs * 4 + 1) * 32;  // + producer warp
constexpr uint32_t kBoxBytes = kDM * 128u;     // one box: 128 rows x 32 floats
constexpr uint32_t kTermBytes = kWgRows * 128u;  // one tf32 term of a warpgroup's half box
constexpr uint32_t kOpStageBytes = 3u * kTermBytes;  // operand stage: xh | xm | xl
constexpr uint32_t kOffOut = kRawStages * kBoxBytes;
constexpr uint32_t kOffB = kOffOut + kMathWGs * 2u * kOpStageBytes;

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// NP: padded score count 16 | 32; BOXES: input columns / 32; FILL: an Imputer is folded in; XT: tf32 terms per input (3: exact,
// 2: xh + round-to-nearest residual, |error| <= 2^-23 |x|)
template <int NP, int BOXES, bool FILL, int XT>
__global__ void __launch_bounds__(kDenseThreads, 1) dense_head_kernel(const __grid_constant__ DenseParams p, const __grid_constant__ KParams kp,
                                                                      const __grid_constant__ CUtensorMap tmap) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  // 128-byte swizzled TMA destinations and wgmma operands need 1024-byte aligned addresses
  unsigned char* smem_dense = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int K = BOXES * 32;
  constexpr uint32_t kBBox = 3u * NP * 128u;  // the weights of one box: rows [wh (NP) | wm (NP) | wl (NP)] x 128 B
  constexpr uint32_t kOffMisc = kOffB + (uint32_t)BOXES * kBBox;
  // accumulator groups: one per box while the registers allow (G x 3 x NP / 2 floats per thread)
  constexpr int G = NP == 16 ? BOXES : (BOXES < 2 ? BOXES : 2);
  constexpr int BPG = (BOXES + G - 1) / G;  // boxes per group
  constexpr int NR = NP / 2;                // accumulator registers per thread of one 64 x NP fragment
  float* s_fill = reinterpret_cast<float*>(smem_dense + kOffMisc);                       // [K]
  int* s_bad = reinterpret_cast<int*>(smem_dense + kOffMisc + 512);                      // [2 warpgroups][2 tiles][64]
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(smem_dense + kOffMisc + 512 + kMathWGs * 2 * kWgRows * 4);
  uint64_t* raw_full = s_bar;                   // [3]  TMA transaction bytes
  uint64_t* raw_empty = s_bar + kRawStages;     // [3]  8 math warps
  float* s_sc = reinterpret_cast<float*>(s_bar + 2 * kRawStages);  // [2 warpgroups][64][NP + 1] final scores

  // ---- one-time setup: barriers, the weights in the wgmma layout (rows = scores, K-major, 128-byte swizzle)
  if (tid == 0) {
    for (int i = 0; i < kRawStages; ++i) {
      mbar_init(&raw_full[i], 1);
      mbar_init(&raw_empty[i], kMathWGs * 4);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = tid; i < NP * K; i += kDenseThreads) {
    const int n = i / K, k = i - n * K;
    const int b = k >> 5, c = (k & 31) >> 2, e = k & 3;
    const uint32_t off = kOffB + (uint32_t)b * kBBox + (uint32_t)n * 128u + (uint32_t)((c ^ (n & 7)) << 4) + (uint32_t)e * 4u;
    *reinterpret_cast<float*>(smem_dense + off) = p.wh[i];  // NP * 128 is a multiple of 1024: the swizzle phase of a row is n & 7 in every term
    *reinterpret_cast<float*>(smem_dense + off + NP * 128u) = p.wm[i];
    *reinterpret_cast<float*>(smem_dense + off + 2u * NP * 128u) = p.wl[i];
  }
  for (int i = tid; i < K; i += kDenseThreads) s_fill[i] = p.fill[i];
  for (int i = tid; i < kMathWGs * 2 * kWgRows; i += kDenseThreads) s_bad[i] = 0;
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores above -> visible to the tensor core
  __syncthreads();
  const int64_t n_tiles = (p.n_rows + kDM - 1) / kDM;
  const uint32_t sbase = smem_u32(smem_dense);

  if (warp == kMathWGs * 4) {
    // =============================================================================================== producer
    if (lane == 0) {
      int q = 0;
      for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x)
        for (int b = 0; b < BOXES; ++b, ++q) {
          const int rs = q % kRawStages, use = q / kRawStages;
          if (use > 0) mbar_wait(&raw_empty[rs], (uint32_t)(use - 1) & 1u);
          mbar_expect_tx(&raw_full[rs], kBoxBytes);
          tensor_load_2d(smem_dense + (size_t)rs * kBoxBytes, &tmap, b * 32, (int)(t * kDM), &raw_full[rs]);  // rows past the end: zeros
        }
    }
  } else {
    // =============================================================================================== math warpgroups
    const int wg = warp >> 2, w = warp & 3;
    const int wtid = tid & 127;
    const uint32_t toff = (uint32_t)lane * 128u;  // row lane (+ 32 j) of the half box; chunk c sits at (c ^ (lane & 7)) << 4
    const uint32_t op_base = kOffOut + (uint32_t)wg * 2u * kOpStageBytes;
    float* sc_stage = s_sc + wg * kWgRows * (NP + 1);
    int q = 0, i = 0;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x, ++i) {
      int* bad = s_bad + (wg * 2 + (i & 1)) * kWgRows;  // two tiles of flags: the next tile's split may run ahead of a reset
      float acc_main[G][NR], acc_s1[G][NR], acc_s2[G][NR];
#pragma unroll
      for (int g = 0; g < G; ++g)
#pragma unroll
        for (int k = 0; k < NR; ++k) acc_main[g][k] = acc_s1[g][k] = acc_s2[g][k] = 0.f;
#pragma unroll
      for (int b = 0; b < BOXES; ++b, ++q) {
        const int rs = q % kRawStages, os = q & 1;
        mbar_wait(&raw_full[rs], (uint32_t)(q / kRawStages) & 1u);
        const unsigned char* src = smem_dense + (size_t)rs * kBoxBytes + (size_t)wg * kTermBytes + toff;
        float4 v[2][2];  // [chunk w | w + 4][row lane | lane + 32]
#pragma unroll
        for (int cc = 0; cc < 2; ++cc)
#pragma unroll
          for (int j = 0; j < 2; ++j)
            v[cc][j] = *reinterpret_cast<const float4*>(src + j * 4096 + (((w + 4 * cc) ^ (lane & 7)) << 4));
        // every warp finished its part of box q - 2, which read this operand stage, before the barrier of box q - 1
        unsigned char* dst = smem_dense + op_base + (size_t)os * kOpStageBytes + toff;
#pragma unroll
        for (int cc = 0; cc < 2; ++cc) {
          const int c = w + 4 * cc;
          float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
          if (FILL) f = *reinterpret_cast<const float4*>(s_fill + (b * 8 + c) * 4);
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const float xs[4] = {v[cc][j].x, v[cc][j].y, v[cc][j].z, v[cc][j].w};
            const float fs[4] = {f.x, f.y, f.z, f.w};
            uint32_t h[4], m[4], l[4];
            float probe = 0.f;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              float x = xs[e];
              if (FILL) x = (x != x) ? fs[e] : x;  // Imputer._impute (feature_store/steps.py:397-406); NaN where nothing is imputed
              probe = fmaf(x, 0.f, probe);              // NaN as soon as one value is NaN or +-Inf
              h[e] = tf32_hi(x);
              const float r1 = x - __uint_as_float(h[e]);  // exact: the low 13 bits of x
              if (XT == 3) {
                m[e] = tf32_hi(r1);
                l[e] = __float_as_uint(r1 - __uint_as_float(m[e]));  // exact: at most 2 significant bits are left
              } else {
                asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(m[e]) : "f"(r1));  // nearest tf32: x = xh + xm up to 2^-23 |x|
                l[e] = 0u;
              }
            }
            unsigned char* d = dst + j * 4096 + ((c ^ (lane & 7)) << 4);
            *reinterpret_cast<uint4*>(d) = make_uint4(h[0], h[1], h[2], h[3]);
            *reinterpret_cast<uint4*>(d + kTermBytes) = make_uint4(m[0], m[1], m[2], m[3]);
            if (XT == 3) *reinterpret_cast<uint4*>(d + 2 * kTermBytes) = make_uint4(l[0], l[1], l[2], l[3]);
            // a non-finite value makes its own row's scores NaN (rows are independent in the product) and flags the row
            if (probe != probe) atomicOr(bad + lane + 32 * j, 1);
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the stores above -> visible to the tensor core
        // the raw stage goes back to the producer only once every lane's loads have been consumed by its stores above: an
        // arrive right after issuing the loads lets the next TMA overwrite rows whose loads are still in flight
        __syncwarp();
        if (lane == 0) mbar_arrive(&raw_empty[rs]);
        wg_sync(wg);
        const uint32_t xh = sbase + op_base + (uint32_t)os * kOpStageBytes, xm = xh + kTermBytes, xl = xm + kTermBytes;
        const uint32_t wb = sbase + kOffB + (uint32_t)b * kBBox;  // rows [wh | wm | wl]
        const int g = b / BPG;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {  // 8 tf32 = 32 bytes per instruction inside the 128-byte swizzle atom
          const uint32_t ko = (uint32_t)kk * 32u;
          const uint32_t wh = wb + ko, wm = wh + NP * 128u, wl = wm + NP * 128u;
          wgmma_tf32<NP>(acc_main[g], gmma_desc(xh + ko), gmma_desc(wh));
          wgmma_tf32<NP>(acc_s1[g], gmma_desc(xh + ko), gmma_desc(wm));
          wgmma_tf32<NP>(acc_s2[g], gmma_desc(xh + ko), gmma_desc(wl));
          wgmma_tf32<NP>(acc_s1[g], gmma_desc(xm + ko), gmma_desc(wh));
          wgmma_tf32<NP>(acc_s2[g], gmma_desc(xm + ko), gmma_desc(wm));
          if (XT == 3) wgmma_tf32<NP>(acc_s1[g], gmma_desc(xl + ko), gmma_desc(wh));
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int gg = 0; gg < G; ++gg) {
          fence_regs(acc_main[gg]);
          fence_regs(acc_s1[gg]);
          fence_regs(acc_s2[gg]);
        }
      }
      // fragment element k of warp w, lane l: row 16 w + l / 4 + 8 ((k >> 1) & 1), column 8 (k >> 2) + 2 (l & 3) + (k & 1)
#pragma unroll
      for (int k = 0; k < NR; ++k) {
        float mainv = 0.f, smallv = 0.f;
#pragma unroll
        for (int gg = 0; gg < G; ++gg) {  // groups in column order; the small terms (2^-11 of the large) on their own
          const float sm = acc_s1[gg][k] + acc_s2[gg][k];
          mainv = gg == 0 ? acc_main[gg][k] : mainv + acc_main[gg][k];
          smallv = gg == 0 ? sm : smallv + sm;
        }
        const int r = 16 * w + (lane >> 2) + 8 * ((k >> 1) & 1), col = 8 * (k >> 2) + 2 * (lane & 3) + (k & 1);
        sc_stage[r * (NP + 1) + col] = mainv + smallv;
      }
      wg_sync(wg);
      if (wtid < kWgRows) {
        const int rr = wtid;
        const uint32_t st = bad[rr] ? 1u : 0u;
        bad[rr] = 0;
        float sc[NP];
#pragma unroll
        for (int k = 0; k < NP; ++k) sc[k] = sc_stage[rr * (NP + 1) + k];
        const int64_t row = t * kDM + wg * kWgRows + rr;
        if (row < p.n_rows) {
          if (p.epi != DENSE_EPI_GENERIC) {
            // ---- fast epilogues: float32 registers only (compile-time indices; the intercepts are constant-bank operands).
            // Merged rows take the same arithmetic as local ones: only the store differs (store_word, one word per target)
#pragma unroll
            for (int k = 0; k < NP; ++k) sc[k] += p.biasf[k];
            if (p.epi == DENSE_EPI_SCORES) {  // out_cols == n_scores consecutive floats per row
              if (kp.n_peers == 0 && (kp.out_cols & 3) == 0) {
                float* o = kp.out + row * kp.out_cols;
#pragma unroll
                for (int k = 0; k < NP; k += 4)
                  if (k < p.n_scores) *reinterpret_cast<float4*>(o + k) = make_float4(sc[k], sc[k + 1], sc[k + 2], sc[k + 3]);
              } else {
#pragma unroll
                for (int k = 0; k < NP; ++k)
                  if (k < p.n_scores) store_word(kp, row, k, __float_as_uint(sc[k]));
              }
            } else if (p.epi == DENSE_EPI_MEAN) {  // VotingEnsemble._mean_vote: sum_m w[m] * pred[m], model order
              float v = 0.f;
#pragma unroll
              for (int k = 0; k < NP; ++k) v = fmaf(p.votewf[k], sc[k], v);  // the padding has zero weight
              store_word(kp, row, 0, __float_as_uint(v));
            } else {  // one multi-class linear classifier: np.argmax (first maximum), then classes_[index]
              int best = 0;
              float bv = sc[0];
#pragma unroll
              for (int k = 1; k < NP; ++k)
                if (k < p.n_scores && sc[k] > bv) {
                  bv = sc[k];
                  best = k;
                }
              int lab = p.labels[0];
#pragma unroll
              for (int k = 1; k < NP; ++k) lab = best == k ? p.labels[k] : lab;
              store_word(kp, row, 0, (uint32_t)lab);
            }
            if (kp.status) kp.status[row] = (int32_t)st;
          } else {
            double scd[NP];
#pragma unroll
            for (int k = 0; k < NP; ++k) scd[k] = k < p.n_scores ? (double)sc[k] + p.bias[k] : 0.0;
            double pred[kMaxModels];
            for (int m = 0; m < kp.n_models; ++m) {
              const ModelDesc md = kp.models[m];
              pred[m] = apply_link(md, scd + md.score_off, kp.classes);
            }
            vote_and_store(kp, pred, row, st);
          }
        }
      }
    }
  }
  __syncthreads();
  merge_signal(kp.sig);
}

template <int NP, int BOXES, bool FILL, int XT>
static cudaError_t dense_go(const DenseParams& p, const KParams& kp, const CUtensorMap& tmap, int grid, int smem, int smem_optin,
                            cudaStream_t st) {
  static std::atomic<bool> attr{false};
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(dense_head_kernel<NP, BOXES, FILL, XT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin);
    if (e != cudaSuccess) return e;
    attr = true;
  }
  dense_head_kernel<NP, BOXES, FILL, XT><<<grid, kDenseThreads, smem, st>>>(p, kp, tmap);
  return cudaGetLastError();
}

cudaError_t dense_launch(const DenseParams& p, const KParams& kp, const CUtensorMap& tmap, int grid, int smem, int smem_optin,
                         cudaStream_t st) {
  const int boxes = p.n_in / 32;
#define B2S_DENSE_CASE(NPV, BX)                                                                          \
  if (p.n_pad == NPV && boxes == BX)                                                                   \
    return p.exact ? (p.any_fill ? dense_go<NPV, BX, true, 3>(p, kp, tmap, grid, smem, smem_optin, st)   \
                                 : dense_go<NPV, BX, false, 3>(p, kp, tmap, grid, smem, smem_optin, st)) \
                   : (p.any_fill ? dense_go<NPV, BX, true, 2>(p, kp, tmap, grid, smem, smem_optin, st)   \
                                 : dense_go<NPV, BX, false, 2>(p, kp, tmap, grid, smem, smem_optin, st));
  B2S_DENSE_CASE(16, 1) B2S_DENSE_CASE(16, 2) B2S_DENSE_CASE(16, 3) B2S_DENSE_CASE(16, 4)
  B2S_DENSE_CASE(32, 1) B2S_DENSE_CASE(32, 2) B2S_DENSE_CASE(32, 3) B2S_DENSE_CASE(32, 4)
#undef B2S_DENSE_CASE
  return cudaErrorInvalidValue;
}

int dense_smem_bytes(int n_in, int n_pad) {  // + 1024: the kernel aligns its base to 1024 bytes
  const int boxes = n_in / 32;
  return (int)(kOffB + 3u * (uint32_t)boxes * (uint32_t)n_pad * 128u) + 512 + kMathWGs * 2 * kWgRows * 4 + 2 * kRawStages * 8 +
         kMathWGs * kWgRows * (n_pad + 1) * 4 + 1024;
}

}  // namespace b2s
