// b2s_trees2.cuh -- tree-ensemble scorer with the model resident in shared memory (sm_90a).
//
// A root->leaf walk is a chain of dependent gathers; from L2 (the generic kernel, tables ~1 MB for
// 4 x 100 depth-6 trees) every level costs ~250 cycles.  Here each persistent CTA owns ONE model of the
// router: its trees are re-packed on the host into complete (heap-ordered) depth-D trees, ~1 KB per
// depth-6 tree, ~100 KB per 100-tree model, copied to shared memory once per kernel (layout below).
// Rows land row-major through cp.async and are transposed in shared memory; thread (g, r) walks the trees
// t = g, g+G, ... of row r, four walks in flight, so one level is three conflict-free LDS (feature offset,
// threshold, feature value) + compare + index update.  The G partial sums of a row are combined in shared
// memory in a fixed order; the link function (identity / >0 / >=0 / argmax) is applied per model and the
// prediction goes to a small fp64 buffer pred[row][model]; `vote_kernel` then applies the VotingEnsemble
// reduce (routers.py:708-741) and the row status.  Rows are read once per model (M x 4*n_in bytes/event,
// mostly from L2): the path is bound by shared-memory gather throughput (wavefronts), not by HBM.
#pragma once
#include "b2s_device.cuh"

namespace b2s {

struct HeapNode {
  int32_t feature;
  float threshold;  // go right when !(x <= threshold)
};

struct T2Model {  // one per model, in global memory
  const HeapNode* nodes;   // [n_trees][n_internal]
  const double* leaves;    // [n_trees][n_leaves]
  const int32_t* slot;     // [n_trees]
  const double* scale;     // [n_trees]
  int32_t n_trees, depth, n_internal, n_leaves;
};

struct T2Params {
  const char* rows;
  int64_t row_stride;
  int64_t n_rows;
  double* pred;        // [n_rows][n_models]
  int32_t* row_bad;    // [n_rows] non-finite input flags (written by the CTAs of model 0)
  int32_t n_in, n_models, tile_rows, pitch, stages, vec_ok, groups;
  int32_t use_tmap;    // the landing tile is filled by TMA box copies (128-byte swizzle) instead of cp.async
  const T2Model* t2;   // [n_models]
  const ModelDesc* models;
  const int32_t* classes;
  const double* bias;  // init scores, indexed by ModelDesc.score_off
  int32_t sm_tables, sm_part, sm_tiles;  // byte offsets
};

constexpr int kT2TileRows = 64;  // rows per tile (threads r = 0..63 of a tree group)
#ifndef B2S_T2_GROUPS
#define B2S_T2_GROUPS 8
#endif
constexpr int kT2Groups = B2S_T2_GROUPS;  // tree groups per CTA: thread (g, r) walks trees g, g+G, ... of row r

// Shared-memory layout of one model (built once per CTA from the T2Model arrays):
//   s_foff[t][1..NI]  byte offset of the node's feature column inside the transposed tile (feature * TR * 4)
//   s_thr [t][1..NI]  float32 threshold                      (1-based heap: children of n are 2n, 2n+1)
//   s_leaf[t][NL]     tree_scale * leaf value (fp64; the product the scalar path computes per visit)
//   s_slot[t]         score slot of the tree (multi-class models)
// The event tile is TRANSPOSED in shared memory (xt[feature][row]): the 32 lanes of a warp are 32 consecutive
// rows walking the same tree, so the feature gather hits 32 different banks whatever features the lanes are
// at; with row-major tiles (pitch = 4 words mod 32) the same gather is a 4-way bank conflict.  Node words of
// one level are consecutive 4-byte words: lanes at different nodes of a level never conflict either.
template <int NS>
__global__ void __launch_bounds__(kT2TileRows * kT2Groups) trees_model_kernel(const __grid_constant__ T2Params p, const __grid_constant__ CUtensorMap tmap) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int tid = threadIdx.x;
  const int m = blockIdx.x % p.n_models;
  const int part = blockIdx.x / p.n_models;
  const int nparts = (gridDim.x - m + p.n_models - 1) / p.n_models;  // CTAs working on model m
  const T2Model tm = p.t2[m];
  const ModelDesc md = p.models[m];
  constexpr int TR = kT2TileRows;  // compile-time: the transpose's index arithmetic is shifts and masks
  constexpr int G = kT2Groups;
  const int NI = tm.n_internal, NL = tm.n_leaves, NT = tm.n_trees;

  // ---- the model's tables -> shared memory (once)
  const int n_nodes = NT * NI;
  int32_t* s_foff = reinterpret_cast<int32_t*>(smem + p.sm_tables);
  float* s_thr = reinterpret_cast<float*>(s_foff + n_nodes);
  double* s_leaf = reinterpret_cast<double*>(smem + p.sm_tables + (((size_t)n_nodes * 8 + 15) / 16) * 16);
  int32_t* s_slot = reinterpret_cast<int32_t*>(s_leaf + (size_t)NT * NL);
  for (int i = tid; i < n_nodes; i += blockDim.x) {
    const HeapNode nd = tm.nodes[i];
    s_foff[i] = nd.feature * TR * 4;
    s_thr[i] = nd.threshold;
  }
  for (int i = tid; i < NT * NL; i += blockDim.x) s_leaf[i] = __dmul_rn(tm.scale[i / NL], tm.leaves[i]);
  for (int i = tid; i < NT; i += blockDim.x) s_slot[i] = tm.slot[i];
  double* s_part = reinterpret_cast<double*>(smem + p.sm_part);  // [groups - 1][tile_rows][NS]
  float* s_stage = reinterpret_cast<float*>(smem + p.sm_tiles);  // row-major landing tile (cp.async / TMA boxes)
  {  // 1024-byte aligned (TMA swizzle atom); the host reserved the slack
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(s_stage);
    s_stage += ((1024u - (a & 1023u)) & 1023u) >> 2;
  }
  float* s_xt = s_stage + (size_t)TR * p.pitch;                  // transposed tile [n_in][TR]
  int* s_bad = reinterpret_cast<int*>(s_xt + (size_t)((p.n_in + 3) / 4 * 4) * TR);  // per-row "non-finite input" flags
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(s_bad + TR);                        // mbarrier of the TMA loads
  if (tid < TR) s_bad[tid] = 0;
  const bool tma = p.use_tmap != 0;
  if (tma && tid == 0) {
    mbar_init(s_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  uint32_t tma_phase = 0;

  const int64_t n_tiles = (p.n_rows + TR - 1) / TR;
  const int g = tid / TR;  // tree group (warp-uniform: TR is a multiple of 32)
  const int r = tid - g * TR;

  const int cprv = p.vec_ok ? (p.n_in >> 2) : p.n_in;
  const int r0 = tid / cprv, c0 = tid - r0 * cprv;
  const int dr = (int)blockDim.x / cprv, dc = (int)blockDim.x - dr * cprv;
  auto issue = [&](int64_t row0) {
    if (tma) {  // one thread: n_in / 32 box copies of (32 floats x TR rows); rows past the end arrive as zeros
      if (tid == 0) {
        const int boxes = p.n_in >> 5;
        mbar_expect_tx(s_bar, (uint32_t)boxes * (uint32_t)TR * 128u);
        for (int b = 0; b < boxes; ++b) tensor_load_2d(s_stage + b * TR * 32, &tmap, b * 32, (int)row0, s_bar);
      }
      return;
    }
    int64_t left = p.n_rows - row0;
    const int rows = left < TR ? (left < 0 ? 0 : (int)left) : TR;
    const char* base = p.rows + row0 * p.row_stride;
    int rr = r0, cc = c0;
    while (rr < rows) {
      if (p.vec_ok)
        cp_async16(s_stage + rr * p.pitch + cc * 4, base + (int64_t)rr * p.row_stride + cc * 16);
      else
        cp_async4(s_stage + rr * p.pitch + cc, base + (int64_t)rr * p.row_stride + cc * 4);
      rr += dr;
      cc += dc;
      if (cc >= cprv) {
        cc -= cprv;
        ++rr;
      }
    }
  };

  if (tma) __syncthreads();  // the barrier is initialised before anybody can wait on it
  if ((int64_t)part < n_tiles) issue((int64_t)part * TR);
  cp_async_commit();
  const char* xt_r = reinterpret_cast<const char*>(s_xt + r);
  const int leaf_bias = NL;  // n - NL is the leaf index
  for (int64_t t = part; t < n_tiles; t += nparts) {
    if (tma) {
      mbar_wait(s_bar, tma_phase);
      tma_phase ^= 1u;
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();  // landing tile (and, first time round, the tables) visible; the previous walk is over
    {                 // transpose: lanes take consecutive rows, so both the LDS and the STS are conflict-free
      const int64_t left = p.n_rows - t * TR;
      const int rows = left < TR ? (int)left : TR;
      // every thread keeps the same row rr = tid % TR through the loop (blockDim is a multiple of TR), so it can also
      // collect "this row holds a non-finite value" on the way; the G threads of a row merge their flags in shared memory
      int bad = 0;
      if ((p.n_in & 3) == 0) {  // one 16-byte LDS per (row, chunk), four 4-byte STS
        for (int i = tid; i < (p.n_in >> 2) * TR; i += blockDim.x) {
          const int c = i / TR, rr = i - c * TR;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (rr < rows)
            v = tma ? *reinterpret_cast<const float4*>(s_stage + (c >> 3) * (TR * 32) + rr * 32 + (((c & 7) ^ (rr & 7)) << 2))
                    : *reinterpret_cast<const float4*>(s_stage + rr * p.pitch + c * 4);
          bad |= (is_finite_f(v.x) && is_finite_f(v.y) && is_finite_f(v.z) && is_finite_f(v.w)) ? 0 : 1;
          float* o = s_xt + (size_t)(c * 4) * TR + rr;
          o[0] = v.x;
          o[TR] = v.y;
          o[2 * TR] = v.z;
          o[3 * TR] = v.w;
        }
      } else {
        for (int i = tid; i < p.n_in * TR; i += blockDim.x) {
          const int f = i / TR, rr = i - f * TR;
          const float v = rr < rows ? s_stage[rr * p.pitch + f] : 0.0f;
          bad |= is_finite_f(v) ? 0 : 1;
          s_xt[i] = v;
        }
      }
      if (m == 0 && bad) atomicOr(&s_bad[tid % TR], 1);
    }
    __syncthreads();  // transposed tile visible; landing tile free
    {
      const int64_t tn = t + nparts;
      if (tn < n_tiles) issue(tn * TR);
      cp_async_commit();
    }
    const int64_t row = t * TR + r;
    const bool live = row < p.n_rows;
    double acc[NS];
#pragma unroll
    for (int k = 0; k < NS; ++k) acc[k] = 0.0;
    if (live) {
      constexpr int U = 4;  // independent root->leaf walks in flight per thread (ILP over the LDS latency)
      int tr = g;
      for (; tr + (U - 1) * G < NT; tr += U * G) {
        int n4[U];
#pragma unroll
        for (int u = 0; u < U; ++u) n4[u] = 4;  // node 1 (byte index)
        for (int d = 0; d < tm.depth; ++d) {
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int at = (tr + u * G) * NI * 4 - 4 + n4[u];  // 1-based
            const int foff = *reinterpret_cast<const int32_t*>(reinterpret_cast<const char*>(s_foff) + at);
            const float thr = *reinterpret_cast<const float*>(reinterpret_cast<const char*>(s_thr) + at);
            const float x = *reinterpret_cast<const float*>(xt_r + foff);
            n4[u] = 2 * n4[u] + ((x <= thr) ? 0 : 4);  // sklearn: left when x <= threshold
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int tu = tr + u * G;
          const double v = s_leaf[tu * NL + (n4[u] >> 2) - leaf_bias];
          if (NS == 1) {
            acc[0] = __dadd_rn(acc[0], v);
          } else {
            const int slot = s_slot[tu];
#pragma unroll
            for (int k = 0; k < NS; ++k)
              if (k == slot) acc[k] = __dadd_rn(acc[k], v);
          }
        }
      }
      for (; tr < NT; tr += G) {  // remaining trees of the group, one at a time (same order of additions)
        int n4 = 4;
        for (int d = 0; d < tm.depth; ++d) {
          const int at = tr * NI * 4 - 4 + n4;
          const int foff = *reinterpret_cast<const int32_t*>(reinterpret_cast<const char*>(s_foff) + at);
          const float thr = *reinterpret_cast<const float*>(reinterpret_cast<const char*>(s_thr) + at);
          const float x = *reinterpret_cast<const float*>(xt_r + foff);
          n4 = 2 * n4 + ((x <= thr) ? 0 : 4);
        }
        const double v = s_leaf[tr * NL + (n4 >> 2) - leaf_bias];
        if (NS == 1) {
          acc[0] = __dadd_rn(acc[0], v);
        } else {
          const int slot = s_slot[tr];
#pragma unroll
          for (int k = 0; k < NS; ++k)
            if (k == slot) acc[k] = __dadd_rn(acc[k], v);
        }
      }
    }
    if (g > 0) {
      double* o = s_part + ((size_t)(g - 1) * TR + r) * NS;
#pragma unroll
      for (int k = 0; k < NS; ++k) o[k] = acc[k];
    }
    __syncthreads();
    if (g == 0 && live) {
      double sc[NS];
#pragma unroll
      for (int k = 0; k < NS; ++k) sc[k] = (k < md.n_scores ? p.bias[md.score_off + k] : 0.0) + acc[k];
      for (int gg = 1; gg < G; ++gg) {
        const double* o = s_part + ((size_t)(gg - 1) * TR + r) * NS;
#pragma unroll
        for (int k = 0; k < NS; ++k) sc[k] += o[k];
      }
      p.pred[row * p.n_models + m] = apply_link(md, sc, p.classes);
    }
    if (m == 0 && g == 1 && live) {  // flags gathered during the transpose; reset for the next tile
      p.row_bad[row] = s_bad[r];
      s_bad[r] = 0;
    }
  }
  cp_async_wait<0>();
}

// VotingEnsemble reduce over pred[row][model] -> out (+ status)
__global__ void __launch_bounds__(256) vote_kernel(KParams kp, const double* __restrict__ pred_buf,
                                                   const int32_t* __restrict__ row_bad) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < kp.n_rows; row += stride) {
    double pred[kMaxModels];
    for (int m = 0; m < kp.n_models; ++m) pred[m] = pred_buf[row * kp.n_models + m];
    vote_and_store(kp, pred, row, row_bad[row] ? 1u : 0u);
  }
  merge_signal(kp.sig);
}

}  // namespace b2s
