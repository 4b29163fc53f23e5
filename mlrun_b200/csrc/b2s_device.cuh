// b2s_device.cuh -- device-side plan tables and the row kernels (sm_90a).
//
// One kernel family, `rows_kernel<MODE, NS>`, runs a *fused row program* over a batch of events:
//
//   HBM rows --cp.async (LDGSTS.128), STAGES-deep ring--> shared-memory tile (padded pitch)
//     stage 1  per-column ops      : Imputer (NaN -> fill), MapValues (value / range maps)
//     stage 2  output schema       : COPY / ONEHOT(category) columns  (never materialised for LINEAR)
//     stage 3  consumer            : LINEAR  fp64 dot with the one-hot folded into a gather
//                                    TREES   root->leaf walks over SoA node tables, fp64 leaf sums
//                                    STORE   write the transformed row
//     stage 4  links + vote        : regression / threshold / argmax, VotingEnsemble mean / majority
//
// Each input byte is read from HBM once and each output word written once: the algorithmic bytes of
// DESIGN.md ("bytes per event") are what the kernel moves.  Persistent grid (a multiple of the SM
// count), one thread per row inside a tile, tables resident in shared memory.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2s {

enum Mode { MODE_LINEAR = 0, MODE_TREES = 1, MODE_STORE = 2 };
enum ModelKind { MK_LINEAR = 0, MK_TREES = 1 };

constexpr int kMaxModels = 16;
constexpr int kMaxScores = 32;
constexpr uint32_t COL_COPIED = 1u;  // column feeds a COPY output (a non-finite value there is an error)
constexpr uint32_t COL_HAS_MAP = 2u;
constexpr uint32_t COL_HAS_CAT = 4u;

struct MapEntry {  // MapValues entry: kind 0: v == a -> val ; kind 1: a <= v < b -> val
  float a, b, val;
  int32_t kind;
};

struct TreeNode {  // 16 B: one LDG.128 per level
  int32_t feature;  // < 0: leaf;  kTreeCatBit | f: a categorical split on column f
  float threshold;  // go left when x <= threshold;  categorical: the bits are the word offset of its set (tree_cat_right)
  int32_t left, right;
};

// Categorical nodes of rows_kernel<TREES>.  The sets follow the node table, each as [header][words]: header = number of
// 32-bit words | (bit 31) the model's code mode (B2S_CAT_TRUNC); `at` is the header's word offset from the start of the
// table.  The node goes right iff x is a valid code whose bit is set.
constexpr int32_t kTreeCatBit = 0x40000000;
__device__ __forceinline__ bool tree_cat_right(const uint32_t* __restrict__ sets, uint32_t at, float x) {
  const uint32_t hdr = __ldg(sets + at);
  // valid codes: x >= 0 (xgboost) or x > -1, i.e. trunc(x) >= 0 (LightGBM); past the set (or past int32) is outside it
  const float lo = (hdr >> 31) ? -0.99999994f : 0.0f;
  if (!(x >= lo && x < __uint2float_rz(hdr & 0x7fffffffu) * 32.0f)) return false;
  const int c = __float2int_rz(x);
  return (__ldg(sets + at + 1 + (c >> 5)) >> (c & 31)) & 1u;
}

struct ModelDesc {
  int32_t kind;        // ModelKind
  int32_t score_off;   // first score slot of this model
  int32_t n_scores;
  int32_t link;        // B2S_LINK_*
  int32_t class_off;   // into classes[]
  int32_t n_classes;
  int32_t tree_begin;  // TREES: range in tree arrays
  int32_t tree_end;
  int32_t w_off;       // generic linear (TREES mode): offset into wgen (n_scores x n_out doubles)
  int32_t pad;
};

// Completion signal of the fused ensemble-merge (b2s_comm_*): when every CTA of the launch that stores the votes has
// finished, the last one publishes `epoch` in slot `rank` of EVERY target's flag array with a system-scope release store;
// a reader that acquires all n flags of its own array at `epoch` therefore sees every shard's rows of that step.
struct MergeSig {
  uint32_t* flags[8];  // the flag array of every target (own GPU included), in peer memory (NVLink)
  uint32_t* counter;   // CTAs of this launch that are done (this GPU's memory; the last one resets it)
  int32_t n;           // 0: no signal
  int32_t rank;
  uint32_t epoch;
  // fused wait (b2s_comm_set_fused_wait): after publishing, the launch's last CTA also acquires THIS rank's n flags until they
  // show wait_epoch (epoch, or epoch - 1 for pipelined steps), so that what follows the kernel on its stream reads a
  // complete response without a separate wait kernel.  0 = no fused wait.
  uint32_t wait_epoch;
  const uint32_t* wait_flags;
  uint32_t* timeout_flag;
  long long timeout_ns;
};

__device__ __forceinline__ void merge_signal(const MergeSig& m) {
  if (m.n <= 0) return;
  // every thread's vote stores -> CTA barrier -> ONE system-scope fence by thread 0 (fences are cumulative: the stores thread 0
  // has observed through the barrier are ordered before everything it writes after the fence).  The fence waits for the CTA's
  // peer stores to be acknowledged: about one NVLink round trip at the tail of the launch.
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    const unsigned prev = atomicAdd(m.counter, 1u);
    if (prev == gridDim.x - 1) {  // every other CTA has fenced its stores and counted itself
      *m.counter = 0;             // launches of a plan are stream ordered: the next one finds a clean counter
      __threadfence_system();
      for (int g = 0; g < m.n; ++g)
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(m.flags[g] + m.rank), "r"(m.epoch) : "memory");
      if (m.wait_epoch) {  // fused wait: every source rank's flag of step wait_epoch (or a later one)
        long long t0 = 0;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
        for (int g = 0; g < m.n; ++g) {
          for (;;) {
            uint32_t v;
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(m.wait_flags + g) : "memory");
            if ((int32_t)(v - m.wait_epoch) >= 0) break;
            long long t1;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
            if (t1 - t0 > m.timeout_ns) {  // a peer died: give up instead of hanging the GPU; b2s_comm_check reports it
              atomicExch(m.timeout_flag, 1u + (uint32_t)g);
              break;
            }
            __nanosleep(100);
          }
        }
      }
    }
  }
}

struct KParams {
  // ---- batch
  const char* rows;
  int64_t row_stride;  // bytes
  int64_t n_rows;
  float* out;          // n_rows x out_cols 4-byte words
  int32_t* status;     // may be null
  // ---- shapes
  int32_t n_in, n_out, out_cols, n_models, n_scores, vote_kind;
  int32_t tile_rows, pitch, stages, vec_ok;  // vec_ok: rows 16B aligned -> 16B cp.async
  int32_t exp_pitch, need_expand, models_pow2, out_is_int;
  // ---- tables (global memory; the small ones are copied to shared memory at kernel start)
  const float* fill;          // [n_in]   NaN = column not imputed
  const uint32_t* col_flags;  // [n_in]
  const int32_t* map_off;     // [n_in+1]
  const MapEntry* maps;
  const int32_t* out_src;     // [n_out]
  const int32_t* out_kind;
  const float* out_arg;
  const int32_t* cat_off;     // [n_in+1]  LINEAR: categories folded per input column
  const float* cat_val;
  const double* wnum;         // [n_in][NS]
  const double* wcat;         // [n_cat][NS]
  const double* bias;         // [NS]   (linear intercepts / tree init scores)
  const ModelDesc* models;    // [n_models]
  const int32_t* classes;
  const double* vote_w;       // [n_models]
  const double* wgen;         // generic linear weights for TREES mode
  const TreeNode* nodes;
  const double* leaf;         // leaf value per node index
  const int32_t* tree_root;   // [n_trees] node index of each tree's root
  const int32_t* tree_slot;   // [n_trees]
  const double* tree_scale;   // [n_trees]
  // ---- shared-memory carve-up (byte offsets), computed on the host
  int32_t sm_fill, sm_flags, sm_mapoff, sm_catoff, sm_catval, sm_wnum, sm_wcat, sm_tiles, sm_exp, sm_pred,
      sm_outsrc, sm_outkind, sm_outarg, sm_total;
  int32_t n_cat, n_maps;
  // ensemble-merge targets: when n_peers > 0 every output row is stored into each peer's buffer (own GPU
  // included) at row `peer_off + row` -- NVLink P2P stores from the epilogue replace a separate all-gather
  float* peers[8];
  int64_t peer_off;
  int32_t n_peers;
  int32_t tpr;                // LINEAR: threads per row (slices of the row's 16-byte chunks)
  int32_t sm_part, sm_pst, sm_chunk;
  const uint8_t* chunk_kind;  // [ceil(n_in/4)] 0 = four plain numeric columns (fast path), 1 = generic
  MergeSig sig;               // completion signal of the ensemble-merge (kernels that store the votes)
};

// ------------------------------------------------------------------------------------------ helpers
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
  uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

__device__ __forceinline__ bool is_finite_f(float x) { return fabsf(x) <= 3.402823466e+38f; }  // false for NaN/Inf

// MapValues._map_value (feature_store/steps.py:189-201): maps run in the order they were added; within a
// range map the first matching [lo, hi) wins; an unmatched value passes through unchanged.
__device__ __forceinline__ float apply_maps(float x, const MapEntry* __restrict__ maps, int lo, int hi) {
  // entries of one column are grouped by the map they belong to via kind sign: a new map starts at an
  // entry whose kind has bit 8 set.  Within one map: first hit wins, then we skip to the next map.
  bool hit = false;
  for (int i = lo; i < hi; ++i) {
    MapEntry e = maps[i];
    if (e.kind & 256) hit = false;  // start of the next map applied to this column
    if (hit) continue;
    int k = e.kind & 255;
    bool m = (k == 0) ? (x == e.a) : (x >= e.a && x < e.b);
    if (m) {
      x = e.val;
      hit = true;
    }
  }
  return x;
}

// issue the asynchronous copy of one tile of rows into shared memory (all threads cooperate)
__device__ __forceinline__ void issue_tile(const KParams& p, float* tile, int64_t row0) {
  int64_t left = p.n_rows - row0;
  int rows = left < p.tile_rows ? (left < 0 ? 0 : (int)left) : p.tile_rows;
  const char* base = p.rows + row0 * p.row_stride;
  // (row, chunk) walk without per-iteration division
  if (p.vec_ok) {
    const int cpr = p.n_in >> 2;  // 16-byte chunks per row
    int r = threadIdx.x / cpr, c = threadIdx.x - r * cpr;
    const int dr = blockDim.x / cpr, dc = blockDim.x - dr * cpr;
    while (r < rows) {
      cp_async16(tile + r * p.pitch + c * 4, base + (int64_t)r * p.row_stride + c * 16);
      r += dr;
      c += dc;
      if (c >= cpr) {
        c -= cpr;
        ++r;
      }
    }
  } else {
    int r = threadIdx.x / p.n_in, c = threadIdx.x - r * p.n_in;
    const int dr = blockDim.x / p.n_in, dc = blockDim.x - dr * p.n_in;
    while (r < rows) {
      cp_async4(tile + r * p.pitch + c, base + (int64_t)r * p.row_stride + c * 4);
      r += dr;
      c += dc;
      if (c >= p.n_in) {
        c -= p.n_in;
        ++r;
      }
    }
  }
}

__device__ __forceinline__ TreeNode load_node(const TreeNode* __restrict__ q) {
  const int4 v = __ldg(reinterpret_cast<const int4*>(q));
  TreeNode n;
  n.feature = v.x;
  n.threshold = __int_as_float(v.y);
  n.left = v.z;
  n.right = v.w;
  return n;
}

// link function of one model: raw scores -> prediction (double for regression, label for classifiers)
__device__ __forceinline__ double apply_link(const ModelDesc& md, const double* __restrict__ s,
                                             const int32_t* __restrict__ classes) {
  switch (md.link) {
    case 1: {  // B2S_LINK_BINARY_GT
      int idx = s[0] > 0.0 ? 1 : 0;
      return md.n_classes ? (double)classes[md.class_off + idx] : (double)idx;
    }
    case 2: {  // B2S_LINK_BINARY_GE
      int idx = s[0] >= 0.0 ? 1 : 0;
      return md.n_classes ? (double)classes[md.class_off + idx] : (double)idx;
    }
    case 3: {  // B2S_LINK_ARGMAX (first max wins, like np.argmax)
      int best = 0;
      double bv = s[0];
      for (int k = 1; k < md.n_scores; ++k)
        if (s[k] > bv) {
          bv = s[k];
          best = k;
        }
      return md.n_classes ? (double)classes[md.class_off + best] : (double)best;
    }
    default:
      return s[0];
  }
}

// one 4-byte output word of row `row`: local buffer, or every merge target (fused ensemble-merge)
template <typename P>
__device__ __forceinline__ void store_word(const P& p, int64_t row, int col, uint32_t bits) {
  if (p.n_peers == 0) {
    reinterpret_cast<uint32_t*>(p.out)[row * p.out_cols + col] = bits;
  } else {
    for (int g = 0; g < p.n_peers; ++g)
      reinterpret_cast<uint32_t*>(p.peers[g])[(p.peer_off + row) * p.out_cols + col] = bits;
  }
}

// VotingEnsemble reduce over per-model predictions (serving/routers.py:708-741); writes out_cols words.
__device__ __forceinline__ void vote_and_store(const KParams& p, const double* __restrict__ pred, int64_t row,
                                               uint32_t st) {
  const int M = p.n_models;
  if (p.vote_kind == 0) {  // B2S_VOTE_NONE: every model's prediction
    for (int m = 0; m < M; ++m)
      store_word(p, row, m, p.out_is_int ? (uint32_t)(int32_t)pred[m] : __float_as_uint((float)pred[m]));
  } else if (p.vote_kind == 1) {  // _mean_vote: (n,m) @ w(m) in fp64, model order
    double acc = 0.0;
    for (int m = 0; m < M; ++m) acc = __dadd_rn(acc, __dmul_rn(pred[m], p.vote_w[m]));
    store_word(p, row, 0, __float_as_uint((float)acc));
  } else {  // _majority_vote: tallies per class in fp64 (model order), argmax with first-max tie break
    int maxlab = -1;
    for (int m = 0; m < M; ++m) {
      int c = (int)pred[m];
      if (c < 0) st |= 2u;  // B2S_ROW_BAD_LABEL: np.arange(max+1) never matches a negative label
      maxlab = c > maxlab ? c : maxlab;
    }
    double best_t = 0.0;
    int best_c = -1;
    for (int m = 0; m < M; ++m) {
      int c = (int)pred[m];
      if (c < 0) continue;
      bool seen = false;
      for (int q = 0; q < m; ++q) seen |= ((int)pred[q] == c);
      if (seen) continue;
      double t = 0.0;
      for (int q = m; q < M; ++q)
        if ((int)pred[q] == c) t = __dadd_rn(t, p.vote_w[q]);
      if (best_c < 0 || t > best_t || (t == best_t && c < best_c)) {
        best_t = t;
        best_c = c;
      }
    }
    // classes nobody voted for have tally 0.0 and take part in the argmax (lowest index wins ties)
    if (maxlab >= 0) {
      int c0 = 0;
      bool used = true;
      while (used && c0 <= maxlab) {
        used = false;
        for (int m = 0; m < M; ++m) used |= ((int)pred[m] == c0);
        if (used) ++c0;
      }
      if (c0 <= maxlab && (best_c < 0 || 0.0 > best_t || (0.0 == best_t && c0 < best_c))) best_c = c0;
    }
    store_word(p, row, 0, (uint32_t)(best_c < 0 ? 0 : best_c));
  }
  if (p.status) p.status[row] = (int32_t)st;
}

// ------------------------------------------------------------------------------------------ the kernel
// NS = number of score slots held in registers per thread (LINEAR: all models' scores; TREES: one model's).
template <int MODE, int NS>
__global__ void __launch_bounds__(512) rows_kernel(const __grid_constant__ KParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  float* s_fill = reinterpret_cast<float*>(smem + p.sm_fill);
  uint32_t* s_flags = reinterpret_cast<uint32_t*>(smem + p.sm_flags);
  int32_t* s_mapoff = reinterpret_cast<int32_t*>(smem + p.sm_mapoff);
  int32_t* s_catoff = reinterpret_cast<int32_t*>(smem + p.sm_catoff);
  float* s_catval = reinterpret_cast<float*>(smem + p.sm_catval);
  double* s_wnum = reinterpret_cast<double*>(smem + p.sm_wnum);
  double* s_wcat = reinterpret_cast<double*>(smem + p.sm_wcat);
  float* s_tiles = reinterpret_cast<float*>(smem + p.sm_tiles);
  float* s_exp = reinterpret_cast<float*>(smem + p.sm_exp);
  double* s_pred = reinterpret_cast<double*>(smem + p.sm_pred);
  int32_t* s_outsrc = reinterpret_cast<int32_t*>(smem + p.sm_outsrc);
  int32_t* s_outkind = reinterpret_cast<int32_t*>(smem + p.sm_outkind);
  double* s_part = reinterpret_cast<double*>(smem + p.sm_part);
  uint32_t* s_pst = reinterpret_cast<uint32_t*>(smem + p.sm_pst);
  uint8_t* s_chunk = reinterpret_cast<uint8_t*>(smem + p.sm_chunk);
  float* s_outarg = reinterpret_cast<float*>(smem + p.sm_outarg);

  const int tid = threadIdx.x;
  const int nthr = blockDim.x;
  const int TR = p.tile_rows;
  const int tile_words = TR * p.pitch;
  const int64_t n_tiles = (p.n_rows + TR - 1) / TR;

  // ---- kick off the first STAGES-1 tiles, then load the tables while they fly
  const int S = p.stages;
  for (int s = 0; s < S - 1; ++s) {
    int64_t t = (int64_t)blockIdx.x + (int64_t)s * gridDim.x;
    if (t < n_tiles) issue_tile(p, s_tiles + s * tile_words, t * TR);
    cp_async_commit();
  }
  for (int i = tid; i < p.n_in; i += nthr) {
    s_fill[i] = p.fill[i];
    s_flags[i] = p.col_flags[i];
  }
  for (int i = tid; i <= p.n_in; i += nthr) {
    s_mapoff[i] = p.map_off[i];
    if (MODE == MODE_LINEAR) s_catoff[i] = p.cat_off[i];
  }
  if (MODE == MODE_LINEAR) {
    for (int i = tid; i < p.n_cat; i += nthr) s_catval[i] = p.cat_val[i];
    for (int i = tid; i < ((p.n_in + 3) >> 2); i += nthr) s_chunk[i] = p.chunk_kind[i];
    for (int i = tid; i < p.n_in * NS; i += nthr) s_wnum[i] = p.wnum[i];
    for (int i = tid; i < p.n_cat * NS; i += nthr) s_wcat[i] = p.wcat[i];
  } else {
    for (int i = tid; i < p.n_out; i += nthr) {
      s_outsrc[i] = p.out_src[i];
      s_outkind[i] = p.out_kind[i];
      s_outarg[i] = p.out_arg[i];
    }
  }

  int stage = 0;
  for (int64_t t = blockIdx.x, it = 0; t < n_tiles; t += gridDim.x, ++it) {
    // tile `t` has landed when at most S-2 younger groups are still pending
    if (S == 1) {
      __syncthreads();  // single buffer: everybody must be done with the previous tile first
      issue_tile(p, s_tiles, t * TR);
      cp_async_commit();
      cp_async_wait<0>();
    } else if (S == 2) {
      cp_async_wait<0>();
    } else if (S == 3) {
      cp_async_wait<1>();
    } else {
      cp_async_wait<2>();
    }
    __syncthreads();  // tile visible to all threads; everybody is done with the previous tile
    if (S > 1) {
      int64_t tn = t + (int64_t)(S - 1) * gridDim.x;
      int sn = stage + S - 1;
      if (sn >= S) sn -= S;
      if (tn < n_tiles) issue_tile(p, s_tiles + sn * tile_words, tn * TR);
      cp_async_commit();
    }
    const float* tile = s_tiles + stage * tile_words;
    const int64_t row0 = t * TR;

    if (MODE == MODE_LINEAR) {
      // -------- TPR threads per row.  Thread (q, r) owns a contiguous slice of row r's 16-byte chunks;
      // q = tid / TR, so a warp is uniform in q: all its lanes work on the same columns (table reads are
      // broadcasts) of 32 consecutive rows (conflict-free LDS.128 with pitch = 16 mod 128 bytes).
      const int q = tid / TR;
      const int r = tid - q * TR;
      const int64_t row = row0 + r;
      double acc[NS];
#pragma unroll
      for (int k = 0; k < NS; ++k) acc[k] = 0.0;
      uint32_t st = 0;
      if (row < p.n_rows) {
        const float* xr = tile + r * p.pitch;
        const int nch = (p.n_in + 3) >> 2;
        const int cps = (nch + p.tpr - 1) / p.tpr;
        const int ch_end = min(nch, (q + 1) * cps);
        for (int ch = q * cps; ch < ch_end; ++ch) {
          const int c = ch << 2;
          const float4 v = *reinterpret_cast<const float4*>(xr + c);  // pad words are never used
          if (s_chunk[ch] == 0) {
            // fast path: 4 plain numeric columns (copied, no maps, no categories)
            const float4 f = *reinterpret_cast<const float4*>(s_fill + c);
            const float x0 = (v.x != v.x) ? f.x : v.x;
            const float x1 = (v.y != v.y) ? f.y : v.y;
            const float x2 = (v.z != v.z) ? f.z : v.z;
            const float x3 = (v.w != v.w) ? f.w : v.w;
            if (!(is_finite_f(x0) && is_finite_f(x1) && is_finite_f(x2) && is_finite_f(x3))) st |= 1u;
            const double* w = s_wnum + c * NS;
            const double d0 = (double)x0, d1 = (double)x1, d2 = (double)x2, d3 = (double)x3;
#pragma unroll
            for (int k = 0; k < NS; ++k) {
              double a = acc[k];
              a = fma(w[k], d0, a);
              a = fma(w[NS + k], d1, a);
              a = fma(w[2 * NS + k], d2, a);
              a = fma(w[3 * NS + k], d3, a);
              acc[k] = a;
            }
          } else {
            const float xs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const int cc = c + u;
              if (cc >= p.n_in) break;
              float x = xs[u];
              const float f = s_fill[cc];
              x = (x != x) ? f : x;  // Imputer: NaN -> fill (fill is NaN for columns without one)
              const uint32_t fl = s_flags[cc];
              if (fl & COL_HAS_MAP) x = apply_maps(x, p.maps, s_mapoff[cc], s_mapoff[cc + 1]);
              if (fl & COL_COPIED) {
                if (!is_finite_f(x)) st |= 1u;
                const double xd = (double)x;
                const double* w = s_wnum + cc * NS;
#pragma unroll
                for (int k = 0; k < NS; ++k) acc[k] = fma(w[k], xd, acc[k]);
              }
              if (fl & COL_HAS_CAT) {
                const int j1 = s_catoff[cc + 1];
                for (int j = s_catoff[cc]; j < j1; ++j) {
                  if (x == s_catval[j]) {  // OneHotEncoder: value == category -> that column is 1
                    const double* w = s_wcat + j * NS;
#pragma unroll
                    for (int k = 0; k < NS; ++k) acc[k] += w[k];
                  }
                }
              }
            }
          }
        }
      }
      if (p.tpr > 1) {  // combine the row's slices in a fixed order (deterministic fp64 sum)
        double* part = s_part + (size_t)(q * TR + r) * NS;
        if (q > 0) {
#pragma unroll
          for (int k = 0; k < NS; ++k) part[k] = acc[k];
          s_pst[q * TR + r] = st;
        }
        __syncthreads();
        if (q == 0) {
          for (int qq = 1; qq < p.tpr; ++qq) {
            const double* o = s_part + (size_t)(qq * TR + r) * NS;
#pragma unroll
            for (int k = 0; k < NS; ++k) acc[k] += o[k];
            st |= s_pst[qq * TR + r];
          }
        }
      }
      if (q == 0 && row < p.n_rows) {
        // links + vote index the scores dynamically: do that on a copy so acc[] stays in registers
        double sl[NS];
#pragma unroll
        for (int k = 0; k < NS; ++k) sl[k] = acc[k] + p.bias[k];
        double pred[kMaxModels];
        for (int m = 0; m < p.n_models; ++m) {
          const ModelDesc md = p.models[m];
          pred[m] = apply_link(md, sl + md.score_off, p.classes);
        }
        vote_and_store(p, pred, row, st);
      }
    } else {
      // -------- TREES / STORE: build the expanded (post one-hot) tile in shared memory when needed
      const float* xt = tile;
      int xpitch = p.pitch;
      if (p.need_expand) {  // (the barrier at the top of the loop already fenced the previous tile's readers)
        for (int r = tid; r < TR; r += nthr) {
          if (row0 + r >= p.n_rows) break;
          const float* xr = tile + r * p.pitch;
          float* er = s_exp + r * p.exp_pitch;
          for (int j = 0; j < p.n_out; ++j) {
            const int cc = s_outsrc[j];
            float x = xr[cc];
            const float f = s_fill[cc];
            x = (x != x) ? f : x;
            if (s_flags[cc] & COL_HAS_MAP) x = apply_maps(x, p.maps, s_mapoff[cc], s_mapoff[cc + 1]);
            er[j] = (s_outkind[j] == 1) ? ((x == s_outarg[j]) ? 1.0f : 0.0f) : x;
          }
        }
        __syncthreads();
        xt = s_exp;
        xpitch = p.exp_pitch;
      }
      if (MODE == MODE_STORE) {
        // coalesced copy-out of the transformed tile
        int64_t left = p.n_rows - row0;
        int rows = left < TR ? (int)left : TR;
        const int total = rows * p.n_out;
        float* o = p.out + row0 * p.n_out;
        for (int i = tid; i < total; i += nthr) {
          int r = i / p.n_out, j = i - r * p.n_out;
          o[i] = xt[r * xpitch + j];
        }
        if (p.status)
          for (int r = tid; r < rows; r += nthr) p.status[row0 + r] = 0;
      } else {
        // one thread per (model, row): warps are uniform in the model -> they walk the same trees
        const int m = tid / TR;
        const int r = tid - m * TR;
        const int64_t row = row0 + r;
        if (m < p.n_models && row < p.n_rows) {
          const ModelDesc md = p.models[m];
          const float* xr = xt + r * xpitch;
          double sc[NS];
#pragma unroll
          for (int k = 0; k < NS; ++k) sc[k] = (k < md.n_scores) ? p.bias[md.score_off + k] : 0.0;
          if (md.kind == MK_TREES) {
            for (int tr = md.tree_begin; tr < md.tree_end; ++tr) {
              int node = p.tree_root[tr];
              TreeNode nd = load_node(p.nodes + node);
              for (;;) {
                // sklearn Tree.apply: go left when X[i, feature] <= threshold (float32 x).  The unsigned compare also
                // leaves the loop at a leaf (feature < 0) and at a categorical node
                while ((uint32_t)nd.feature < (uint32_t)kTreeCatBit) {
                  const float x = xr[nd.feature];
                  node = (x <= nd.threshold) ? nd.left : nd.right;
                  nd = load_node(p.nodes + node);
                }
                if (nd.feature < 0) break;
                const float x = xr[nd.feature & (kTreeCatBit - 1)];
                node = tree_cat_right(reinterpret_cast<const uint32_t*>(p.nodes), __float_as_uint(nd.threshold), x) ? nd.right : nd.left;
                nd = load_node(p.nodes + node);
              }
              const double v = __dmul_rn(p.tree_scale[tr], __ldg(p.leaf + node));
              const int slot = p.tree_slot[tr];
#pragma unroll
              for (int k = 0; k < NS; ++k)
                if (k == slot) sc[k] = __dadd_rn(sc[k], v);
            }
          } else {  // generic linear model inside a mixed ensemble
            const double* w = p.wgen + md.w_off;
            for (int j = 0; j < p.n_out; ++j) {
              const double xd = (double)xr[j];
#pragma unroll
              for (int k = 0; k < NS; ++k)
                if (k < md.n_scores) sc[k] = fma(w[k * p.n_out + j], xd, sc[k]);
            }
          }
          s_pred[r * p.models_pow2 + m] = apply_link(md, sc, p.classes);
        }
        __syncthreads();
        if (tid < TR && row0 + tid < p.n_rows) {
          // status: any non-finite value in the row the models saw
          uint32_t st = 0;
          const float* xr = xt + tid * xpitch;
          const int nf = p.need_expand ? p.n_out : p.n_in;
          for (int j = 0; j < nf; ++j)
            if (!is_finite_f(xr[j])) st |= 1u;
          double pred[kMaxModels];
          for (int mm = 0; mm < p.n_models; ++mm) pred[mm] = s_pred[tid * p.models_pow2 + mm];
          vote_and_store(p, pred, row0 + tid, st);
        }
      }
    }
    ++stage;
    if (stage == S) stage = 0;
  }
  cp_async_wait<0>();
  if (MODE != MODE_STORE) merge_signal(p.sig);
}

}  // namespace b2s
