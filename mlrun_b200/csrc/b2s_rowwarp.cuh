// b2s_rowwarp.cuh -- the HBM-bound linear path: a register-resident "row-warp" kernel (sm_90a).
//
// Imputer -> OneHotEncoder -> {linear scorers} -> vote is a (B x F)·(F x NS) product with a tiny NS
// (1..8 scores), i.e. a streaming, HBM-bound row reduction -- not GEMM-shaped work, so no tensor cores.
// Layout of the work:
//
//   * L lanes own one event row; lane j loads CPL 16-byte chunks of it (chunks j, j+L) straight from
//     HBM -- coalesced LDG.128s covering whole 128-byte lines, 32/L consecutive rows per warp
//     instruction, no shared-memory staging: every byte is read exactly once and used from registers;
//   * each lane keeps the weights of *its* 4*CPL columns for all NS scores, and their Imputer fills,
//     in registers for the whole kernel (persistent warps, grid = SMs x resident blocks);
//   * U row slots are in flight per lane (U*CPL independent loads), giving V = U*NS partial sums per
//     lane; the cross-lane sum is a reduce-scatter butterfly (V/2 + V/4 + ... exchanges instead of
//     V*log2 L), fp64 throughout, after which lane i holds one finished score (row i / NS, score i % NS);
//   * categorical (one-hot) columns are handed to the lanes of the row round-robin with shuffles, so
//     that each lane resolves at most CS category look-ups per row; the one-hot row is never built:
//     "onehot(x) . w" is the gather  w[cat_base + index_of(x)];
//   * a non-finite model input shows up as a non-finite score (NaN/Inf survive every fma, also with a
//     zero weight), so the per-row status costs one test on the finished score;
//   * epilogue: bias, link, VotingEnsemble mean (a second, log2 NS-step butterfly) or the generic
//     link / majority-vote path on one lane per row; coalesced 4-byte stores.
#pragma once
#include "b2s_device.cuh"

namespace b2s {

struct RWParams {
  const char* rows;
  int64_t row_stride;
  int64_t n_rows;
  float* out;
  int32_t* status;
  int32_t n_in, nch, out_cols, n_models, vote_kind, out_is_int, fast_epilogue, n_cat_slots;
  // per-lane tables (global, read once per warp at kernel start); column c lives in lane (c/4) % L,
  // chunk slot (c/4) / L, component c % 4
  const float* fill;        // [CPL*L*4]   index (slot*L + lane)*4 + comp
  const uint32_t* copied;   // [CPL*L]     bit u: that column feeds a COPY output
  const double* w;          // [CPL*L*4*NS]
  const int32_t* cat_src;   // [CS*L] source position (slot*L + lane) of the categorical column a lane resolves; -1 none
  const int32_t* cat_comp;  // [CS*L] component (0..3) inside that chunk
  const int32_t* cat_base;  // [CS*L] first entry in cat_val / wcat
  const int32_t* cat_n;     // [CS*L] number of categories
  const float* cat_val;     // [n_cat]
  const double* wcat;       // [n_cat*NS]
  const double* bias;       // [NS]
  const double* vote_w;     // [n_models]
  const ModelDesc* models;
  const int32_t* classes;
  int32_t n_cat;
  uint32_t cat_pos_mask;  // bit (slot*4+comp): some lane holds a categorical column at that chunk position
};

__device__ __forceinline__ float4 ldg_stream(const void* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}

__device__ __forceinline__ double shfl_xor_d(double v, int off) {
  int lo = __double2loint(v), hi = __double2hiint(v);
  lo = __shfl_xor_sync(0xffffffffu, lo, off);
  hi = __shfl_xor_sync(0xffffffffu, hi, off);
  return __hiloint2double(hi, lo);
}
__device__ __forceinline__ double shfl_idx_d(double v, int src) {
  int lo = __double2loint(v), hi = __double2hiint(v);
  lo = __shfl_sync(0xffffffffu, lo, src);
  hi = __shfl_sync(0xffffffffu, hi, src);
  return __hiloint2double(hi, lo);
}
__device__ __forceinline__ bool is_finite_d(double x) { return fabs(x) <= 1.7976931348623157e308; }

// L lanes per row, CPL chunks per lane, NS score slots, U row slots in flight, CS categorical slots per lane
template <int L, int CPL, int NS, int U, int CS>
__global__ void __launch_bounds__(128, 3) rowwarp_kernel(const __grid_constant__ RWParams p) {
  constexpr int RPW = 32 / L;  // rows per warp instruction
  constexpr int V = U * NS;    // partial sums per lane
  static_assert(V <= L, "U is chosen so that U*NS <= L");
  constexpr int REP = L / V;       // lanes holding replicas of one finished value
  constexpr int GROUP = U * RPW;   // rows per warp iteration
  constexpr int CSA = CS > 0 ? CS : 1;
  constexpr int KC = 4;            // categories cached in registers per categorical slot

  extern __shared__ __align__(16) unsigned char smem[];
  float* s_catval = reinterpret_cast<float*>(smem);
  double* s_wcat = reinterpret_cast<double*>(smem + ((p.n_cat * 4 + 15) / 16) * 16);
  for (int i = threadIdx.x; i < p.n_cat; i += blockDim.x) s_catval[i] = p.cat_val[i];
  for (int i = threadIdx.x; i < p.n_cat * NS; i += blockDim.x) s_wcat[i] = p.wcat[i];
  for (int i = threadIdx.x; i < NS; i += blockDim.x) s_wcat[p.n_cat * NS + i] = 0.0;
  __syncthreads();

  const int lane = threadIdx.x & 31;
  const int lir = lane & (L - 1);  // lane in row
  const int half = lane / L;       // which of the RPW rows of a warp instruction

  // ---- per-lane constants, resident in registers for the whole kernel
  float fill[CPL][4];
  double w[CPL][4][NS];
  uint32_t cmask[CPL][4];  // all-ones where the column feeds a COPY output, else 0 (x & 0 = +0.0f)
  bool has_chunk[CPL];
#pragma unroll
  for (int c = 0; c < CPL; ++c) {
    const int pos = c * L + lir;
    has_chunk[c] = pos < p.nch;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      cmask[c][u] = ((p.copied[pos] >> u) & 1u) ? 0xffffffffu : 0u;
      fill[c][u] = p.fill[pos * 4 + u];
#pragma unroll
      for (int k = 0; k < NS; ++k) w[c][u][k] = p.w[(pos * 4 + u) * NS + k];
    }
  }
  int cat_lane[CSA], cat_sel[CSA], cat_base[CSA], cat_n[CSA];
  float cat_c[CSA][KC];
#pragma unroll
  for (int s = 0; s < CS; ++s) {
    const int src = p.cat_src[s * L + lir];
    cat_lane[s] = src < 0 ? -1 : (src % L);
    cat_sel[s] = src < 0 ? -1 : (src / L) * 4 + p.cat_comp[s * L + lir];  // which of the CPL*4 values
    cat_base[s] = p.cat_base[s * L + lir];
    cat_n[s] = p.cat_n[s * L + lir];
#pragma unroll
    for (int j = 0; j < KC; ++j) cat_c[s][j] = (src >= 0 && j < cat_n[s]) ? p.cat_val[cat_base[s] + j] : __int_as_float(0x7fc00000);
  }
  // after the butterfly this lane owns value index `own` = (row slot, score slot)
  const int own = lir / REP;
  const int own_i = own / NS, own_k = own % NS;
  const double my_bias = p.bias[own_k];
  const double my_vw = (p.vote_kind == 1) ? p.vote_w[own_k < p.n_models ? own_k : 0] : 1.0;

  const int warps_per_block = blockDim.x >> 5;
  const int64_t n_groups = (p.n_rows + GROUP - 1) / GROUP;
  const int64_t gstride = (int64_t)gridDim.x * warps_per_block;
  const int64_t row_step = (int64_t)RPW * p.row_stride;
  // U*CPL independent 16-byte loads per lane; the next group's loads are issued before this group's math
  auto load_group = [&](int64_t g, float4 (&dst)[U][CPL]) {
    const int64_t base = g * GROUP;
    const bool full = base + GROUP <= p.n_rows;
    const char* gp = p.rows + (base + half) * p.row_stride + lir * 16;
#pragma unroll
    for (int i = 0; i < U; ++i) {
#pragma unroll
      for (int c = 0; c < CPL; ++c) {
        if (has_chunk[c] && (full || base + i * RPW + half < p.n_rows))
          dst[i][c] = ldg_stream(gp + i * row_step + c * (L * 16));
        else
          dst[i][c] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  };
  int64_t g = (int64_t)blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  float4 xn[U][CPL];
  if (g < n_groups) load_group(g, xn);
  for (; g < n_groups; g += gstride) {
    const int64_t base = g * GROUP;
    float4 x[U][CPL];
#pragma unroll
    for (int i = 0; i < U; ++i)
#pragma unroll
      for (int c = 0; c < CPL; ++c) x[i][c] = xn[i][c];
    if (g + gstride < n_groups) load_group(g + gstride, xn);
    double v[V];
#pragma unroll
    for (int i = 0; i < U; ++i) {
      float xs[CPL * 4];
      double a[NS];
#pragma unroll
      for (int k = 0; k < NS; ++k) a[k] = 0.0;
#pragma unroll
      for (int c = 0; c < CPL; ++c) {
        const float xr[4] = {x[i][c].x, x[i][c].y, x[i][c].z, x[i][c].w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          float xv = xr[u];
          xv = (xv != xv) ? fill[c][u] : xv;  // Imputer (fill is NaN where the column has none)
          xs[c * 4 + u] = xv;
          const double xd = (double)__uint_as_float(__float_as_uint(xv) & cmask[c][u]);
#pragma unroll
          for (int k = 0; k < NS; ++k) a[k] = fma(w[c][u][k], xd, a[k]);
        }
      }
      if (CS > 0 && p.n_cat_slots > 0) {
        // hand the categorical columns of this row to the lanes of the row, one value position per round
#pragma unroll
        for (int s = 0; s < CS; ++s) {
          float xc = 0.f;
          const int src_lane = half * L + (cat_lane[s] < 0 ? 0 : cat_lane[s]);
#pragma unroll
          for (int c = 0; c < CPL * 4; ++c) {
            if ((p.cat_pos_mask >> c) & 1u) {  // warp-uniform: skip positions without categorical columns
              const float t = __shfl_sync(0xffffffffu, xs[c], src_lane);
              if (cat_sel[s] == c) xc = t;
            }
          }
          int j = p.n_cat;  // row n_cat of s_wcat is all zeros: "no category matched" (or no column here)
          if (cat_n[s] <= KC) {  // categories cached in registers (NaN padding never matches)
#pragma unroll
            for (int q = KC - 1; q >= 0; --q) j = (xc == cat_c[s][q]) ? cat_base[s] + q : j;
          } else if (cat_lane[s] >= 0) {
            for (int q = 0; q < cat_n[s]; ++q)
              if (xc == s_catval[cat_base[s] + q]) j = cat_base[s] + q;  // de-duplicated: one match at most
          }
          const double* wc = s_wcat + (size_t)j * NS;
#pragma unroll
          for (int k = 0; k < NS; ++k) a[k] += wc[k];
        }
      }
#pragma unroll
      for (int k = 0; k < NS; ++k) v[i * NS + k] = a[k];
    }
    // ---- reduce-scatter butterfly over the L lanes of a row (fp64)
    {
      int n = V;
#pragma unroll
      for (int off = L / 2; off >= 1; off >>= 1) {
        if (n > 1) {
          const bool upper = (lir & off) != 0;
          const int hn = n / 2;
#pragma unroll
          for (int j = 0; j < V / 2; ++j) {
            if (j < hn) {
              const double keep = upper ? v[j + hn] : v[j];
              const double send = upper ? v[j] : v[j + hn];
              v[j] = keep + shfl_xor_d(send, off);
            }
          }
          n = hn;
        } else {
          v[0] += shfl_xor_d(v[0], off);
        }
      }
    }
    const int64_t my_row = base + own_i * RPW + half;
    double s = v[0] + my_bias;
    // a row is bad when any of its scores is non-finite; the NS score lanes of a row sit REP apart
    uint32_t my_bad = is_finite_d(s) ? 0u : 1u;
#pragma unroll
    for (int off = 1; off < NS; off <<= 1) my_bad |= __shfl_xor_sync(0xffffffffu, my_bad, off * REP);
    if (p.fast_epilogue) {
      // identity links, one score per model: VOTE_NONE writes every score, VOTE_MEAN sums w_k * s_k
      if (p.vote_kind == 1) {
        s *= my_vw;
        if (own_k >= p.n_models) s = 0.0;
#pragma unroll
        for (int off = 1; off < NS; off <<= 1) s += shfl_xor_d(s, off * REP);
        if (own_k == 0 && (lir % REP) == 0 && my_row < p.n_rows) {
          p.out[my_row] = (float)s;
          if (p.status) p.status[my_row] = (int32_t)my_bad;
        }
      } else {
        if ((lir % REP) == 0 && own_k < p.n_models && my_row < p.n_rows) {
          p.out[my_row * p.out_cols + own_k] = (float)s;
          if (p.status && own_k == 0) p.status[my_row] = (int32_t)my_bad;
        }
      }
    } else {
      // generic epilogue: collect the row's NS scores on its first lane, then links + vote there
      double sc[NS];
#pragma unroll
      for (int k = 0; k < NS; ++k) sc[k] = shfl_idx_d(s, half * L + (own_i * NS + k) * REP);
      if (own_k == 0 && (lir % REP) == 0 && my_row < p.n_rows) {
        double pred[kMaxModels];
        for (int m = 0; m < p.n_models; ++m) {
          const ModelDesc md = p.models[m];
          pred[m] = apply_link(md, sc + md.score_off, p.classes);
        }
        KParams kp;  // vote_and_store only reads these fields
        kp.out = p.out;
        kp.out_cols = p.out_cols;
        kp.n_models = p.n_models;
        kp.vote_kind = p.vote_kind;
        kp.out_is_int = p.out_is_int;
        kp.vote_w = p.vote_w;
        kp.status = p.status;
        kp.n_peers = 0;
        vote_and_store(kp, pred, my_row, my_bad);
      }
    }
  }
}

}  // namespace b2s
