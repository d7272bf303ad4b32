// DIN's activation unit applied as target attention over a behaviour sequence, and the Dice activation.
//   keras/models/ranking/din.py:59-71 (ActivationUnit.call) and :110-121 (Dice.call); the backward is TensorFlow
//   autodiff there.
//
// Attention unit, for example b, position t, k = keys[b,t,:], q = query[b,:]:
//   u      = [k | q | f(k, q)]          f: none, k - q or k * q
//   h      = act(u . W1 + b1)           W1 [(2|3)*D, U] = [Wk; Wq; Wi]
//   score  = h . w2 + b2
//   pooled = sum_t score[b,t] * k       (DIN's unnormalised weighted sum)
// A plain port materialises u ([B*T, 3D]) and h ([B*T, U]).  Here a CTA owns `epc` whole examples and walks their
// B*T rows in chunks of 64: the chunk's keys are staged in shared memory with the interaction block generated next to
// them, the q block q . Wq + b1 is computed once per example, and the score reduction over U and the pooling over t
// happen in the epilogue in a fixed order.  Neither u nor h reaches global memory.  The weight blocks are kept apart
// (no k.(Wk + Wi) fold): the rounding then stays bounded by the reference's own terms when k ~ q.
// The backward recomputes h per chunk and forms G = dscore * w2 * act'(h) in shared memory, then
//   g_u = G . W1^T (keys and the interaction block per row, the q block once per example from sum_t G),
//   gW1 += u^T G (per CTA in shared memory when it fits, else red.global.add per chunk).
// Arithmetic: fp32 FFMA.  Thread (ty, tx) of 16 x 16 owns rows ty*4 + i and columns tx + 16*j of the [64, 16*NU]
// tile; W1 is read through L1 (a row segment of 16 consecutive floats per half warp).
#include "common.cuh"

namespace dr {

namespace {

constexpr int DIN_THREADS = 256;
constexpr int DIN_R = 64;                       // rows (example, position) per chunk
constexpr int DIN_MAX_D = 128;
constexpr int DIN_MAX_U = 256;
constexpr int DIN_WT_KV = 64, DIN_WT_C = 32, DIN_WT_LD = DIN_WT_KV + 4;
constexpr int DIN_FWD_SMEM = 100 * 1024;        // two CTAs per SM
constexpr int DIN_BWD_SMEM = 200 * 1024;
constexpr int DIN_GW_SMEM = 110 * 1024;         // the backward keeps gW1 in shared memory below this total

struct DinArgs {
  const float* keys;      // [B, T, D]
  const float* query;     // [B, D]
  const float* w1;        // [(2|3)D, U]
  const float* b1;        // [U] or NULL
  const float* w2;        // [U]
  const float* b2;        // [1] or NULL
  const float* g_pooled;  // [B, D] or NULL
  const float* g_score;   // [B, T] or NULL
  float* score;           // [B, T] or NULL
  float* pooled;          // [B, D] or NULL
  float* g_keys;
  float* g_query;
  float* gw1;
  float* gb1;
  float* gw2;
  float* gb2;
  int64_t B;
  int T, D, U, Dp, Kvp, lda, interact, act, epc, gw_smem;
};

// shared-memory carve-up (in floats), the same arithmetic on the host (size) and the device (offsets)
struct DinLayout {
  int as, ex, sc, ds, qw, acc, gu, gs, wt, gps, gws, total;
};

__host__ __device__ inline DinLayout din_layout(int Kvp, int lda, int UP, int epc, int D, bool bwd, bool gw_smem) {
  DinLayout L{};
  int o = 0;
  L.as = o; o += DIN_R * lda;
  L.ex = o; o += DIN_R;
  L.sc = o; o += DIN_R;
  L.ds = o; o += DIN_R;
  L.qw = o; o += epc * UP;
  L.acc = o; o += epc * D;
  if (bwd) {
    L.gu = o; o += DIN_R * (Kvp + 1);
    L.gs = o; o += DIN_R * (UP + 1);
    L.wt = o; o += DIN_WT_C * DIN_WT_LD;
    L.gps = o; o += epc * UP;
    L.gws = o; if (gw_smem) o += Kvp * UP;
  }
  L.total = (o + 3) & ~3;
  return L;
}

// q . Wq + b1 for the CTA's examples: qw[e][c], zero for the padding columns c >= U.
__device__ __forceinline__ void din_q_block(const DinArgs& g, int UP, int64_t b0, int nex, float* qw) {
  for (int i = threadIdx.x; i < nex * UP; i += DIN_THREADS) {
    const int e = i / UP, c = i - e * UP;
    float s = 0.f;
    if (c < g.U) {
      const float* q = g.query + (b0 + e) * g.D;
      const float* w = g.w1 + (int64_t)g.D * g.U + c;
      for (int d = 0; d < g.D; ++d) s = fmaf(__ldg(q + d), __ldg(w + (int64_t)d * g.U), s);
      if (g.b1) s += __ldg(g.b1 + c);
    }
    qw[i] = s;
  }
}

// Stage the chunk: ex[r] = example of row r (-1 past the end), As[r] = [k | pad | f(k, q) | pad].
__device__ __forceinline__ void din_stage(const DinArgs& g, float* As, int* ex, int64_t n0, int nrows, int64_t b0) {
  const int t = threadIdx.x;
  if (t < DIN_R) ex[t] = t < nrows ? ((int)(n0 - b0 * g.T) + t) / g.T : -1;   // the CTA's rows fit in an int
  __syncthreads();
  const float* kp = g.keys + n0 * g.D;
  const int valid = nrows * g.D;
  for (int i = t; i < DIN_R * g.D; i += DIN_THREADS) {
    const int r = i / g.D, d = i - r * g.D;
    float k = 0.f, f = 0.f;
    if (i < valid) {
      k = __ldg(kp + i);
      if (g.interact != DR_DIN_INTERACT_NONE) {
        const float q = __ldg(g.query + (b0 + ex[r]) * g.D + d);
        f = g.interact == DR_DIN_INTERACT_SUB ? k - q : k * q;
      }
    }
    As[r * g.lda + d] = k;
    if (g.interact != DR_DIN_INTERACT_NONE) As[r * g.lda + g.Dp + d] = f;
  }
  __syncthreads();
}

// acc[i][j] = sum over the k and interaction blocks of As[row_i] . W1[:, col_j]  (the q block is added separately).
template <int NU>
__device__ __forceinline__ void din_unit_gemm(const DinArgs& g, const float* As, float (&acc)[4][NU], int ty, int tx) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < NU; ++j) acc[i][j] = 0.f;
  int cl[NU];
#pragma unroll
  for (int j = 0; j < NU; ++j) cl[j] = min(tx + 16 * j, g.U - 1);   // padding columns are discarded later
  const int nblk = g.interact != DR_DIN_INTERACT_NONE ? 2 : 1;
  for (int blk = 0; blk < nblk; ++blk) {
    const float* W = g.w1 + (int64_t)(blk ? 2 * g.D : 0) * g.U;
    const float* A = As + ty * 4 * g.lda + blk * g.Dp;
    for (int d0 = 0; d0 < g.Dp; d0 += 4) {
      float4 a[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const float4*>(A + i * g.lda + d0);
#pragma unroll
      for (int dd = 0; dd < 4; ++dd) {
        const float* wr = W + (int64_t)min(d0 + dd, g.D - 1) * g.U;   // As is zero past D
        float w[NU];
#pragma unroll
        for (int j = 0; j < NU; ++j) w[j] = __ldg(wr + cl[j]);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float av = dd == 0 ? a[i].x : dd == 1 ? a[i].y : dd == 2 ? a[i].z : a[i].w;
#pragma unroll
          for (int j = 0; j < NU; ++j) acc[i][j] = fmaf(av, w[j], acc[i][j]);
        }
      }
    }
  }
}

// h = act(acc + qw) in place; returns the row's score partial over this thread's columns, summed over the 16 column
// groups of the row (a fixed butterfly).
template <int NU>
__device__ __forceinline__ void din_hidden(const DinArgs& g, int UP, const int* ex, const float* qw,
                                           const float (&w2r)[NU], float (&acc)[4][NU], float (&part)[4], int ty,
                                           int tx) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int e = ex[ty * 4 + i];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < NU; ++j) {
      const float v = act_apply(acc[i][j] + (e >= 0 ? qw[e * UP + tx + 16 * j] : 0.f), g.act);
      acc[i][j] = v;
      s = fmaf(v, w2r[j], s);
    }
    part[i] = group_sum<16>(s);
  }
}

// rows [r0, r1) of the chunk that belong to example e of the CTA
__device__ __forceinline__ void din_rows_of(const DinArgs& g, int64_t b0, int e, int64_t n0, int nrows, int& r0,
                                            int& r1) {
  const int64_t eb = (b0 + e) * g.T;
  r0 = (int)max((int64_t)0, eb - n0);
  r1 = (int)min((int64_t)nrows, eb + g.T - n0);
}

}  // namespace

// grid = ceil(B / epc); one CTA owns examples [b0, b0 + epc).
template <int NU>
__global__ void __launch_bounds__(DIN_THREADS) din_attn_fwd_kernel(const DinArgs g) {
  constexpr int UP = 16 * NU;
  extern __shared__ __align__(16) float sm[];
  const DinLayout L = din_layout(g.Kvp, g.lda, UP, g.epc, g.D, false, false);
  float* As = sm + L.as;
  int* ex = reinterpret_cast<int*>(sm + L.ex);
  float* sc = sm + L.sc;
  float* qw = sm + L.qw;
  float* pacc = sm + L.acc;
  const int t = threadIdx.x, ty = t >> 4, tx = t & 15;
  const int64_t b0 = (int64_t)blockIdx.x * g.epc;
  const int nex = (int)min((int64_t)g.epc, g.B - b0);
  const int64_t n_end = (b0 + nex) * g.T;

  for (int i = t; i < DIN_R * g.lda; i += DIN_THREADS) As[i] = 0.f;   // the padding columns stay zero
  for (int i = t; i < nex * g.D; i += DIN_THREADS) pacc[i] = 0.f;
  din_q_block(g, UP, b0, nex, qw);
  float w2r[NU];
#pragma unroll
  for (int j = 0; j < NU; ++j) w2r[j] = tx + 16 * j < g.U ? __ldg(g.w2 + tx + 16 * j) : 0.f;
  const float b2v = g.b2 ? __ldg(g.b2) : 0.f;

  for (int64_t n0 = b0 * g.T; n0 < n_end; n0 += DIN_R) {
    const int nrows = (int)min((int64_t)DIN_R, n_end - n0);
    din_stage(g, As, ex, n0, nrows, b0);
    float acc[4][NU], part[4];
    din_unit_gemm<NU>(g, As, acc, ty, tx);
    din_hidden<NU>(g, UP, ex, qw, w2r, acc, part, ty, tx);
    if (tx == 0) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = ty * 4 + i;
        if (row < nrows) {
          const float v = part[i] + b2v;
          sc[row] = v;
          if (g.score) g.score[n0 + row] = v;
        }
      }
    }
    __syncthreads();
    if (g.pooled) {
      for (int i = t; i < nex * g.D; i += DIN_THREADS) {
        const int e = i / g.D, d = i - e * g.D;
        int r0, r1;
        din_rows_of(g, b0, e, n0, nrows, r0, r1);
        float s = 0.f;
        for (int r = r0; r < r1; ++r) s = fmaf(sc[r], As[r * g.lda + d], s);
        pacc[i] += s;
      }
    }
    __syncthreads();
  }
  if (g.pooled)
    for (int i = t; i < nex * g.D; i += DIN_THREADS) g.pooled[b0 * g.D + i] = pacc[i];
}

template <int NU>
__global__ void __launch_bounds__(DIN_THREADS, 1) din_attn_bwd_kernel(const DinArgs g) {
  constexpr int UP = 16 * NU;
  constexpr int LDG = UP + 1;
  extern __shared__ __align__(16) float sm[];
  const DinLayout L = din_layout(g.Kvp, g.lda, UP, g.epc, g.D, true, g.gw_smem);
  float* As = sm + L.as;
  int* ex = reinterpret_cast<int*>(sm + L.ex);
  float* sc = sm + L.sc;
  float* ds = sm + L.ds;
  float* qw = sm + L.qw;
  float* gqa = sm + L.acc;
  float* GU = sm + L.gu;
  float* Gs = sm + L.gs;
  float* Wt = sm + L.wt;
  float* gps = sm + L.gps;
  float* gws = g.gw_smem ? sm + L.gws : nullptr;
  const int t = threadIdx.x, ty = t >> 4, tx = t & 15, warp = t >> 5, lane = t & 31;
  const int64_t b0 = (int64_t)blockIdx.x * g.epc;
  const int nex = (int)min((int64_t)g.epc, g.B - b0);
  const int64_t n_end = (b0 + nex) * g.T;
  const int ldu = g.Kvp + 1;
  const bool inter = g.interact != DR_DIN_INTERACT_NONE;
  const bool sub = g.interact == DR_DIN_INTERACT_SUB;

  for (int i = t; i < DIN_R * g.lda; i += DIN_THREADS) As[i] = 0.f;
  for (int i = t; i < nex * g.D; i += DIN_THREADS) gqa[i] = 0.f;
  for (int i = t; i < nex * UP; i += DIN_THREADS) gps[i] = 0.f;
  if (gws)
    for (int i = t; i < g.Kvp * UP; i += DIN_THREADS) gws[i] = 0.f;
  din_q_block(g, UP, b0, nex, qw);
  float w2r[NU], gw2a[NU], gb1a[NU];
#pragma unroll
  for (int j = 0; j < NU; ++j) {
    w2r[j] = tx + 16 * j < g.U ? __ldg(g.w2 + tx + 16 * j) : 0.f;
    gw2a[j] = 0.f;
    gb1a[j] = 0.f;
  }
  float gb2a = 0.f;
  const float b2v = g.b2 ? __ldg(g.b2) : 0.f;

  for (int64_t n0 = b0 * g.T; n0 < n_end; n0 += DIN_R) {
    const int nrows = (int)min((int64_t)DIN_R, n_end - n0);
    din_stage(g, As, ex, n0, nrows, b0);
    // dscore = g_score + g_pooled . k  (one warp per row, fixed butterfly)
    for (int r = warp; r < DIN_R; r += DIN_THREADS / 32) {
      float s = 0.f;
      if (r < nrows && g.g_pooled) {
        const float* gp = g.g_pooled + (b0 + ex[r]) * g.D;
        for (int d = lane; d < g.D; d += 32) s = fmaf(__ldg(gp + d), As[r * g.lda + d], s);
      }
      s = group_sum<32>(s);
      if (lane == 0) ds[r] = r < nrows ? s + (g.g_score ? __ldg(g.g_score + n0 + r) : 0.f) : 0.f;
    }
    __syncthreads();
    // recompute h and the score, then G = dscore * w2 * act'(h)
    {
      float acc[4][NU], part[4];
      din_unit_gemm<NU>(g, As, acc, ty, tx);
      din_hidden<NU>(g, UP, ex, qw, w2r, acc, part, ty, tx);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = ty * 4 + i;
        const float dsr = ds[row];
        if (tx == 0) {
          sc[row] = part[i] + b2v;
          gb2a += dsr;
        }
#pragma unroll
        for (int j = 0; j < NU; ++j) {
          const float h = acc[i][j];
          const float gz = dsr * w2r[j] * act_grad_from_y(h, g.act);
          Gs[row * LDG + tx + 16 * j] = gz;
          gw2a[j] = fmaf(dsr, h, gw2a[j]);
          gb1a[j] += gz;
        }
      }
    }
    __syncthreads();
    // per-example sums of G (the q block's gradient is formed from them once per example)
    for (int i = t; i < nex * UP; i += DIN_THREADS) {
      const int e = i / UP, c = i - e * UP;
      int r0, r1;
      din_rows_of(g, b0, e, n0, nrows, r0, r1);
      float s = 0.f;
      for (int r = r0; r < r1; ++r) s += Gs[r * LDG + c];
      gps[i] += s;
    }
    // GU[r][kv] = sum_c G[r][c] * W1v[kv][c] over the k and interaction blocks, 64 kv x 32 c staged at a time
    for (int kv0 = 0; kv0 < g.Kvp; kv0 += DIN_WT_KV) {
      float a2[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) a2[i][j] = 0.f;
      for (int c0 = 0; c0 < UP; c0 += DIN_WT_C) {
        __syncthreads();
        for (int i = t; i < DIN_WT_KV * DIN_WT_C; i += DIN_THREADS) {
          const int kvl = i / DIN_WT_C, cc = i - kvl * DIN_WT_C;
          const int kv = kv0 + kvl, c = c0 + cc;
          const int blk = kv >= g.Dp, d = kv - blk * g.Dp;
          float v = 0.f;
          if (kv < g.Kvp && d < g.D && c < g.U) v = __ldg(g.w1 + (int64_t)(blk ? 2 * g.D + d : d) * g.U + c);
          Wt[cc * DIN_WT_LD + kvl] = v;
        }
        __syncthreads();
        const int ccn = min(DIN_WT_C, UP - c0);
#pragma unroll 4
        for (int cc = 0; cc < ccn; ++cc) {
          float a[4], w[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) a[i] = Gs[(ty * 4 + i) * LDG + c0 + cc];
#pragma unroll
          for (int j = 0; j < 4; ++j) w[j] = Wt[cc * DIN_WT_LD + tx + 16 * j];
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) a2[i][j] = fmaf(a[i], w[j], a2[i][j]);
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int kv = kv0 + tx + 16 * j;
          if (kv < g.Kvp) GU[(ty * 4 + i) * ldu + kv] = a2[i][j];
        }
    }
    // gW1 (k and interaction blocks) += u^T G, 64 kv rows per pass
    for (int kv0 = 0; kv0 < g.Kvp; kv0 += 64) {
      float a3[4][NU];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < NU; ++j) a3[i][j] = 0.f;
      int kvc[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) kvc[i] = min(kv0 + ty + 16 * i, g.Kvp - 1);
      for (int r = 0; r < nrows; ++r) {
        float a[4], gg[NU];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = As[r * g.lda + kvc[i]];
#pragma unroll
        for (int j = 0; j < NU; ++j) gg[j] = Gs[r * LDG + tx + 16 * j];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < NU; ++j) a3[i][j] = fmaf(a[i], gg[j], a3[i][j]);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int kv = kv0 + ty + 16 * i;
        const int blk = kv >= g.Dp, d = kv - blk * g.Dp;
        if (kv >= g.Kvp || d >= g.D) continue;
        const int wrow = blk ? 2 * g.D + d : d;
#pragma unroll
        for (int j = 0; j < NU; ++j) {
          const int c = tx + 16 * j;
          if (c >= g.U) continue;
          if (gws) gws[kv * UP + c] += a3[i][j];
          else red_add_f32(g.gw1 + (int64_t)wrow * g.U + c, a3[i][j]);
        }
      }
    }
    __syncthreads();
    // g_keys = GU_k + GU_i * df/dk + score * g_pooled  (overwritten, one owner per element)
    for (int i = t; i < nrows * g.D; i += DIN_THREADS) {
      const int r = i / g.D, d = i - r * g.D;
      const int64_t b = b0 + ex[r];
      float v = GU[r * ldu + d];
      if (inter) {
        const float gi = GU[r * ldu + g.Dp + d];
        v += sub ? gi : gi * __ldg(g.query + b * g.D + d);
      }
      if (g.g_pooled) v = fmaf(sc[r], __ldg(g.g_pooled + b * g.D + d), v);
      g.g_keys[(n0 + r) * g.D + d] = v;
    }
    // the interaction block's share of g_query: sum over the example's rows of GU_i * df/dq
    if (inter) {
      for (int i = t; i < nex * g.D; i += DIN_THREADS) {
        const int e = i / g.D, d = i - e * g.D;
        int r0, r1;
        din_rows_of(g, b0, e, n0, nrows, r0, r1);
        float s = 0.f;
        for (int r = r0; r < r1; ++r) {
          const float gi = GU[r * ldu + g.Dp + d];
          s = sub ? s - gi : fmaf(gi, As[r * g.lda + d], s);
        }
        gqa[i] += s;
      }
    }
    __syncthreads();
  }

  // g_query = (interaction share) + (sum_t G) . Wq^T
  for (int i = t; i < nex * g.D; i += DIN_THREADS) {
    const int e = i / g.D, d = i - e * g.D;
    const float* wq = g.w1 + (int64_t)(g.D + d) * g.U;
    float s = 0.f;
    for (int c = 0; c < g.U; ++c) s = fmaf(gps[e * UP + c], __ldg(wq + c), s);
    g.g_query[b0 * g.D + i] = s + gqa[i];
  }
  // gWq[d][c] = sum over the CTA's examples of q[b][d] * sum_t G[b,t][c]
  for (int i = t; i < g.D * g.U; i += DIN_THREADS) {
    const int d = i / g.U, c = i - d * g.U;
    float s = 0.f;
    for (int e = 0; e < nex; ++e) s = fmaf(__ldg(g.query + (b0 + e) * g.D + d), gps[e * UP + c], s);
    red_add_f32(g.gw1 + (int64_t)(g.D + d) * g.U + c, s);
  }
  if (gws) {
    for (int i = t; i < g.Kvp * UP; i += DIN_THREADS) {
      const int kv = i / UP, c = i - kv * UP;
      const int blk = kv >= g.Dp, d = kv - blk * g.Dp;
      if (d < g.D && c < g.U) red_add_f32(g.gw1 + (int64_t)(blk ? 2 * g.D + d : d) * g.U + c, gws[i]);
    }
  }
  // gw2, gb1, gb2: the 16 row groups summed in order through shared memory (Gs is free now)
  float* red = Gs;
#pragma unroll
  for (int j = 0; j < NU; ++j) {
    red[ty * UP + tx + 16 * j] = gw2a[j];
    red[16 * UP + ty * UP + tx + 16 * j] = gb1a[j];
  }
  if (tx == 0) red[32 * UP + ty] = gb2a;
  __syncthreads();
  for (int c = t; c < g.U; c += DIN_THREADS) {
    float s2 = 0.f, s1 = 0.f;
    for (int y = 0; y < 16; ++y) {
      s2 += red[y * UP + c];
      s1 += red[16 * UP + y * UP + c];
    }
    red_add_f32(g.gw2 + c, s2);
    if (g.gb1) red_add_f32(g.gb1 + c, s1);
  }
  if (t == 0 && g.gb2) {
    float s = 0.f;
    for (int y = 0; y < 16; ++y) s += red[32 * UP + y];
    red_add_f32(g.gb2, s);
  }
}

// ---- Dice ----------------------------------------------------------------------------------------------------------
// Per row of x [N, U]: mu = mean, sigma = population std, p = sigmoid((x - mu) / sqrt(sigma + eps)) (the square root of
// the std, as the reference computes it), a = PReLU(x) with alpha [U], y = a > 0 ? p*a : (1 - p)*a.
// One warp per row.

struct DiceRow {
  float mu, sigma, den;
};

__device__ __forceinline__ DiceRow dice_row_stats(const float* xr, int U, float eps, int lane) {
  float s = 0.f;
  for (int c = lane; c < U; c += 32) s += __ldg(xr + c);
  const float mu = group_sum<32>(s) / (float)U;
  float v = 0.f;
  for (int c = lane; c < U; c += 32) {
    const float dlt = __ldg(xr + c) - mu;
    v = fmaf(dlt, dlt, v);
  }
  const float sigma = sqrtf(group_sum<32>(v) / (float)U);
  return DiceRow{mu, sigma, sqrtf(sigma + eps)};
}

__global__ void __launch_bounds__(256) dice_fwd_kernel(const float* __restrict__ x, const float* __restrict__ alpha,
                                                       int64_t N, int U, float eps, float* __restrict__ y) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < N; r += nwarps) {
    const float* xr = x + r * U;
    const DiceRow st = dice_row_stats(xr, U, eps, lane);
    for (int c = lane; c < U; c += 32) {
      const float xv = __ldg(xr + c);
      const float p = 1.f / (1.f + expf(-((xv - st.mu) / st.den)));
      const float a = xv > 0.f ? xv : __ldg(alpha + c) * xv;
      y[r * U + c] = a > 0.f ? p * a : (1.f - p) * a;
    }
  }
}

// gx through PReLU, p, mu and sigma; galpha[c] = column sums (per-CTA shared-memory sums, then red.global.add).
// A constant row (sigma = 0) gets no gradient through sigma (TensorFlow's autodiff gives NaN there).
__global__ void __launch_bounds__(256) dice_bwd_kernel(const float* __restrict__ x, const float* __restrict__ alpha,
                                                       const float* __restrict__ gy, int64_t N, int U, float eps,
                                                       float* __restrict__ gx, float* __restrict__ galpha) {
  extern __shared__ float s_ga[];
  for (int c = threadIdx.x; c < U; c += blockDim.x) s_ga[c] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < N; r += nwarps) {
    const float* xr = x + r * U;
    const float* gr = gy + r * U;
    const DiceRow st = dice_row_stats(xr, U, eps, lane);
    float s1 = 0.f, s2 = 0.f;   // sum gz, sum gz * (x - mu), gz = dL/dz with z = (x - mu) / den
    for (int c = lane; c < U; c += 32) {
      const float xv = __ldg(xr + c), g = __ldg(gr + c);
      const float p = 1.f / (1.f + expf(-((xv - st.mu) / st.den)));
      const float a = xv > 0.f ? xv : __ldg(alpha + c) * xv;
      const float gz = g * (a > 0.f ? a : -a) * p * (1.f - p);
      s1 += gz;
      s2 = fmaf(gz, xv - st.mu, s2);
    }
    s1 = group_sum<32>(s1);
    s2 = group_sum<32>(s2);
    // d den / dx_j = (x_j - mu) / (2 den U sigma);  dL/d den = -s2 / den^2
    const float coef = st.sigma > 0.f ? (-s2 / (st.den * st.den)) / (2.f * st.den * (float)U * st.sigma) : 0.f;
    const float mean_term = s1 / st.den / (float)U;
    for (int c = lane; c < U; c += 32) {
      const float xv = __ldg(xr + c), g = __ldg(gr + c), al = __ldg(alpha + c);
      const float p = 1.f / (1.f + expf(-((xv - st.mu) / st.den)));
      const float a = xv > 0.f ? xv : al * xv;
      const float ga = g * (a > 0.f ? p : 1.f - p);
      const float gz = g * (a > 0.f ? a : -a) * p * (1.f - p);
      const float da = xv > 0.f ? 1.f : (xv < 0.f ? al : 0.f);
      gx[r * U + c] = ga * da + gz / st.den - mean_term + coef * (xv - st.mu);
      if (xv < 0.f) atomicAdd(&s_ga[c], ga * xv);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < U; c += blockDim.x) red_add_f32(galpha + c, s_ga[c]);
}

// ---- host ----------------------------------------------------------------------------------------------------------
static int din_pick_nu(int U) {
  const int need = (U + 15) / 16;
  static const int nus[] = {1, 2, 3, 4, 6, 8, 12, 16};
  for (int v : nus)
    if (v >= need) return v;
  return 16;
}

template <int NU>
static int din_launch(const DinArgs& a, bool bwd, int smem, cudaStream_t st) {
  const unsigned grid = (unsigned)((a.B + a.epc - 1) / a.epc);
  if (bwd) {
    DR_CUDA_CALL(cudaFuncSetAttribute(din_attn_bwd_kernel<NU>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    din_attn_bwd_kernel<NU><<<grid, DIN_THREADS, smem, st>>>(a);
    DR_CUDA_LAUNCH_CHECK("din_attn_bwd");
  } else {
    DR_CUDA_CALL(cudaFuncSetAttribute(din_attn_fwd_kernel<NU>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    din_attn_fwd_kernel<NU><<<grid, DIN_THREADS, smem, st>>>(a);
    DR_CUDA_LAUNCH_CHECK("din_attn_fwd");
  }
  return DR_OK;
}

static int din_check(const char* who, int64_t B, int T, int D, int U, int interact, int act) {
  DR_REQUIRE(B >= 0 && T >= 1 && D >= 1 && U >= 1, DR_EINVAL, "%s: bad shape B=%lld T=%d D=%d U=%d", who,
             (long long)B, T, D, U);
  DR_REQUIRE(interact >= DR_DIN_INTERACT_NONE && interact <= DR_DIN_INTERACT_MUL, DR_EINVAL,
             "%s: unknown interaction %d", who, interact);
  DR_REQUIRE(act >= DR_ACT_NONE && act <= DR_ACT_TANH, DR_EINVAL, "%s: unknown activation %d", who, act);
  DR_REQUIRE(D <= DIN_MAX_D && U <= DIN_MAX_U, DR_ENOTSUP, "%s: D=%d U=%d above the served caps (D <= %d, U <= %d)",
             who, D, U, DIN_MAX_D, DIN_MAX_U);
  DR_REQUIRE(B * (int64_t)T < (int64_t)1 << 31, DR_ENOTSUP, "%s: B*T = %lld rows above the served cap 2^31", who,
             (long long)(B * (int64_t)T));
  return DR_OK;
}

// Fills the shape fields, picks examples per CTA (~512 rows per CTA, at most 64 examples) within the shared-memory
// budget; returns the dynamic shared-memory size in bytes.
static int din_plan(DinArgs& a, bool bwd) {
  const int UP = 16 * din_pick_nu(a.U);
  a.Dp = (a.D + 3) & ~3;
  a.Kvp = a.interact != DR_DIN_INTERACT_NONE ? 2 * a.Dp : a.Dp;
  a.lda = a.Kvp + 4;
  int epc = (512 + a.T - 1) / a.T;
  if (epc > 64) epc = 64;
  const int budget = bwd ? DIN_BWD_SMEM : DIN_FWD_SMEM;
  auto bytes = [&](int e, bool gws) {
    return 4 * din_layout(a.Kvp, a.lda, UP, e, a.D, bwd, gws).total;
  };
  while (epc > 1 && bytes(epc, false) > budget) epc = (epc + 1) / 2;
  a.epc = epc;
  a.gw_smem = bwd && bytes(epc, true) <= DIN_GW_SMEM;
  return bytes(epc, a.gw_smem);
}

static int din_dispatch(const DinArgs& a, bool bwd, int smem, cudaStream_t st) {
  switch (din_pick_nu(a.U)) {
    case 1: return din_launch<1>(a, bwd, smem, st);
    case 2: return din_launch<2>(a, bwd, smem, st);
    case 3: return din_launch<3>(a, bwd, smem, st);
    case 4: return din_launch<4>(a, bwd, smem, st);
    case 6: return din_launch<6>(a, bwd, smem, st);
    case 8: return din_launch<8>(a, bwd, smem, st);
    case 12: return din_launch<12>(a, bwd, smem, st);
    default: return din_launch<16>(a, bwd, smem, st);
  }
}

}  // namespace dr

using namespace dr;

extern "C" int dr_din_attn_fwd(const float* keys, const float* query, const float* w1, const float* b1,
                               const float* w2, const float* b2, int64_t B, int T, int D, int U, int interact, int act,
                               float* score, float* pooled, void* stream) {
  DR_REQUIRE(w1 && w2 && (B == 0 || (keys && query && (score || pooled))), DR_EINVAL, "dr_din_attn_fwd: null pointer");
  if (int rc = din_check("dr_din_attn_fwd", B, T, D, U, interact, act)) return rc;
  if (B == 0) return DR_OK;
  DinArgs a{};
  a.keys = keys; a.query = query; a.w1 = w1; a.b1 = b1; a.w2 = w2; a.b2 = b2;
  a.score = score; a.pooled = pooled;
  a.B = B; a.T = T; a.D = D; a.U = U; a.interact = interact; a.act = act;
  const int smem = din_plan(a, false);
  return din_dispatch(a, false, smem, (cudaStream_t)stream);
}

extern "C" int dr_din_attn_bwd(const float* keys, const float* query, const float* w1, const float* b1,
                               const float* w2, const float* b2, const float* g_pooled, const float* g_score,
                               int64_t B, int T, int D, int U, int interact, int act, float* g_keys, float* g_query,
                               float* gw1, float* gb1, float* gw2, float* gb2, void* stream) {
  DR_REQUIRE(w1 && w2 && gw1 && gw2 && (B == 0 || (keys && query && g_keys && g_query)), DR_EINVAL,
             "dr_din_attn_bwd: null pointer");
  DR_REQUIRE(B == 0 || g_pooled || g_score, DR_EINVAL, "dr_din_attn_bwd: g_pooled and g_score are both NULL");
  DR_REQUIRE((b1 == nullptr) == (gb1 == nullptr) && (b2 == nullptr) == (gb2 == nullptr), DR_EINVAL,
             "dr_din_attn_bwd: a bias gradient must be given exactly when its bias is");
  if (int rc = din_check("dr_din_attn_bwd", B, T, D, U, interact, act)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int rows1 = (interact != DR_DIN_INTERACT_NONE ? 3 : 2) * D;
  DR_CUDA_CALL(cudaMemsetAsync(gw1, 0, sizeof(float) * (size_t)rows1 * U, st));
  DR_CUDA_CALL(cudaMemsetAsync(gw2, 0, sizeof(float) * U, st));
  if (gb1) DR_CUDA_CALL(cudaMemsetAsync(gb1, 0, sizeof(float) * U, st));
  if (gb2) DR_CUDA_CALL(cudaMemsetAsync(gb2, 0, sizeof(float), st));
  if (B == 0) return DR_OK;
  DinArgs a{};
  a.keys = keys; a.query = query; a.w1 = w1; a.b1 = b1; a.w2 = w2; a.b2 = b2;
  a.g_pooled = g_pooled; a.g_score = g_score;
  a.g_keys = g_keys; a.g_query = g_query; a.gw1 = gw1; a.gb1 = gb1; a.gw2 = gw2; a.gb2 = gb2;
  a.B = B; a.T = T; a.D = D; a.U = U; a.interact = interact; a.act = act;
  const int smem = din_plan(a, true);
  return din_dispatch(a, true, smem, st);
}

extern "C" int dr_dice_fwd(const float* x, const float* alpha, int64_t N, int U, float eps, float* y, void* stream) {
  DR_REQUIRE(alpha && (N == 0 || (x && y)), DR_EINVAL, "dr_dice_fwd: null pointer");
  DR_REQUIRE(N >= 0 && U >= 1, DR_EINVAL, "dr_dice_fwd: bad shape N=%lld U=%d", (long long)N, U);
  if (N == 0) return DR_OK;
  int64_t ctas = (N + 7) / 8;
  if (ctas > (int64_t)num_sms() * 16) ctas = (int64_t)num_sms() * 16;
  dice_fwd_kernel<<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(x, alpha, N, U, eps, y);
  DR_CUDA_LAUNCH_CHECK("dice_fwd");
  return DR_OK;
}

extern "C" int dr_dice_bwd(const float* x, const float* alpha, const float* gy, int64_t N, int U, float eps,
                           float* gx, float* galpha, void* stream) {
  DR_REQUIRE(alpha && galpha && (N == 0 || (x && gy && gx)), DR_EINVAL, "dr_dice_bwd: null pointer");
  DR_REQUIRE(N >= 0 && U >= 1, DR_EINVAL, "dr_dice_bwd: bad shape N=%lld U=%d", (long long)N, U);
  DR_REQUIRE(U <= 8192, DR_ENOTSUP, "dr_dice_bwd: U=%d above the served cap 8192", U);
  cudaStream_t st = (cudaStream_t)stream;
  DR_CUDA_CALL(cudaMemsetAsync(galpha, 0, sizeof(float) * U, st));
  if (N == 0) return DR_OK;
  int64_t ctas = (N + 7) / 8;
  if (ctas > (int64_t)num_sms() * 8) ctas = (int64_t)num_sms() * 8;
  dice_bwd_kernel<<<(unsigned)ctas, 256, sizeof(float) * U, st>>>(x, alpha, gy, N, U, eps, gx, galpha);
  DR_CUDA_LAUNCH_CHECK("dice_bwd");
  return DR_OK;
}
