// Scaled dot-product attention with MultiHeadAttention's head split and merge folded into strides, LayerNorm of a
// residual sum, and a row softmax.
//   keras/models/nlp/multi_head_attention.py:45-58 (mask, future_mask), :72-84 (ScaledDotProductAttention.call),
//   :134-147 (head split / merge); keras/models/nlp/transformer.py:109-113 (LayerNormalization.call), :264-265 (the
//   decoder's softmax).  The backward is TensorFlow autodiff there.
//
// Attention, logical row r = h*B + b (the reference's head-major concat), query i, key j:
//   s_ij = (q_i . k_j) / fl32(sqrt(dh))
//   s_ij = s_ij + mask[r % Bm, j] * C         C = fl32(-2^32 + 1) = -4294967296.0f, added (not -inf)
//   s_ij = C where j > i                      (causal: replaced, as tf.where does)
//   p    = softmax_j(s),  out_i = sum_j drop(p_ij) v_j
// FlashAttention-2 form: a CTA owns 64 query rows of one r and streams the keys through shared memory in tiles of 64
// with an online softmax; only the per-row log-sum-exp is saved.  It is saved in float64: a row whose keys are all
// padding has every score equal to C, so its log-sum-exp is C + log(Lk), which fp32 (ulp 512 at 2^32) cannot hold.
// The backward splits it once per row into hi = fl32(lse) and lo = fl32(lse - hi) and takes p = exp((s - hi) - lo)
// in fp32.
// Backward: D_i = rowsum(dO * O); ds = p * (dp - D_i), zero where the causal rule replaced the score.  dK / dV come
// from a CTA that owns 64 keys and loops over every query; dQ from a CTA that owns 64 queries and loops over every key.
// Each output element has one owner, so reruns are bit-identical.  No tile is skipped under the causal rule: a query
// whose keys 0..i are all padding has uniform weights over all Lk keys, future ones included.
// Arithmetic: fp32 FFMA.  A row (query or key) belongs to a group of G adjacent lanes; lane g of the group holds head
// columns [g*DT, (g+1)*DT), and dot products are summed over the group with a fixed butterfly.
#include "common.cuh"

#include <math.h>

namespace dr {

namespace {

constexpr float ATT_NEG = -4294967296.0f;   // fl32(-2**32 + 1)
constexpr int ATT_ROWS = 64;                // rows a CTA owns (one lane group each)
constexpr int ATT_TILE = 64;                // rows staged per pass
constexpr int ATT_CHUNK = 8;                // keys per online-softmax rescale in the forward
constexpr int ATT_MAX_DH = 128;

struct AttArgs {
  const float* q;      // [B, Lq, H*dh]
  const float* k;      // [B, Lk, H*dh]
  const float* v;      // [B, Lk, H*dh]
  const float* mask;   // [Bm, Lk] or NULL
  const float* out;    // [B, Lq, H*dh] (backward)
  const double* lse_in;
  const float* g_out;
  float* o;
  double* lse;         // [H*B, Lq]
  float* gq;
  float* gk;
  float* gv;
  int64_t B, Bm;
  int H, Lq, Lk, dh, ntiles, causal, drop;
  uint32_t thr;        // keep iff hash >> 40 >= thr
  float div;           // fl32(sqrt(dh))
  float rdiv;          // fl32(1 / div): the backward scales ds by it (within an ulp of ds / div)
  float keep_scale;    // fl32(1 / (1 - rate))
  uint64_t seed;
};

__device__ __forceinline__ bool att_keep(const AttArgs& a, int64_t r, int i, int j) {
  const uint64_t ctr = ((uint64_t)r * (uint64_t)a.Lq + (uint64_t)i) * (uint64_t)a.Lk + (uint64_t)j;
  uint64_t z = a.seed + (ctr + 1ull) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (uint32_t)(z >> 40) >= a.thr;
}

// The score after the scale, the padding mask and the causal rule (tf ops in the reference's order, no contraction).
__device__ __forceinline__ float att_score(const AttArgs& a, float dot, float mval, int i, int j, bool& replaced) {
  float s = dot / a.div;
  if (a.mask) s = __fadd_rn(s, __fmul_rn(mval, ATT_NEG));
  replaced = a.causal && j > i;
  return replaced ? ATT_NEG : s;
}

// Stage rows [j0, j0 + ATT_TILE) of one head of a [B, L, H*dh] tensor; element (row, d) goes to
// row * LD + (d / DT) * (DT + 4) + d % DT (the +4 keeps the G slices of one row on distinct banks).  Zero past L / dh.
template <int DT, int G>
__device__ __forceinline__ void att_stage(const float* src, int64_t b, int h, int L, int dh, int H, int j0,
                                          float* dst) {
  constexpr int DHP = DT * G, SL = DT + 4, LD = G * SL;
  const int64_t HD = (int64_t)H * dh;
  for (int e = threadIdx.x; e < ATT_TILE * DHP; e += blockDim.x) {
    const int row = e / DHP, d = e - row * DHP;
    const int j = j0 + row;
    float x = 0.f;
    if (j < L && d < dh) x = __ldg(src + ((int64_t)b * L + j) * HD + (int64_t)h * dh + d);
    dst[row * LD + (d / DT) * SL + d % DT] = x;
  }
}

template <int DT>
__device__ __forceinline__ float att_dot(const float (&x)[DT], const float* y) {
  float s = 0.f;
#pragma unroll
  for (int d = 0; d < DT; d += 4) {
    const float4 w = *reinterpret_cast<const float4*>(y + d);
    s = fmaf(x[d], w.x, s);
    s = fmaf(x[d + 1], w.y, s);
    s = fmaf(x[d + 2], w.z, s);
    s = fmaf(x[d + 3], w.w, s);
  }
  return s;
}

template <int DT>
__device__ __forceinline__ void att_axpy(float (&acc)[DT], float c, const float* y) {
#pragma unroll
  for (int d = 0; d < DT; d += 4) {
    const float4 w = *reinterpret_cast<const float4*>(y + d);
    acc[d] = fmaf(c, w.x, acc[d]);
    acc[d + 1] = fmaf(c, w.y, acc[d + 1]);
    acc[d + 2] = fmaf(c, w.z, acc[d + 2]);
    acc[d + 3] = fmaf(c, w.w, acc[d + 3]);
  }
}

template <int DT>
__device__ __forceinline__ void att_load_row(const float* p, int g, int dh, bool valid, float (&x)[DT]) {
#pragma unroll
  for (int d = 0; d < DT; ++d) {
    const int c = g * DT + d;
    x[d] = valid && c < dh ? __ldg(p + c) : 0.f;
  }
}

template <int DT>
__device__ __forceinline__ void att_store_row(float* p, int g, int dh, const float (&x)[DT], float scale) {
#pragma unroll
  for (int d = 0; d < DT; ++d) {
    const int c = g * DT + d;
    if (c < dh) p[c] = x[d] * scale;
  }
}

}  // namespace

// grid = H*B*ntiles; CTA (r, tile) owns queries [tile*64, tile*64 + 64) of logical row r.
template <int DT, int G>
__global__ void __launch_bounds__(ATT_ROWS * G) mha_attn_fwd_kernel(const AttArgs a) {
  constexpr int SL = DT + 4, LD = G * SL;
  extern __shared__ __align__(16) float sm[];
  float* Ks = sm;
  float* Vs = Ks + ATT_TILE * LD;
  float* Ms = Vs + ATT_TILE * LD;
  const int t = threadIdx.x, row = t / G, g = t - row * G;
  const int64_t r = blockIdx.x / a.ntiles;
  const int tile = (int)(blockIdx.x - r * a.ntiles);
  const int h = (int)(r / a.B);
  const int64_t b = r - (int64_t)h * a.B;
  const int i = tile * ATT_ROWS + row;
  const bool valid = i < a.Lq;
  const int64_t HD = (int64_t)a.H * a.dh;
  const int64_t qoff = ((int64_t)b * a.Lq + i) * HD + (int64_t)h * a.dh;
  float qr[DT], o[DT];
  att_load_row<DT>(a.q + (valid ? qoff : 0), g, a.dh, valid, qr);
#pragma unroll
  for (int d = 0; d < DT; ++d) o[d] = 0.f;
  float m = -INFINITY, l = 0.f;
  const float* mrow = a.mask ? a.mask + (r % a.Bm) * a.Lk : nullptr;

  for (int j0 = 0; j0 < a.Lk; j0 += ATT_TILE) {
    __syncthreads();
    att_stage<DT, G>(a.k, b, h, a.Lk, a.dh, a.H, j0, Ks);
    att_stage<DT, G>(a.v, b, h, a.Lk, a.dh, a.H, j0, Vs);
    if (mrow)
      for (int e = t; e < ATT_TILE; e += blockDim.x) Ms[e] = j0 + e < a.Lk ? __ldg(mrow + j0 + e) : 0.f;
    __syncthreads();
    const int n = min(ATT_TILE, a.Lk - j0);
    for (int jc = 0; jc < n; jc += ATT_CHUNK) {
      float s[ATT_CHUNK];
      float cm = -INFINITY;
#pragma unroll
      for (int u = 0; u < ATT_CHUNK; ++u) {
        const int jj = jc + u;
        const float dot = group_sum<G>(att_dot<DT>(qr, Ks + jj * LD + g * SL));
        bool rep;
        const float sv = att_score(a, dot, mrow ? Ms[jj] : 0.f, i, j0 + jj, rep);
        s[u] = jj < n ? sv : -INFINITY;
        cm = fmaxf(cm, s[u]);
      }
      const float mn = fmaxf(m, cm);
      const float alpha = expf(m - mn);
      l *= alpha;
#pragma unroll
      for (int d = 0; d < DT; ++d) o[d] *= alpha;
#pragma unroll
      for (int u = 0; u < ATT_CHUNK; ++u) {
        const int jj = jc + u;
        const float p = expf(s[u] - mn);
        l += p;
        float pd = p;
        if (a.drop) pd = (jj < n && att_keep(a, r, i, j0 + jj)) ? p * a.keep_scale : 0.f;
        att_axpy<DT>(o, pd, Vs + jj * LD + g * SL);
      }
      m = mn;
    }
  }
  if (valid) {
    att_store_row<DT>(a.o + qoff, g, a.dh, o, 1.f / l);
    if (g == 0) a.lse[r * a.Lq + i] = (double)m + log((double)l);
  }
}

// grid = H*B*ceil(Lk / 64); CTA (r, tile) owns keys [tile*64, tile*64 + 64) and loops over every query of r.
template <int DT, int G>
__global__ void __launch_bounds__(ATT_ROWS * G) mha_attn_bwd_kv_kernel(const AttArgs a) {
  constexpr int SL = DT + 4, LD = G * SL;
  extern __shared__ __align__(16) float sm[];
  float* Qs = sm;
  float* Gs = Qs + ATT_TILE * LD;
  float* Ds = Gs + ATT_TILE * LD;
  float* Lh = Ds + ATT_TILE;
  float* Ll = Lh + ATT_TILE;
  const int t = threadIdx.x, row = t / G, g = t - row * G;
  const int64_t r = blockIdx.x / a.ntiles;
  const int tile = (int)(blockIdx.x - r * a.ntiles);
  const int h = (int)(r / a.B);
  const int64_t b = r - (int64_t)h * a.B;
  const int j = tile * ATT_ROWS + row;
  const bool valid = j < a.Lk;
  const int64_t HD = (int64_t)a.H * a.dh;
  const int64_t koff = ((int64_t)b * a.Lk + j) * HD + (int64_t)h * a.dh;
  float kr[DT], vr[DT], dk[DT], dv[DT];
  att_load_row<DT>(a.k + (valid ? koff : 0), g, a.dh, valid, kr);
  att_load_row<DT>(a.v + (valid ? koff : 0), g, a.dh, valid, vr);
#pragma unroll
  for (int d = 0; d < DT; ++d) dk[d] = dv[d] = 0.f;
  const float mval = a.mask && valid ? __ldg(a.mask + (r % a.Bm) * a.Lk + j) : 0.f;

  for (int i0 = 0; i0 < a.Lq; i0 += ATT_TILE) {
    __syncthreads();
    att_stage<DT, G>(a.q, b, h, a.Lq, a.dh, a.H, i0, Qs);
    att_stage<DT, G>(a.g_out, b, h, a.Lq, a.dh, a.H, i0, Gs);
    {   // D_i = rowsum(dO * O) for the tile's queries, lane group `row` takes query i0 + row
      const int i = i0 + row;
      const bool iv = i < a.Lq;
      const int64_t off = iv ? ((int64_t)b * a.Lq + i) * HD + (int64_t)h * a.dh : 0;
      float s = 0.f;
      for (int d = g * DT; d < min(a.dh, (g + 1) * DT); ++d) s = fmaf(__ldg(a.g_out + off + d), __ldg(a.out + off + d), s);
      s = group_sum<G>(s);
      if (g == 0) {
        const double l = iv ? a.lse_in[r * a.Lq + i] : 0.0;
        Ds[row] = s;
        Lh[row] = (float)l;
        Ll[row] = (float)(l - (double)(float)l);
      }
    }
    __syncthreads();
    const int n = min(ATT_TILE, a.Lq - i0);
    for (int ii = 0; ii < n; ++ii) {
      const int i = i0 + ii;
      const float* qi = Qs + ii * LD + g * SL;
      const float* gi = Gs + ii * LD + g * SL;
      const float dot = group_sum<G>(att_dot<DT>(kr, qi));
      const float dp = group_sum<G>(att_dot<DT>(vr, gi));
      bool rep;
      const float s = att_score(a, dot, mval, i, j, rep);
      const float p = expf((s - Lh[ii]) - Ll[ii]);
      float pd = p, dpp = dp;
      if (a.drop) {
        const bool kp = att_keep(a, r, i, j);
        pd = kp ? p * a.keep_scale : 0.f;
        dpp = kp ? dp * a.keep_scale : 0.f;
      }
      att_axpy<DT>(dv, pd, gi);
      const float ds = rep ? 0.f : p * (dpp - Ds[ii]);
      att_axpy<DT>(dk, ds * a.rdiv, qi);
    }
  }
  if (valid) {
    att_store_row<DT>(a.gk + koff, g, a.dh, dk, 1.f);
    att_store_row<DT>(a.gv + koff, g, a.dh, dv, 1.f);
  }
}

// grid = H*B*ceil(Lq / 64); CTA (r, tile) owns queries [tile*64, tile*64 + 64) and loops over every key of r.
template <int DT, int G>
__global__ void __launch_bounds__(ATT_ROWS * G) mha_attn_bwd_q_kernel(const AttArgs a) {
  constexpr int SL = DT + 4, LD = G * SL;
  extern __shared__ __align__(16) float sm[];
  float* Ks = sm;
  float* Vs = Ks + ATT_TILE * LD;
  float* Ms = Vs + ATT_TILE * LD;
  const int t = threadIdx.x, row = t / G, g = t - row * G;
  const int64_t r = blockIdx.x / a.ntiles;
  const int tile = (int)(blockIdx.x - r * a.ntiles);
  const int h = (int)(r / a.B);
  const int64_t b = r - (int64_t)h * a.B;
  const int i = tile * ATT_ROWS + row;
  const bool valid = i < a.Lq;
  const int64_t HD = (int64_t)a.H * a.dh;
  const int64_t qoff = valid ? ((int64_t)b * a.Lq + i) * HD + (int64_t)h * a.dh : 0;
  float qr[DT], gr[DT], dq[DT];
  att_load_row<DT>(a.q + qoff, g, a.dh, valid, qr);
  att_load_row<DT>(a.g_out + qoff, g, a.dh, valid, gr);
  float Di = 0.f;
  {
    float orow[DT];
    att_load_row<DT>(a.out + qoff, g, a.dh, valid, orow);
#pragma unroll
    for (int d = 0; d < DT; ++d) {
      Di = fmaf(gr[d], orow[d], Di);
      dq[d] = 0.f;
    }
    Di = group_sum<G>(Di);
  }
  const double li = valid ? a.lse_in[r * a.Lq + i] : 0.0;
  const float lh = (float)li, ll = (float)(li - (double)lh);
  const float* mrow = a.mask ? a.mask + (r % a.Bm) * a.Lk : nullptr;

  for (int j0 = 0; j0 < a.Lk; j0 += ATT_TILE) {
    __syncthreads();
    att_stage<DT, G>(a.k, b, h, a.Lk, a.dh, a.H, j0, Ks);
    att_stage<DT, G>(a.v, b, h, a.Lk, a.dh, a.H, j0, Vs);
    if (mrow)
      for (int e = t; e < ATT_TILE; e += blockDim.x) Ms[e] = j0 + e < a.Lk ? __ldg(mrow + j0 + e) : 0.f;
    __syncthreads();
    const int n = min(ATT_TILE, a.Lk - j0);
    for (int jj = 0; jj < n; ++jj) {
      const int j = j0 + jj;
      const float* kj = Ks + jj * LD + g * SL;
      const float dot = group_sum<G>(att_dot<DT>(qr, kj));
      const float dp = group_sum<G>(att_dot<DT>(gr, Vs + jj * LD + g * SL));
      bool rep;
      const float s = att_score(a, dot, mrow ? Ms[jj] : 0.f, i, j, rep);
      const float p = expf((s - lh) - ll);
      float dpp = dp;
      if (a.drop) dpp = att_keep(a, r, i, j) ? dp * a.keep_scale : 0.f;
      const float ds = rep ? 0.f : p * (dpp - Di);
      att_axpy<DT>(dq, ds * a.rdiv, kj);
    }
  }
  if (valid) att_store_row<DT>(a.gq + qoff, g, a.dh, dq, 1.f);
}

// ---- LayerNorm of x + residual, row softmax (one warp per row) ------------------------------------------------------
__device__ __forceinline__ float ln_in(const float* x, const float* res, int64_t off) {
  return res ? __fadd_rn(__ldg(x + off), __ldg(res + off)) : __ldg(x + off);
}

struct LnRow {
  float mu, den;
};

// tf.nn.moments: mean, then the mean of the squared differences (population variance); den = (var + eps) ** 0.5
__device__ __forceinline__ LnRow ln_stats(const float* x, const float* res, int64_t base, int C, float eps, int lane) {
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += ln_in(x, res, base + c);
  const float mu = group_sum<32>(s) / (float)C;
  float v = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float d = ln_in(x, res, base + c) - mu;
    v = fmaf(d, d, v);
  }
  const float var = group_sum<32>(v) / (float)C;
  return LnRow{mu, sqrtf(var + eps)};
}

__global__ void __launch_bounds__(256) add_layernorm_fwd_kernel(const float* __restrict__ x,
                                                                const float* __restrict__ res,
                                                                const float* __restrict__ gamma,
                                                                const float* __restrict__ beta, int64_t N, int C,
                                                                float eps, float* __restrict__ y) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < N; r += nwarps) {
    const int64_t base = r * C;
    const LnRow st = ln_stats(x, res, base, C, eps, lane);
    for (int c = lane; c < C; c += 32) {
      const float nv = (ln_in(x, res, base + c) - st.mu) / st.den;
      y[base + c] = __fadd_rn(__fmul_rn(__ldg(gamma + c), nv), __ldg(beta + c));
    }
  }
}

// gx = (gn - mean(gn) - n * mean(gn * n)) / den with gn = gy * gamma; ggamma, gbeta: per-CTA shared-memory column
// sums, then red.global.add.
__global__ void __launch_bounds__(256) add_layernorm_bwd_kernel(const float* __restrict__ x,
                                                                const float* __restrict__ res,
                                                                const float* __restrict__ gamma,
                                                                const float* __restrict__ gy, int64_t N, int C,
                                                                float eps, float* __restrict__ gx,
                                                                float* __restrict__ ggamma,
                                                                float* __restrict__ gbeta) {
  extern __shared__ float s_g[];   // [2C]: ggamma, gbeta
  for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) s_g[c] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < N; r += nwarps) {
    const int64_t base = r * C;
    const LnRow st = ln_stats(x, res, base, C, eps, lane);
    float s1 = 0.f, s2 = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float nv = (ln_in(x, res, base + c) - st.mu) / st.den;
      const float g = __ldg(gy + base + c);
      const float gn = g * __ldg(gamma + c);
      s1 += gn;
      s2 = fmaf(gn, nv, s2);
      atomicAdd(&s_g[c], g * nv);
      atomicAdd(&s_g[C + c], g);
    }
    const float m1 = group_sum<32>(s1) / (float)C, m2 = group_sum<32>(s2) / (float)C;
    for (int c = lane; c < C; c += 32) {
      const float nv = (ln_in(x, res, base + c) - st.mu) / st.den;
      const float gn = __ldg(gy + base + c) * __ldg(gamma + c);
      gx[base + c] = (gn - m1 - nv * m2) / st.den;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    red_add_f32(ggamma + c, s_g[c]);
    red_add_f32(gbeta + c, s_g[C + c]);
  }
}

// y = exp(x - max) / sum (tf.nn.softmax over the last axis)
__global__ void __launch_bounds__(256) softmax_rows_fwd_kernel(const float* __restrict__ x, int64_t N, int V,
                                                               float* __restrict__ y) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < N; r += nwarps) {
    const float* xr = x + r * V;
    float m = -INFINITY;
    for (int c = lane; c < V; c += 32) m = fmaxf(m, __ldg(xr + c));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int c = lane; c < V; c += 32) s += expf(__ldg(xr + c) - m);
    s = group_sum<32>(s);
    for (int c = lane; c < V; c += 32) y[r * V + c] = expf(__ldg(xr + c) - m) / s;
  }
}

// gx = y * (gy - sum(gy * y))
__global__ void __launch_bounds__(256) softmax_rows_bwd_kernel(const float* __restrict__ y,
                                                               const float* __restrict__ gy, int64_t N, int V,
                                                               float* __restrict__ gx) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < N; r += nwarps) {
    const float* yr = y + r * V;
    const float* gr = gy + r * V;
    float s = 0.f;
    for (int c = lane; c < V; c += 32) s = fmaf(__ldg(gr + c), __ldg(yr + c), s);
    s = group_sum<32>(s);
    for (int c = lane; c < V; c += 32) gx[r * V + c] = __ldg(yr + c) * (__ldg(gr + c) - s);
  }
}

// ---- host ----------------------------------------------------------------------------------------------------------
enum class AttPass { kFwd, kBwdKV, kBwdQ };

template <int DT, int G>
static int att_launch(AttArgs a, AttPass pass, cudaStream_t st) {
  constexpr int LD = G * (DT + 4);
  const int L = pass == AttPass::kBwdKV ? a.Lk : a.Lq;
  a.ntiles = (L + ATT_ROWS - 1) / ATT_ROWS;
  const int64_t grid = (int64_t)a.H * a.B * a.ntiles;
  const int threads = ATT_ROWS * G;
  const int smem = (int)sizeof(float) * (2 * ATT_TILE * LD + (pass == AttPass::kBwdKV ? 3 : 1) * ATT_TILE);
  switch (pass) {
    case AttPass::kFwd:
      DR_CUDA_CALL(cudaFuncSetAttribute(mha_attn_fwd_kernel<DT, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      mha_attn_fwd_kernel<DT, G><<<(unsigned)grid, threads, smem, st>>>(a);
      DR_CUDA_LAUNCH_CHECK("mha_attn_fwd");
      break;
    case AttPass::kBwdKV:
      DR_CUDA_CALL(
          cudaFuncSetAttribute(mha_attn_bwd_kv_kernel<DT, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      mha_attn_bwd_kv_kernel<DT, G><<<(unsigned)grid, threads, smem, st>>>(a);
      DR_CUDA_LAUNCH_CHECK("mha_attn_bwd_kv");
      break;
    case AttPass::kBwdQ:
      DR_CUDA_CALL(
          cudaFuncSetAttribute(mha_attn_bwd_q_kernel<DT, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      mha_attn_bwd_q_kernel<DT, G><<<(unsigned)grid, threads, smem, st>>>(a);
      DR_CUDA_LAUNCH_CHECK("mha_attn_bwd_q");
      break;
  }
  return DR_OK;
}

// head columns per lane DT and lanes per row G: dh <= 4, 8, 16 take one lane; 32, 64, 128 take 2, 4, 8 lanes of 16
static int att_dispatch(const AttArgs& a, AttPass pass, cudaStream_t st) {
  if (a.dh <= 4) return att_launch<4, 1>(a, pass, st);
  if (a.dh <= 8) return att_launch<8, 1>(a, pass, st);
  if (a.dh <= 16) return att_launch<16, 1>(a, pass, st);
  if (a.dh <= 32) return att_launch<16, 2>(a, pass, st);
  if (a.dh <= 64) return att_launch<16, 4>(a, pass, st);
  return att_launch<16, 8>(a, pass, st);
}

static int att_setup(const char* who, AttArgs& a, const float* mask, int64_t B, int H, int Lq, int Lk, int dh,
                     int64_t Bm, int causal, float rate, uint64_t seed) {
  DR_REQUIRE(B >= 0 && H >= 1 && Lq >= 1 && Lk >= 1 && dh >= 1, DR_EINVAL,
             "%s: bad shape B=%lld H=%d Lq=%d Lk=%d dh=%d", who, (long long)B, H, Lq, Lk, dh);
  DR_REQUIRE(!mask || (Bm >= 1 && (H * B) % Bm == 0), DR_EINVAL, "%s: mask rows Bm=%lld do not divide H*B=%lld", who,
             (long long)Bm, (long long)(H * B));
  DR_REQUIRE(!causal || Lq == Lk, DR_EINVAL, "%s: causal masking needs Lq == Lk (got %d, %d)", who, Lq, Lk);
  DR_REQUIRE(rate >= 0.f && rate < 1.f, DR_EINVAL, "%s: dropout rate %g outside [0, 1)", who, (double)rate);
  DR_REQUIRE(dh <= ATT_MAX_DH, DR_ENOTSUP, "%s: dh=%d above the served cap %d", who, dh, ATT_MAX_DH);
  DR_REQUIRE((int64_t)H * B * (Lq > Lk ? Lq : Lk) < ((int64_t)1 << 31), DR_ENOTSUP,
             "%s: H*B*max(Lq, Lk) above the served cap 2^31", who);
  a.mask = mask;
  a.B = B; a.Bm = mask ? Bm : 1;
  a.H = H; a.Lq = Lq; a.Lk = Lk; a.dh = dh;
  a.causal = causal != 0;
  a.drop = rate > 0.f;
  a.thr = (uint32_t)((double)rate * 16777216.0);
  a.keep_scale = 1.0f / (1.0f - rate);
  a.div = (float)sqrt((double)dh);
  a.rdiv = 1.0f / a.div;
  a.seed = seed;
  return DR_OK;
}

static int64_t warp_rows_grid(int64_t N) {
  int64_t ctas = (N + 7) / 8;
  const int64_t cap = (int64_t)num_sms() * 16;
  return ctas > cap ? cap : ctas;
}

}  // namespace dr

using namespace dr;

extern "C" int dr_mha_attn_fwd(const float* q, const float* k, const float* v, const float* mask, int64_t B, int H,
                               int Lq, int Lk, int dh, int64_t Bm, int causal, float rate, uint64_t seed, float* out,
                               double* lse, void* stream) {
  DR_REQUIRE(B == 0 || (q && k && v && out && lse), DR_EINVAL, "dr_mha_attn_fwd: null pointer");
  AttArgs a{};
  if (int rc = att_setup("dr_mha_attn_fwd", a, mask, B, H, Lq, Lk, dh, Bm, causal, rate, seed)) return rc;
  if (B == 0) return DR_OK;
  a.q = q; a.k = k; a.v = v; a.o = out; a.lse = lse;
  return att_dispatch(a, AttPass::kFwd, (cudaStream_t)stream);
}

extern "C" int dr_mha_attn_bwd(const float* q, const float* k, const float* v, const float* mask, const float* out,
                               const double* lse, const float* g_out, int64_t B, int H, int Lq, int Lk, int dh,
                               int64_t Bm, int causal, float rate, uint64_t seed, float* gq, float* gk, float* gv,
                               void* stream) {
  DR_REQUIRE(B == 0 || (q && k && v && out && lse && g_out && gq && gk && gv), DR_EINVAL,
             "dr_mha_attn_bwd: null pointer");
  AttArgs a{};
  if (int rc = att_setup("dr_mha_attn_bwd", a, mask, B, H, Lq, Lk, dh, Bm, causal, rate, seed)) return rc;
  if (B == 0) return DR_OK;
  a.q = q; a.k = k; a.v = v; a.out = out; a.lse_in = lse; a.g_out = g_out;
  a.gq = gq; a.gk = gk; a.gv = gv;
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = att_dispatch(a, AttPass::kBwdKV, st)) return rc;
  return att_dispatch(a, AttPass::kBwdQ, st);
}

extern "C" int dr_add_layernorm_fwd(const float* x, const float* residual, const float* gamma, const float* beta,
                                    int64_t N, int C, float eps, float* y, void* stream) {
  DR_REQUIRE(gamma && beta && (N == 0 || (x && y)), DR_EINVAL, "dr_add_layernorm_fwd: null pointer");
  DR_REQUIRE(N >= 0 && C >= 1, DR_EINVAL, "dr_add_layernorm_fwd: bad shape N=%lld C=%d", (long long)N, C);
  if (N == 0) return DR_OK;
  add_layernorm_fwd_kernel<<<(unsigned)warp_rows_grid(N), 256, 0, (cudaStream_t)stream>>>(x, residual, gamma, beta,
                                                                                           N, C, eps, y);
  DR_CUDA_LAUNCH_CHECK("add_layernorm_fwd");
  return DR_OK;
}

extern "C" int dr_add_layernorm_bwd(const float* x, const float* residual, const float* gamma, const float* gy,
                                    int64_t N, int C, float eps, float* gx, float* ggamma, float* gbeta,
                                    void* stream) {
  DR_REQUIRE(gamma && ggamma && gbeta && (N == 0 || (x && gy && gx)), DR_EINVAL,
             "dr_add_layernorm_bwd: null pointer");
  DR_REQUIRE(N >= 0 && C >= 1, DR_EINVAL, "dr_add_layernorm_bwd: bad shape N=%lld C=%d", (long long)N, C);
  DR_REQUIRE(C <= 4096, DR_ENOTSUP, "dr_add_layernorm_bwd: C=%d above the served cap 4096", C);
  cudaStream_t st = (cudaStream_t)stream;
  DR_CUDA_CALL(cudaMemsetAsync(ggamma, 0, sizeof(float) * C, st));
  DR_CUDA_CALL(cudaMemsetAsync(gbeta, 0, sizeof(float) * C, st));
  if (N == 0) return DR_OK;
  int64_t ctas = warp_rows_grid(N);
  if (ctas > (int64_t)num_sms() * 8) ctas = (int64_t)num_sms() * 8;
  add_layernorm_bwd_kernel<<<(unsigned)ctas, 256, 2 * sizeof(float) * C, st>>>(x, residual, gamma, gy, N, C, eps, gx,
                                                                                 ggamma, gbeta);
  DR_CUDA_LAUNCH_CHECK("add_layernorm_bwd");
  return DR_OK;
}

extern "C" int dr_softmax_rows_fwd(const float* x, int64_t N, int V, float* y, void* stream) {
  DR_REQUIRE(N == 0 || (x && y), DR_EINVAL, "dr_softmax_rows_fwd: null pointer");
  DR_REQUIRE(N >= 0 && V >= 1, DR_EINVAL, "dr_softmax_rows_fwd: bad shape N=%lld V=%d", (long long)N, V);
  if (N == 0) return DR_OK;
  softmax_rows_fwd_kernel<<<(unsigned)warp_rows_grid(N), 256, 0, (cudaStream_t)stream>>>(x, N, V, y);
  DR_CUDA_LAUNCH_CHECK("softmax_rows_fwd");
  return DR_OK;
}

extern "C" int dr_softmax_rows_bwd(const float* y, const float* gy, int64_t N, int V, float* gx, void* stream) {
  DR_REQUIRE(N == 0 || (y && gy && gx), DR_EINVAL, "dr_softmax_rows_bwd: null pointer");
  DR_REQUIRE(N >= 0 && V >= 1, DR_EINVAL, "dr_softmax_rows_bwd: bad shape N=%lld V=%d", (long long)N, V);
  if (N == 0) return DR_OK;
  softmax_rows_bwd_kernel<<<(unsigned)warp_rows_grid(N), 256, 0, (cudaStream_t)stream>>>(y, gy, N, V, gx);
  DR_CUDA_LAUNCH_CHECK("softmax_rows_bwd");
  return DR_OK;
}
