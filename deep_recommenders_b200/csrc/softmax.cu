// Row R (+R1, R2) of SURVEY.md section 8(a): the two-tower in-batch softmax loss,
//   keras/models/retrieval/sbcnm.py:120-151 (Retrieval.call), :78-86, :52-75,
// as ONE kernel per direction that fuses Q @ C^T with the soft-max statistics, so the
// [nq, nc] score matrix (1 GiB at B=16384) never exists in HBM:
//   FWD   : CTA keeps 64 query rows resident, streams 64-row candidate tiles, online
//           log-sum-exp per row, picks the diagonal; loss = sum_i w_i (lse_i - s_ii).
//   BWD_Q : same streaming; recomputes the tile, P = gl*w_i*inv_tau*(exp(s-lse_i) - [i==j]),
//           gQ_tile += P @ C_tile.
//   BWD_C : CTA keeps 64 candidate rows resident, streams query tiles, gC_tile += P^T @ Q_tile.
// fp32 FFMA throughout (parity bar 1e-5; see gemm.cuh for why not single-pass TF32).
// Requires D % 4 == 0, D <= 256.
#include "common.cuh"
#include <float.h>
#include <math.h>

namespace dr {

constexpr int SM_T = 64;          // tile edge (rows of Q and rows of C per tile)
constexpr int SM_LD = SM_T + 4;   // padded leading dim of the transposed tiles
enum { MODE_FWD = 0, MODE_BWD_Q = 1, MODE_BWD_C = 2 };

struct SoftmaxParams {
  const float* q; const float* c; const float* w; const float* p; const int64_t* ids;
  float inv_tau;
  int64_t nq, nc;
  int D;
  float* lse_out; float* loss_out;          // FWD
  const float* lse; const float* gloss;     // BWD
  float* gq; float* gc;
};

__host__ __device__ inline size_t softmax_smem_floats(int D, int mode) {
  size_t f = 2 * (size_t)D * SM_LD;                       // Rs^T, Ts^T  ([D][68])
  if (mode != MODE_FWD) f += (size_t)SM_T * (D + 4)       // Tr row-major ([64][D+4])
                             + (size_t)SM_T * SM_LD;      // P tile
  f += 4 * SM_T;                                          // logp[64], w[64], lse[64], spare
  return f;
}

// Load rows [row0, row0+64) of src[nrows, D] into the transposed tile Xt[d][r] and, if Xr is
// given, also row-major Xr[r][d] (ld = D+4).  Rows past nrows are zero.
__device__ __forceinline__ void load_tile(const float* __restrict__ src, int64_t row0, int64_t nrows, int D,
                                          float* __restrict__ Xt, float* __restrict__ Xr) {
  const int nvec = SM_T * (D / 4);
  for (int f = threadIdx.x; f < nvec; f += blockDim.x) {
    const int r = f / (D / 4), dq = f % (D / 4);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row0 + r < nrows) v = ldg4(src + (size_t)(row0 + r) * D + dq * 4);
    Xt[(dq * 4 + 0) * SM_LD + r] = v.x;
    Xt[(dq * 4 + 1) * SM_LD + r] = v.y;
    Xt[(dq * 4 + 2) * SM_LD + r] = v.z;
    Xt[(dq * 4 + 3) * SM_LD + r] = v.w;
    if (Xr) *reinterpret_cast<float4*>(Xr + (size_t)r * (D + 4) + dq * 4) = v;
  }
}

template <int MODE>
__global__ void __launch_bounds__(256) inbatch_softmax_kernel(const SoftmaxParams p) {
  extern __shared__ __align__(16) float smem[];
  const int D = p.D;
  float* Rt = smem;                         // resident tile, transposed
  float* Tt = Rt + (size_t)D * SM_LD;       // streamed tile, transposed
  float* Tr = Tt + (size_t)D * SM_LD;       // streamed tile, row-major (BWD only)
  float* Ps = (MODE == MODE_FWD) ? Tr : Tr + (size_t)SM_T * (D + 4);
  float* s_logp = (MODE == MODE_FWD) ? Tr : Ps + (size_t)SM_T * SM_LD;
  float* s_w = s_logp + SM_T;
  float* s_lse = s_w + SM_T;
  __shared__ int64_t s_idm[SM_T], s_idn[SM_T];
  __shared__ float s_loss[8];

  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const bool has_ids = p.ids != nullptr;
  const float NEG_INF = -INFINITY;
  const float MIN_FLOAT = -FLT_MAX / 100.0f;   // sbcnm.py:10

  // The resident tile indexes queries (FWD, BWD_Q) or candidates (BWD_C).
  const int64_t res0 = (int64_t)blockIdx.x * SM_T;
  const int64_t m_res0 = (MODE == MODE_BWD_C) ? 0 : res0;
  const int64_t n_res0 = (MODE == MODE_BWD_C) ? res0 : 0;
  load_tile((MODE == MODE_BWD_C) ? p.c : p.q, res0, (MODE == MODE_BWD_C) ? p.nc : p.nq, D, Rt, nullptr);

  const float gscale = (MODE == MODE_FWD) ? 0.f : __ldg(p.gloss) * p.inv_tau;

  // per-thread state
  float run_m[4], run_l[4], diag[4];
  constexpr int NCH = 4;   // up to 4 chunks of 64 output columns (D <= 256)
  float oacc[(MODE == MODE_FWD) ? 1 : NCH][4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { run_m[i] = NEG_INF; run_l[i] = 0.f; diag[i] = 0.f; }
  if (MODE != MODE_FWD) {
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch)
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) oacc[ch][i][j] = 0.f;
  }
  const int nch = (D + 63) / 64;

  const int64_t stream_rows = (MODE == MODE_BWD_C) ? p.nq : p.nc;
  for (int64_t s0 = 0; s0 < stream_rows; s0 += SM_T) {
    __syncthreads();   // previous iteration done with Tt / Tr / Ps / side arrays
    load_tile((MODE == MODE_BWD_C) ? p.q : p.c, s0, stream_rows, D, Tt, (MODE == MODE_FWD) ? nullptr : Tr);
    const int64_t m0 = (MODE == MODE_BWD_C) ? s0 : m_res0;   // first query row of the S tile
    const int64_t n0 = (MODE == MODE_BWD_C) ? n_res0 : s0;   // first candidate of the S tile
    if (t < SM_T) {
      const int64_t n = n0 + t, m = m0 + t;
      s_logp[t] = (p.p && n < p.nc) ? logf(__ldg(p.p + n)) : 0.f;
      s_w[t] = (m < p.nq) ? (p.w ? __ldg(p.w + m) : 1.f) : 0.f;
      if (MODE != MODE_FWD) s_lse[t] = (m < p.nq) ? __ldg(p.lse + m) : 0.f;
      if (has_ids) {
        s_idn[t] = (n < p.nc) ? __ldg(p.ids + n) : -1;
        s_idm[t] = (m < p.nc) ? __ldg(p.ids + m) : -2;   // positive of query m is candidate m
      }
    }
    __syncthreads();

    // ---- S tile: rows = queries (ty), cols = candidates (tx) ----------------------------
    const float* Qt = (MODE == MODE_BWD_C) ? Tt : Rt;
    const float* Ct = (MODE == MODE_BWD_C) ? Rt : Tt;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 4
    for (int d = 0; d < D; ++d) {
      const float4 a = *reinterpret_cast<const float4*>(Qt + (size_t)d * SM_LD + ty * 4);
      const float4 b = *reinterpret_cast<const float4*>(Ct + (size_t)d * SM_LD + tx * 4);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    // corrections, in the reference's order: -log p, + dup*MIN_FLOAT, then / temperature
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t m = m0 + ty * 4 + i;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int64_t n = n0 + tx * 4 + j;
        float s = acc[i][j];
        if (p.p) s = s - s_logp[tx * 4 + j];
        if (has_ids && m != n && s_idn[tx * 4 + j] == s_idm[ty * 4 + i]) s = s + MIN_FLOAT;
        s = s * p.inv_tau;
        if (n >= p.nc || m >= p.nq) s = NEG_INF;
        acc[i][j] = s;
      }
    }

    if (MODE == MODE_FWD) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int64_t m = m0 + ty * 4 + i;
        float tmax = fmaxf(fmaxf(acc[i][0], acc[i][1]), fmaxf(acc[i][2], acc[i][3]));
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, o));
        const float mnew = fmaxf(run_m[i], tmax);
        float add = 0.f;
        if (mnew != NEG_INF) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            add += expf(acc[i][j] - mnew);
            if (m == n0 + tx * 4 + j && m < p.nq) diag[i] = acc[i][j];
          }
        }
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) add += __shfl_xor_sync(0xffffffffu, add, o);
        if (mnew != NEG_INF) {
          run_l[i] = run_l[i] * expf(run_m[i] - mnew) + add;
          run_m[i] = mnew;
        }
      }
    } else {
      // P tile = gl * w_m * inv_tau * (softmax - onehot); masked entries are exactly 0
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int64_t m = m0 + ty * 4 + i;
        const float wm = s_w[ty * 4 + i] * gscale, lse = s_lse[ty * 4 + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int64_t n = n0 + tx * 4 + j;
          float pv = 0.f;
          if (acc[i][j] != NEG_INF) pv = expf(acc[i][j] - lse);
          if (m == n && m < p.nq) pv -= 1.f;
          acc[i][j] = pv * wm;
        }
      }
      // stage P as Ps[k][o]: (k,o) = (n,m) for BWD_Q, (m,n) for BWD_C
      if (MODE == MODE_BWD_Q) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          *reinterpret_cast<float4*>(Ps + (size_t)(tx * 4 + j) * SM_LD + ty * 4) =
              make_float4(acc[0][j], acc[1][j], acc[2][j], acc[3][j]);
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
          *reinterpret_cast<float4*>(Ps + (size_t)(ty * 4 + i) * SM_LD + tx * 4) =
              make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
      }
      __syncthreads();
      // out[o = ty*4+i][d = ch*64 + tx*4+j] += sum_k Ps[k][o] * Tr[k][d]
      // BWD_C: output rows are candidates -> thread rows must follow the n index: the S tile
      // used ty for m and tx for n, but Ps is [m][n] so reading Ps[k][ty*4+i] walks n. OK.
#pragma unroll 2
      for (int k = 0; k < SM_T; ++k) {
        const float4 a = *reinterpret_cast<const float4*>(Ps + (size_t)k * SM_LD + ty * 4);
        const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
        for (int ch = 0; ch < NCH; ++ch) {
          if (ch < nch) {
            const int d = ch * 64 + tx * 4;
            if (d < D) {
              const float4 b = *reinterpret_cast<const float4*>(Tr + (size_t)k * (D + 4) + d);
              const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
              for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) oacc[ch][i][j] = fmaf(av[i], bv[j], oacc[ch][i][j]);
            }
          }
        }
      }
    }
  }

  if (MODE == MODE_FWD) {
    float part = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t m = res0 + ty * 4 + i;
      float dg = diag[i];
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) dg += __shfl_xor_sync(0xffffffffu, dg, o);
      if (tx == 0 && m < p.nq) {
        const float lse = run_m[i] + logf(run_l[i]);
        p.lse_out[m] = lse;
        const float wm = p.w ? __ldg(p.w + m) : 1.f;
        // rows with no positive (m >= nc) have an all-zero label row: loss term is 0
        if (m < p.nc) part += wm * (lse - dg);
      }
    }
    part = group_sum<32>(part);
    if ((t & 31) == 0) s_loss[t >> 5] = part;
    __syncthreads();
    if (t == 0) {
      float tot = 0.f;
      for (int wi = 0; wi < 8; ++wi) tot += s_loss[wi];
      red_add_f32(p.loss_out, tot);
    }
  } else {
    float* out = (MODE == MODE_BWD_Q) ? p.gq : p.gc;
    const int64_t nrows = (MODE == MODE_BWD_Q) ? p.nq : p.nc;
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      if (ch >= nch) break;
      const int d = ch * 64 + tx * 4;
      if (d >= D) continue;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int64_t r = res0 + ty * 4 + i;
        if (r < nrows)
          *reinterpret_cast<float4*>(out + (size_t)r * D + d) =
              make_float4(oacc[ch][i][0], oacc[ch][i][1], oacc[ch][i][2], oacc[ch][i][3]);
      }
    }
  }
}

template <int MODE>
static int launch_softmax(const SoftmaxParams& p, int64_t res_rows, cudaStream_t st) {
  const size_t smem = softmax_smem_floats(p.D, MODE) * sizeof(float);
  auto k = inbatch_softmax_kernel<MODE>;
  DR_CUDA_CALL(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t ctas = (res_rows + SM_T - 1) / SM_T;
  k<<<(unsigned)ctas, 256, smem, st>>>(p);
  DR_CUDA_LAUNCH_CHECK("inbatch_softmax");
  return DR_OK;
}

// ---- Row R3: per-row top-k of logits + eye*MAX_FLOAT (sbcnm.py:33-49) ----------------------
// One warp per row; k rounds of warp-wide arg-max over the row (k <= 1024, rows are B wide).
__global__ void __launch_bounds__(256) hard_negative_topk_kernel(const float* __restrict__ logits, int64_t nq,
                                                                  int64_t nc, int k, float* __restrict__ out_logits,
                                                                  float* __restrict__ out_labels,
                                                                  int32_t* __restrict__ out_idx) {
  const int lane = threadIdx.x & 31;
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= nq) return;
  const float MAX_FLOAT = FLT_MAX / 100.0f;
  const float* lr = logits + (size_t)row * nc;
  float prev_v = INFINITY;
  int64_t prev_i = -1;
  for (int r = 0; r < k; ++r) {
    // largest (value, -index) strictly below (prev_v, -prev_i) in lexicographic order
    float best_v = -INFINITY;
    int64_t best_i = INT64_MAX;
    for (int64_t j = lane; j < nc; j += 32) {
      float v = __ldg(lr + j);
      if (j == row) v = v + MAX_FLOAT;
      const bool below = (v < prev_v) || (v == prev_v && j > prev_i);
      if (below && (v > best_v || (v == best_v && j < best_i))) { best_v = v; best_i = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best_v, o);
      const int64_t oi = __shfl_xor_sync(0xffffffffu, best_i, o);
      if (ov > best_v || (ov == best_v && oi < best_i)) { best_v = ov; best_i = oi; }
    }
    prev_v = best_v; prev_i = best_i;
    if (lane == 0) {
      const bool valid = best_i != INT64_MAX;
      out_idx[(size_t)row * k + r] = valid ? (int32_t)best_i : -1;
      out_logits[(size_t)row * k + r] = valid ? __ldg(lr + best_i) : 0.f;
      out_labels[(size_t)row * k + r] = (valid && best_i == row) ? 1.f : 0.f;
    }
  }
}

}  // namespace dr

using namespace dr;


namespace dr {
// ---- tensor-core form (round 2): the contraction Q C^T (sbcnm.py:129) and the two gradient contractions run on the
// wgmma 3xTF32 GEMM core; the score block [rb, nc] of rb query rows lives in a caller-provided workspace between the
// GEMM and two one-pass kernels (the FFMA kernels above never materialise scores but reach ~18 TFLOP/s; this form trades
// rb * nc * 4 B of scratch traffic -- ~1 ms / GiB at HBM speed -- for tensor-core contractions).
int softmax_scores_block(const float* q_blk, const float* c, const float* p, const int64_t* ids, int64_t row0, int64_t rb,
                         int64_t nc, int D, float* ws, cudaStream_t st);
int softmax_grad_block(const float* g_ws, const float* q_blk, const float* c, int64_t rb, int64_t nc, int D, float* gq_blk,
                       float* gc, cudaStream_t st);

// one warp per query row: online log-sum-exp over the row of raw scores (x inv_tau), diagonal pick, weighted loss
__global__ void __launch_bounds__(256) softmax_rows_fwd_kernel(const float* __restrict__ S, int64_t rb, int64_t nc,
                                                                int64_t row0, int64_t nq, float inv_tau,
                                                                const float* __restrict__ w, float* __restrict__ lse_out,
                                                                float* __restrict__ loss_out) {
  __shared__ float s_part[8];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t r = (int64_t)blockIdx.x * 8 + wid;
  float contrib = 0.f;
  if (r < rb) {
    const float* row = S + r * nc;
    float mx = -INFINITY, sum = 0.f;
    const bool vec = (nc & 3) == 0;
    if (vec) {
      for (int64_t j = lane * 4; j < nc; j += 128) {
        const float4 v = ldg_nc_na(row + j);
        const float a = v.x * inv_tau, b = v.y * inv_tau, c = v.z * inv_tau, d = v.w * inv_tau;
        const float m4 = fmaxf(fmaxf(a, b), fmaxf(c, d));
        if (m4 > mx) { sum *= expf(mx - m4); mx = m4; }
        sum += expf(a - mx) + expf(b - mx) + expf(c - mx) + expf(d - mx);
      }
    } else {
      for (int64_t j = lane; j < nc; j += 32) {
        const float a = __ldg(row + j) * inv_tau;
        if (a > mx) { sum *= expf(mx - a); mx = a; }
        sum += expf(a - mx);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, mx, o), os = __shfl_xor_sync(0xffffffffu, sum, o);
      const float nm = fmaxf(mx, om);
      sum = (nm == -INFINITY) ? 0.f : sum * expf(mx - nm) + os * expf(om - nm);
      mx = nm;
    }
    const float lse = mx + logf(sum);
    const int64_t m = row0 + r;
    if (lane == 0) {
      lse_out[m] = lse;
      const float diag = (m < nc) ? __ldg(row + m) * inv_tau : 0.f;
      contrib = (w ? __ldg(w + m) : 1.f) * (lse - diag);
    }
  }
  if (lane == 0) s_part[wid] = contrib;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += s_part[i];
    red_add_f32(loss_out, t);
  }
}

// in place: G[r, n] = gloss * w_m * inv_tau * (exp(s - lse_m) - [n == m]),  s = S[r, n] * inv_tau,  m = row0 + r
__global__ void __launch_bounds__(256) softmax_rows_bwd_kernel(float* __restrict__ S, int64_t rb, int64_t nc, int64_t row0,
                                                                float inv_tau, const float* __restrict__ w,
                                                                const float* __restrict__ lse,
                                                                const float* __restrict__ gloss) {
  const float gs = __ldg(gloss) * inv_tau;
  const int64_t n4 = nc / 4;
  const bool vec = (nc & 3) == 0;
  const int64_t total = vec ? rb * n4 : rb * nc;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < total; f += stride) {
    if (vec) {
      const int64_t r = f / n4, j = (f - r * n4) * 4;
      const int64_t m = row0 + r;
      const float wm = (w ? __ldg(w + m) : 1.f) * gs, l = __ldg(lse + m);
      float4 v = *reinterpret_cast<float4*>(S + r * nc + j);
      v.x = (expf(v.x * inv_tau - l) - (j + 0 == m ? 1.f : 0.f)) * wm;
      v.y = (expf(v.y * inv_tau - l) - (j + 1 == m ? 1.f : 0.f)) * wm;
      v.z = (expf(v.z * inv_tau - l) - (j + 2 == m ? 1.f : 0.f)) * wm;
      v.w = (expf(v.w * inv_tau - l) - (j + 3 == m ? 1.f : 0.f)) * wm;
      *reinterpret_cast<float4*>(S + r * nc + j) = v;
    } else {
      const int64_t r = f / nc, j = f - r * nc;
      const int64_t m = row0 + r;
      const float wm = (w ? __ldg(w + m) : 1.f) * gs;
      S[f] = (expf(S[f] * inv_tau - __ldg(lse + m)) - (j == m ? 1.f : 0.f)) * wm;
    }
  }
}
}  // namespace dr

static int check_softmax(const char* fn, const float* q, const float* c, int64_t nq, int64_t nc, int D) {
  DR_REQUIRE(q && c, DR_EINVAL, "%s: null Q/C", fn);
  DR_REQUIRE(nq >= 1 && nc >= 1, DR_EINVAL, "%s: empty batch (nq=%lld nc=%lld)", fn, (long long)nq, (long long)nc);
  DR_REQUIRE(D >= 4 && D <= 256 && D % 4 == 0, DR_EINVAL, "%s: D=%d unsupported (need D %% 4 == 0, D <= 256)", fn, D);
  DR_REQUIRE(aligned16(q) && aligned16(c), DR_EALIGN, "%s: Q/C not 16-B aligned", fn);
  return DR_OK;
}

extern "C" int dr_inbatch_softmax_fwd(const float* q, const float* c, const float* w, const float* p,
                                      const int64_t* cand_ids, float inv_tau, int64_t nq, int64_t nc, int D,
                                      float* lse_out, float* loss_out, void* stream) {
  if (int rc = check_softmax("dr_inbatch_softmax_fwd", q, c, nq, nc, D)) return rc;
  DR_REQUIRE(lse_out && loss_out, DR_EINVAL, "dr_inbatch_softmax_fwd: null output");
  cudaStream_t st = (cudaStream_t)stream;
  DR_CUDA_CALL(cudaMemsetAsync(loss_out, 0, sizeof(float), st));
  SoftmaxParams sp{};
  sp.q = q; sp.c = c; sp.w = w; sp.p = p; sp.ids = cand_ids; sp.inv_tau = inv_tau; sp.nq = nq; sp.nc = nc;
  sp.D = D; sp.lse_out = lse_out; sp.loss_out = loss_out;
  return launch_softmax<MODE_FWD>(sp, nq, st);
}

extern "C" int dr_inbatch_softmax_bwd(const float* q, const float* c, const float* w, const float* p,
                                      const int64_t* cand_ids, float inv_tau, int64_t nq, int64_t nc, int D,
                                      const float* lse, const float* gloss, float* gq, float* gc, void* stream) {
  if (int rc = check_softmax("dr_inbatch_softmax_bwd", q, c, nq, nc, D)) return rc;
  DR_REQUIRE(lse && gloss && gq && gc, DR_EINVAL, "dr_inbatch_softmax_bwd: null pointer");
  DR_REQUIRE(aligned16(gq) && aligned16(gc), DR_EALIGN, "dr_inbatch_softmax_bwd: gq/gc not 16-B aligned");
  cudaStream_t st = (cudaStream_t)stream;
  SoftmaxParams sp{};
  sp.q = q; sp.c = c; sp.w = w; sp.p = p; sp.ids = cand_ids; sp.inv_tau = inv_tau; sp.nq = nq; sp.nc = nc;
  sp.D = D; sp.lse = lse; sp.gloss = gloss; sp.gq = gq; sp.gc = gc;
  if (int rc = launch_softmax<MODE_BWD_Q>(sp, nq, st)) return rc;
  return launch_softmax<MODE_BWD_C>(sp, nc, st);
}


extern "C" int dr_inbatch_softmax_fwd_ws(const float* q, const float* c, const float* w, const float* p,
                                         const int64_t* cand_ids, float inv_tau, int64_t nq, int64_t nc, int D,
                                         float* scores_ws, int64_t ws_rows, float* lse_out, float* loss_out,
                                         void* stream) {
  if (int rc = check_softmax("dr_inbatch_softmax_fwd_ws", q, c, nq, nc, D)) return rc;
  DR_REQUIRE(lse_out && loss_out && scores_ws && ws_rows >= 1, DR_EINVAL, "dr_inbatch_softmax_fwd_ws: null output / workspace");
  DR_REQUIRE(aligned16(scores_ws), DR_EALIGN, "dr_inbatch_softmax_fwd_ws: workspace not 16-B aligned");
  cudaStream_t st = (cudaStream_t)stream;
  DR_CUDA_CALL(cudaMemsetAsync(loss_out, 0, sizeof(float), st));
  for (int64_t r0 = 0; r0 < nq; r0 += ws_rows) {
    const int64_t rb = nq - r0 < ws_rows ? nq - r0 : ws_rows;
    if (int rc = softmax_scores_block(q + r0 * D, c, p, cand_ids, r0, rb, nc, D, scores_ws, st)) return rc;
    softmax_rows_fwd_kernel<<<(unsigned)((rb + 7) / 8), 256, 0, st>>>(scores_ws, rb, nc, r0, nq, inv_tau, w, lse_out, loss_out);
    DR_CUDA_LAUNCH_CHECK("softmax_rows_fwd");
  }
  return DR_OK;
}

extern "C" int dr_inbatch_softmax_bwd_ws(const float* q, const float* c, const float* w, const float* p,
                                         const int64_t* cand_ids, float inv_tau, int64_t nq, int64_t nc, int D,
                                         const float* lse, const float* gloss, float* scores_ws, int64_t ws_rows,
                                         int scores_valid, float* gq, float* gc, void* stream) {
  if (int rc = check_softmax("dr_inbatch_softmax_bwd_ws", q, c, nq, nc, D)) return rc;
  DR_REQUIRE(lse && gloss && gq && gc && scores_ws && ws_rows >= 1, DR_EINVAL, "dr_inbatch_softmax_bwd_ws: null pointer");
  DR_REQUIRE(aligned16(gq) && aligned16(gc) && aligned16(scores_ws), DR_EALIGN,
             "dr_inbatch_softmax_bwd_ws: gq / gc / workspace not 16-B aligned");
  cudaStream_t st = (cudaStream_t)stream;
  DR_CUDA_CALL(cudaMemsetAsync(gc, 0, sizeof(float) * (size_t)nc * D, st));
  const bool reuse = scores_valid && ws_rows >= nq;      // the forward's raw scores of ALL rows are still in the workspace
  for (int64_t r0 = 0; r0 < nq; r0 += ws_rows) {
    const int64_t rb = nq - r0 < ws_rows ? nq - r0 : ws_rows;
    if (!reuse)
      if (int rc = softmax_scores_block(q + r0 * D, c, p, cand_ids, r0, rb, nc, D, scores_ws, st)) return rc;
    const int64_t work = rb * ((nc & 3) ? nc : nc / 4);
    int64_t ctas = (work + 255) / 256;
    if (ctas > (int64_t)num_sms() * 16) ctas = (int64_t)num_sms() * 16;
    softmax_rows_bwd_kernel<<<(unsigned)ctas, 256, 0, st>>>(scores_ws, rb, nc, r0, inv_tau, w, lse, gloss);
    DR_CUDA_LAUNCH_CHECK("softmax_rows_bwd");
    if (int rc = softmax_grad_block(scores_ws, q + r0 * D, c, rb, nc, D, gq + r0 * D, gc, st)) return rc;
  }
  return DR_OK;
}

extern "C" int dr_hard_negative_topk(const float* logits, int64_t nq, int64_t nc, int k, float* out_logits,
                                     float* out_labels, int32_t* out_idx, void* stream) {
  DR_REQUIRE(logits && out_logits && out_labels && out_idx, DR_EINVAL, "dr_hard_negative_topk: null pointer");
  DR_REQUIRE(nq >= 0 && nc >= 1 && k >= 1 && k <= nc, DR_EINVAL, "dr_hard_negative_topk: bad shape/k");
  if (nq == 0) return DR_OK;
  const int64_t ctas = (nq * 32 + 255) / 256;
  hard_negative_topk_kernel<<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(logits, nq, nc, k, out_logits,
                                                                                out_labels, out_idx);
  DR_CUDA_LAUNCH_CHECK("hard_negative_topk");
  return DR_OK;
}
