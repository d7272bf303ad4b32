// Rows D and X of SURVEY.md section 8(a): Dense layer and DCN-v2 Cross layer, forward and
// backward, as GEMMs with fused epilogues (gemm.cuh) plus two small bandwidth-bound helpers.
//   keras/models/ranking/deepfm.py:30-34 ; estimator/models/feature_interaction/dnn.py:9-31
//   keras/models/ranking/dcn.py:35-88
#include "gemm.cuh"

namespace dr {

// gz = gy * act'(y) (in place allowed) and gb[n] += sum_m gz[m,n].  blockDim = (32, 8).
__global__ void __launch_bounds__(256) actgrad_colsum_kernel(const float* __restrict__ gy,
                                                              const float* __restrict__ y, int act, int64_t M,
                                                              int64_t N, int64_t rows_per_cta,
                                                              float* __restrict__ gz, float* __restrict__ gb) {
  __shared__ float part[8][33];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_cta;
  const int64_t r1 = min(M, r0 + rows_per_cta);
  for (int64_t nb = 0; nb < N; nb += 32) {
    const int64_t n = nb + tx;
    float acc = 0.f;
    if (n < N) {
      for (int64_t r = r0 + ty; r < r1; r += 8) {
        float v = gy[r * N + n];
        if (act != DR_ACT_NONE) {
          v *= act_grad_from_y(__ldg(y + r * N + n), act);
          gz[r * N + n] = v;
        }
        acc += v;
      }
    }
    part[ty][tx] = acc;
    __syncthreads();
    if (ty == 0 && n < N && gb) {
      float t = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) t += part[i][tx];
      red_add_f32(gb + n, t);
    }
    __syncthreads();
  }
}

// Same, for 16-B aligned rows with N a multiple of 4 and N <= 128 * NV: one warp owns whole rows (float4 per lane, NV per
// row), four rows in flight per warp, column sums in registers until the end (the generic kernel above walks 32-column
// strips with one 4-byte load in flight per thread).
template <int NV>
__global__ void __launch_bounds__(256) actgrad_colsum_v4_kernel(const float* gy, const float* __restrict__ y, int act,
                                                                 int64_t M, int N, float* gz, float* __restrict__ gb) {
  extern __shared__ float s_part[];          // [warps][N]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
  const int n4 = N >> 2;
  float4 acc[NV];
#pragma unroll
  for (int v = 0; v < NV; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
  const int64_t wid = (int64_t)blockIdx.x * warps + warp, nw = (int64_t)gridDim.x * warps;
  constexpr int R = 4;
  for (int64_t r0 = wid * R; r0 < M; r0 += nw * R) {
    float4 g[R][NV];
#pragma unroll
    for (int i = 0; i < R; ++i)
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        const int c = lane + 32 * v;
        g[i][v] = (r0 + i < M && c < n4) ? __ldcs(reinterpret_cast<const float4*>(gy + (r0 + i) * N) + c)
                                         : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    if (act != DR_ACT_NONE) {
#pragma unroll
      for (int i = 0; i < R; ++i)
#pragma unroll
        for (int v = 0; v < NV; ++v) {
          const int c = lane + 32 * v;
          if (r0 + i < M && c < n4) {
            const float4 yv = __ldg(reinterpret_cast<const float4*>(y + (r0 + i) * N) + c);
            g[i][v].x *= act_grad_from_y(yv.x, act); g[i][v].y *= act_grad_from_y(yv.y, act);
            g[i][v].z *= act_grad_from_y(yv.z, act); g[i][v].w *= act_grad_from_y(yv.w, act);
            reinterpret_cast<float4*>(gz + (r0 + i) * N)[c] = g[i][v];
          }
        }
    }
#pragma unroll
    for (int i = 0; i < R; ++i)
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        acc[v].x += g[i][v].x; acc[v].y += g[i][v].y; acc[v].z += g[i][v].z; acc[v].w += g[i][v].w;
      }
  }
  if (!gb) return;
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const int c = lane + 32 * v;
    if (c < n4) reinterpret_cast<float4*>(s_part + (size_t)warp * N)[c] = acc[v];
  }
  __syncthreads();
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    float t = 0.f;
    for (int w = 0; w < warps; ++w) t += s_part[(size_t)w * N + n];
    red_add_f32(gb + n, t);
  }
}

// gz = gy * act'(y), gb += column sums: picks the vectorised kernel when the layout allows it
static int launch_actgrad_colsum(const float* gy, const float* y, int act, int64_t M, int64_t N, int64_t rows_per_cta,
                                 float* gz, float* gb, cudaStream_t st) {
  const bool vec = (N & 3) == 0 && N <= 1024 && aligned16(gy) && (act == DR_ACT_NONE || (aligned16(y) && aligned16(gz)));
  if (vec) {
    const int nv = (int)((N / 4 + 31) / 32);
    const int threads = 256, warps = threads / 32;
    int64_t ctas = (M + warps * 4 - 1) / (warps * 4);
    if (ctas > (int64_t)num_sms() * 4) ctas = (int64_t)num_sms() * 4;
    if (ctas < 1) ctas = 1;
    const size_t smem = (size_t)warps * N * sizeof(float);
    if (nv <= 1) actgrad_colsum_v4_kernel<1><<<(unsigned)ctas, threads, smem, st>>>(gy, y, act, M, (int)N, gz, gb);
    else if (nv <= 2) actgrad_colsum_v4_kernel<2><<<(unsigned)ctas, threads, smem, st>>>(gy, y, act, M, (int)N, gz, gb);
    else if (nv <= 4) actgrad_colsum_v4_kernel<4><<<(unsigned)ctas, threads, smem, st>>>(gy, y, act, M, (int)N, gz, gb);
    else actgrad_colsum_v4_kernel<8><<<(unsigned)ctas, threads, smem, st>>>(gy, y, act, M, (int)N, gz, gb);
    DR_CUDA_LAUNCH_CHECK("actgrad_colsum_v4");
    return DR_OK;
  }
  const int64_t ctas = (M + rows_per_cta - 1) / rows_per_cta;
  actgrad_colsum_kernel<<<(unsigned)ctas, dim3(32, 8), 0, st>>>(gy, y, act, M, N, rows_per_cta, gz, gb);
  DR_CUDA_LAUNCH_CHECK("actgrad_colsum");
  return DR_OK;
}

// Cross backward prologue: h = g*x0 ; gx0 = g*u ; gb[n] += sum_m h[m,n].
__global__ void __launch_bounds__(256) cross_bwd_prologue_kernel(const float* __restrict__ g,
                                                                  const float* __restrict__ x0,
                                                                  const float* __restrict__ u, int64_t M,
                                                                  int64_t N, int64_t rows_per_cta,
                                                                  float* __restrict__ h, float* __restrict__ gx0,
                                                                  float* __restrict__ gb) {
  __shared__ float part[8][33];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_cta;
  const int64_t r1 = min(M, r0 + rows_per_cta);
  for (int64_t nb = 0; nb < N; nb += 32) {
    const int64_t n = nb + tx;
    float acc = 0.f;
    if (n < N) {
      for (int64_t r = r0 + ty; r < r1; r += 8) {
        const float gv = g[r * N + n];
        const float hv = gv * __ldg(x0 + r * N + n);
        h[r * N + n] = hv;
        if (gx0) gx0[r * N + n] = gv * __ldg(u + r * N + n);
        acc += hv;
      }
    }
    part[ty][tx] = acc;
    __syncthreads();
    if (ty == 0 && n < N && gb) {
      float t = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) t += part[i][tx];
      red_add_f32(gb + n, t);
    }
    __syncthreads();
  }
}

// The same prologue for a caller that builds the x0 gradient in place (dr_cross_bwd_acc): h = g*x0 ; gx0 += g*u ;
// gb[n] += sum_m h[m,n].  V = 4 when every row is 16-B aligned and d % 4 == 0 (N = d / 4 columns of Vec<4>), else V = 1.
// blockDim = (32, 8): a warp reads 32 consecutive columns of a row (512 B at V = 4), four rows in flight per thread.
template <int V>
__global__ void __launch_bounds__(256) cross_bwd_prologue_acc_kernel(const Vec<V>* __restrict__ g,
                                                                      const Vec<V>* __restrict__ x0,
                                                                      const Vec<V>* __restrict__ u, int64_t M, int64_t N,
                                                                      int64_t rows_per_cta, Vec<V>* __restrict__ h,
                                                                      Vec<V>* __restrict__ gx0, float* __restrict__ gb) {
  __shared__ Vec<V> part[8][33];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_cta;
  const int64_t r1 = min(M, r0 + rows_per_cta);
  constexpr int R = 4;
  for (int64_t nb = 0; nb < N; nb += 32) {
    const int64_t n = nb + tx;
    Vec<V> acc = {};
    if (n < N) {
      for (int64_t r = r0 + ty; r < r1; r += 8 * R) {
        Vec<V> gv[R], xv[R], uv[R], ov[R];
#pragma unroll
        for (int i = 0; i < R; ++i) {
          const int64_t o = (r + 8 * i) * N + n;
          if (r + 8 * i < r1) {
            gv[i] = g[o];
            xv[i] = x0[o];
            if (gx0) { uv[i] = u[o]; ov[i] = gx0[o]; }
          }
        }
#pragma unroll
        for (int i = 0; i < R; ++i) {
          const int64_t o = (r + 8 * i) * N + n;
          if (r + 8 * i < r1) {
            Vec<V> hv;
#pragma unroll
            for (int e = 0; e < V; ++e) {
              hv.v[e] = gv[i].v[e] * xv[i].v[e];
              acc.v[e] += hv.v[e];
              if (gx0) ov[i].v[e] += gv[i].v[e] * uv[i].v[e];
            }
            h[o] = hv;
            if (gx0) gx0[o] = ov[i];
          }
        }
      }
    }
    part[ty][tx] = acc;
    __syncthreads();
    if (ty == 0 && n < N && gb) {
#pragma unroll
      for (int e = 0; e < V; ++e) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += part[i][tx].v[e];
        red_add_f32(gb + n * V + e, t);
      }
    }
    __syncthreads();
  }
}

int g_tune_tc_dw_stages = 0;  // 2: weight-gradient GEMMs use the two-stage ring (co-residency with the embedding update)
int g_tune_tc_dw_share = 0;    // 1: weight-gradient GEMMs use the co-residency build (capped registers, smaller staging)

static int64_t rows_per_cta_for(int64_t M) {
  int64_t r = (M + (int64_t)num_sms() * 4 - 1) / ((int64_t)num_sms() * 4);
  r = (r + 7) / 8 * 8;
  return r < 8 ? 8 : r;
}

static int splitk_for(int64_t Mo, int64_t No, int64_t K) {
  if (g_tune_gemm_splitk > 0) return g_tune_gemm_splitk;
  const int64_t bn = No > 64 ? 128 : (No > 16 ? 32 : 16);
  const int64_t bm = No > 16 ? 128 : 256;
  const int64_t tiles = ((Mo + bm - 1) / bm) * ((No + bn - 1) / bn);
  int64_t s = (2 * num_sms() + tiles - 1) / tiles;
  const int64_t ktiles = (K + 15) / 16;
  if (s > ktiles / 8) s = ktiles / 8;
  if (s < 1) s = 1;
  if (s > 1024) s = 1024;
  return (int)s;
}

static GemmArgs mk(const float* A, const float* B, float* C, int64_t M, int64_t N, int64_t K, int64_t lda,
                   int64_t ldb, int64_t ldc, int epi) {
  GemmArgs a{};
  a.A = A; a.B = B; a.C = C; a.M = M; a.N = N; a.K = K; a.lda = lda; a.ldb = ldb; a.ldc = ldc;
  a.epi = epi; a.splitk = 1;
  return a;
}

// gW[Kw,N] = X^T[Kw,M] @ G[M,N] (split-K over the batch, atomics into zeroed gW); ldx / ldg: row pitches of X and G
// (0 = packed)
static int gemm_xt_g(const float* X, const float* G, float* gW, int64_t M, int64_t Kw, int64_t N,
                     cudaStream_t st, bool accumulate = false, int64_t ldx = 0, int64_t ldg = 0) {
  if (!accumulate) DR_CUDA_CALL(cudaMemsetAsync(gW, 0, sizeof(float) * Kw * N, st));
  GemmArgs a = mk(X, G, gW, Kw, N, M, ldx ? ldx : Kw, ldg ? ldg : N, N, EPI_ATOMIC);
  a.splitk = splitk_for(Kw, N, M);
  a.stages = g_tune_tc_dw_stages;
  a.share = g_tune_tc_dw_share;
  return gemm_launch(a, /*transA=*/true, /*transB=*/false, st);
}

// ---- GEMM legs of the tensor-core in-batch softmax (softmax.cu) -------------------------------------------------------
// raw corrected scores of query rows [row0, row0 + rb): S = Q_blk C^T - log p[n] + dup * MIN_FLOAT  -> ws [rb, nc]
int softmax_scores_block(const float* q_blk, const float* c, const float* p, const int64_t* ids, int64_t row0, int64_t rb,
                         int64_t nc, int D, float* ws, cudaStream_t st) {
  GemmArgs a = mk(q_blk, c, ws, rb, nc, D, D, D, nc, (p || ids) ? EPI_SCORES : EPI_STORE);
  a.bias = p; a.cand_ids = ids; a.row0 = row0;
  return gemm_launch(a, false, true, st);
}
// gQ_blk [rb, D] = G [rb, nc] @ C [nc, D];   gC [nc, D] += G^T @ Q_blk  (split-K atomics; gC zeroed by the caller)
int softmax_grad_block(const float* g_ws, const float* q_blk, const float* c, int64_t rb, int64_t nc, int D, float* gq_blk,
                       float* gc, cudaStream_t st) {
  GemmArgs a = mk(g_ws, c, gq_blk, rb, D, nc, nc, D, D, EPI_STORE);
  // few query rows (a sharded rank's b x (G b) block): rb / 128 output tiles cannot fill the SMs -- split the long
  // contraction over the candidates instead (partial sums meet through global reductions into the zeroed gq block)
  const int64_t tiles = ((rb + 127) / 128) * ((D + 63) / 64);
  if (tiles < num_sms() / 2 && nc >= 1024) {
    int64_t sk = (num_sms() + tiles - 1) / tiles;
    if (sk > nc / 256) sk = nc / 256;
    if (sk > 1) {
      DR_CUDA_CALL(cudaMemsetAsync(gq_blk, 0, sizeof(float) * (size_t)rb * D, st));
      a.epi = EPI_ATOMIC;
      a.splitk = (int)sk;
    }
  }
  if (int rc = gemm_launch(a, false, false, st)) return rc;
  return gemm_xt_g(g_ws, q_blk, gc, rb, nc, D, st, /*accumulate=*/true);
}

}  // namespace dr

using namespace dr;

extern "C" int dr_dense_fwd(const float* x, const float* w, const float* b, int64_t M, int K, int N, int act,
                            float* y, void* stream) {
  DR_REQUIRE(x && w && y, DR_EINVAL, "dr_dense_fwd: null pointer");
  DR_REQUIRE(M >= 0 && K >= 1 && N >= 1, DR_EINVAL, "dr_dense_fwd: bad shape");
  DR_REQUIRE(act >= DR_ACT_NONE && act <= DR_ACT_TANH, DR_EINVAL, "dr_dense_fwd: unknown activation %d", act);
  GemmArgs a = mk(x, w, y, M, N, K, K, N, N, EPI_BIAS_ACT);
  a.bias = b; a.act = act;
  return gemm_launch(a, false, false, (cudaStream_t)stream);
}

// prev_y != NULL: gx is written as (gz @ W^T) * act'(prev_y), i.e. ALREADY the pre-activation gradient of the layer
// that produced x = act(prev_z) -- the activation-gradient pass of that layer disappears into this GEMM's epilogue.
static int dense_bwd_impl(const float* x, const float* w, const float* y, const float* gy, int64_t M, int K, int N,
                          int act, float* gz_ws, float* gx, float* gw, float* gb, const float* prev_y, int prev_act,
                          cudaStream_t st) {
  if (gb) DR_CUDA_CALL(cudaMemsetAsync(gb, 0, sizeof(float) * N, st));
  if (M == 0) {
    if (gw) DR_CUDA_CALL(cudaMemsetAsync(gw, 0, sizeof(float) * (size_t)K * N, st));
    return DR_OK;
  }
  const float* gz = gy;
  if (act != DR_ACT_NONE || gb) {
    if (int rc = launch_actgrad_colsum(gy, y, act, M, N, rows_per_cta_for(M), gz_ws, gb, st)) return rc;
    if (act != DR_ACT_NONE) gz = gz_ws;
  }
  if (gx) {
    const bool chain = prev_y != nullptr && prev_act != DR_ACT_NONE;
    GemmArgs a = mk(gz, w, gx, M, K, N, N, N, K, chain ? EPI_ACTGRAD : EPI_STORE);   // gx[M,K] = gz[M,N] @ W^T
    if (chain) { a.aux0 = prev_y; a.act = prev_act; }
    if (int rc = gemm_launch(a, false, true, st)) return rc;
  }
  if (!gw) return DR_OK;      // caller computes the weight gradient in a second call (e.g. on another stream)
  return gemm_xt_g(x, gz, gw, M, K, N, st);
}

extern "C" int dr_dense_bwd(const float* x, const float* w, const float* y, const float* gy, int64_t M,
                            int K, int N, int act, float* gz_ws, float* gx, float* gw, float* gb,
                            void* stream) {
  DR_REQUIRE(x && w && gy && (gw || gx), DR_EINVAL, "dr_dense_bwd: null pointer");
  DR_REQUIRE(M >= 0 && K >= 1 && N >= 1, DR_EINVAL, "dr_dense_bwd: bad shape");
  DR_REQUIRE(act >= DR_ACT_NONE && act <= DR_ACT_TANH, DR_EINVAL, "dr_dense_bwd: unknown activation %d", act);
  DR_REQUIRE(act == DR_ACT_NONE || (y && gz_ws), DR_EINVAL, "dr_dense_bwd: activation needs y and gz_ws");
  return dense_bwd_impl(x, w, y, gy, M, K, N, act, gz_ws, gx, gw, gb, nullptr, DR_ACT_NONE, (cudaStream_t)stream);
}

extern "C" int dr_dense_bwd_chain(const float* x, const float* w, const float* y, const float* gy, int64_t M,
                                  int K, int N, int act, float* gz_ws, float* gx, float* gw, float* gb,
                                  const float* prev_y, int prev_act, void* stream) {
  DR_REQUIRE(x && w && gy && (gw || gx), DR_EINVAL, "dr_dense_bwd_chain: null pointer");
  DR_REQUIRE(M >= 0 && K >= 1 && N >= 1, DR_EINVAL, "dr_dense_bwd_chain: bad shape");
  DR_REQUIRE(act >= DR_ACT_NONE && act <= DR_ACT_TANH && prev_act >= DR_ACT_NONE && prev_act <= DR_ACT_TANH, DR_EINVAL,
             "dr_dense_bwd_chain: unknown activation %d / %d", act, prev_act);
  DR_REQUIRE(act == DR_ACT_NONE || (y && gz_ws), DR_EINVAL, "dr_dense_bwd_chain: activation needs y and gz_ws");
  DR_REQUIRE(prev_act == DR_ACT_NONE || (prev_y && gx), DR_EINVAL, "dr_dense_bwd_chain: prev_act needs prev_y and gx");
  return dense_bwd_impl(x, w, y, gy, M, K, N, act, gz_ws, gx, gw, gb, prev_y, prev_act, (cudaStream_t)stream);
}

// The activation-gradient and bias-gradient pass of dense_bwd_impl on its own, for an epilogue fused into a kernel other
// than the GEMM (the SpMM of spmm.cu), whose backward needs this pass and no GEMM.
extern "C" int dr_act_bwd_colsum(const float* y, const float* gy, int64_t M, int N, int act, float* gz, float* gb,
                                 void* stream) {
  DR_REQUIRE(M >= 0 && N >= 1, DR_EINVAL, "dr_act_bwd_colsum: bad shape M=%lld N=%d", (long long)M, N);
  DR_REQUIRE(act >= DR_ACT_NONE && act <= DR_ACT_TANH, DR_EINVAL, "dr_act_bwd_colsum: unknown activation %d", act);
  DR_REQUIRE(M == 0 || gy, DR_EINVAL, "dr_act_bwd_colsum: null pointer");
  DR_REQUIRE(act == DR_ACT_NONE || M == 0 || (y && gz), DR_EINVAL, "dr_act_bwd_colsum: activation needs y and gz");
  cudaStream_t st = (cudaStream_t)stream;
  if (gb) DR_CUDA_CALL(cudaMemsetAsync(gb, 0, sizeof(float) * N, st));
  if (M == 0 || (act == DR_ACT_NONE && !gb)) return DR_OK;
  return launch_actgrad_colsum(gy, y, act, M, N, rows_per_cta_for(M), gz, gb, st);
}

// G Dense layers of one shape on column blocks: x [M, G*K], w [G, K, N], b [G, N], y [M, G*N].  Group g is the plain
// Dense call on x[:, g*K ..] and y[:, g*N ..], run as one strided GEMM per group (the TMA path takes the strides when
// it can, the eligibility check sends the others to FFMA).
extern "C" int dr_dense_grouped_fwd(const float* x, const float* w, const float* b, int64_t M, int G, int K, int N,
                                    int act, float* y, void* stream) {
  DR_REQUIRE(x && w && y, DR_EINVAL, "dr_dense_grouped_fwd: null pointer");
  DR_REQUIRE(M >= 0 && G >= 1 && K >= 1 && N >= 1, DR_EINVAL, "dr_dense_grouped_fwd: bad shape");
  DR_REQUIRE((int64_t)G * K < ((int64_t)1 << 31) && (int64_t)G * N < ((int64_t)1 << 31), DR_EINVAL,
             "dr_dense_grouped_fwd: G*K and G*N must stay below 2^31");
  DR_REQUIRE(act >= DR_ACT_NONE && act <= DR_ACT_TANH, DR_EINVAL, "dr_dense_grouped_fwd: unknown activation %d", act);
  const int64_t ldx = (int64_t)G * K, ldy = (int64_t)G * N;
  for (int g = 0; g < G; ++g) {
    GemmArgs a = mk(x + (int64_t)g * K, w + (int64_t)g * K * N, y + (int64_t)g * N, M, N, K, ldx, N, ldy, EPI_BIAS_ACT);
    a.bias = b ? b + (int64_t)g * N : nullptr; a.act = act;
    if (int rc = gemm_launch(a, false, false, (cudaStream_t)stream)) return rc;
  }
  return DR_OK;
}

// Backward: one activation-gradient + column-sum pass over the whole [M, G*N] block (elementwise, so the Dense pass
// with N' = G*N writes gb [G, N] directly), then per group the strided dX GEMM and the split-K dW GEMM.
extern "C" int dr_dense_grouped_bwd(const float* x, const float* w, const float* y, const float* gy, int64_t M, int G,
                                    int K, int N, int act, float* gz_ws, float* gx, float* gw, float* gb, void* stream) {
  DR_REQUIRE(x && w && gy && (gw || gx), DR_EINVAL, "dr_dense_grouped_bwd: null pointer");
  DR_REQUIRE(M >= 0 && G >= 1 && K >= 1 && N >= 1, DR_EINVAL, "dr_dense_grouped_bwd: bad shape");
  DR_REQUIRE((int64_t)G * K < ((int64_t)1 << 31) && (int64_t)G * N < ((int64_t)1 << 31), DR_EINVAL,
             "dr_dense_grouped_bwd: G*K and G*N must stay below 2^31");
  DR_REQUIRE(act >= DR_ACT_NONE && act <= DR_ACT_TANH, DR_EINVAL, "dr_dense_grouped_bwd: unknown activation %d", act);
  DR_REQUIRE(act == DR_ACT_NONE || (y && gz_ws), DR_EINVAL, "dr_dense_grouped_bwd: activation needs y and gz_ws");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t ldx = (int64_t)G * K, ldy = (int64_t)G * N;
  if (gb) DR_CUDA_CALL(cudaMemsetAsync(gb, 0, sizeof(float) * ldy, st));
  if (M == 0) {
    if (gw) DR_CUDA_CALL(cudaMemsetAsync(gw, 0, sizeof(float) * (size_t)G * K * N, st));
    return DR_OK;
  }
  const float* gz = gy;
  if (act != DR_ACT_NONE || gb) {
    if (int rc = launch_actgrad_colsum(gy, y, act, M, ldy, rows_per_cta_for(M), gz_ws, gb, st)) return rc;
    if (act != DR_ACT_NONE) gz = gz_ws;
  }
  for (int g = 0; g < G; ++g) {
    const float* gz_g = gz + (int64_t)g * N;
    const float* w_g = w + (int64_t)g * K * N;
    if (gx) {
      GemmArgs a = mk(gz_g, w_g, gx + (int64_t)g * K, M, K, N, ldy, N, ldx, EPI_STORE);   // gx_g = gz_g @ W_g^T
      if (int rc = gemm_launch(a, false, true, st)) return rc;
    }
    if (gw) {
      if (int rc = gemm_xt_g(x + (int64_t)g * K, gz_g, gw + (int64_t)g * K * N, M, K, N, st, false, ldx, ldy)) return rc;
    }
  }
  return DR_OK;
}

extern "C" int dr_cross_fwd(const float* x0, const float* x, const float* w, const float* uk, const float* vk,
                            const float* b, float alpha, int64_t B, int d, int r, float* xu_ws, float* u_out,
                            float* y, void* stream) {
  DR_REQUIRE(x0 && x && y, DR_EINVAL, "dr_cross_fwd: null pointer");
  DR_REQUIRE(B >= 0 && d >= 1 && r >= 0, DR_EINVAL, "dr_cross_fwd: bad shape");
  DR_REQUIRE(alpha >= 0.f, DR_EINVAL, "dr_cross_fwd: diag scale must be non-negative, got %g", (double)alpha);
  cudaStream_t st = (cudaStream_t)stream;
  if (r == 0) {
    DR_REQUIRE(w, DR_EINVAL, "dr_cross_fwd: full-rank kernel W is NULL");
    GemmArgs a = mk(x, w, y, B, d, d, d, d, d, EPI_CROSS);
    a.bias = b; a.alpha = alpha; a.aux0 = x0; a.aux1 = x; a.out2 = u_out;
    return gemm_launch(a, false, false, st);
  }
  DR_REQUIRE(uk && vk && xu_ws, DR_EINVAL, "dr_cross_fwd: low-rank needs U, V and xu_ws");
  GemmArgs a1 = mk(x, uk, xu_ws, B, r, d, d, r, r, EPI_STORE);
  if (int rc = gemm_launch(a1, false, false, st)) return rc;
  GemmArgs a2 = mk(xu_ws, vk, y, B, d, r, r, d, d, EPI_CROSS);
  a2.bias = b; a2.alpha = alpha; a2.aux0 = x0; a2.aux1 = x; a2.out2 = u_out;
  return gemm_launch(a2, false, false, st);
}

extern "C" int dr_cross_bwd(const float* x0, const float* x, const float* w, const float* uk, const float* vk,
                            float alpha, const float* u_saved, const float* xu_saved, const float* g, int64_t B,
                            int d, int r, float* h_ws, float* t_ws, float* gx0, float* gx, float* gw,
                            float* guk, float* gvk, float* gb, void* stream) {
  DR_REQUIRE(x0 && x && g && h_ws && gx, DR_EINVAL, "dr_cross_bwd: null pointer");
  DR_REQUIRE(B >= 0 && d >= 1 && r >= 0, DR_EINVAL, "dr_cross_bwd: bad shape");
  DR_REQUIRE(!gx0 || u_saved, DR_EINVAL, "dr_cross_bwd: gx0 requested but u_saved is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  if (gb) DR_CUDA_CALL(cudaMemsetAsync(gb, 0, sizeof(float) * d, st));
  if (B == 0) return DR_OK;
  {
    const int64_t rpc = rows_per_cta_for(B);
    const int64_t ctas = (B + rpc - 1) / rpc;
    cross_bwd_prologue_kernel<<<(unsigned)ctas, dim3(32, 8), 0, st>>>(g, x0, u_saved, B, d, rpc, h_ws, gx0, gb);
    DR_CUDA_LAUNCH_CHECK("cross_bwd_prologue");
  }
  if (r == 0) {
    DR_REQUIRE(w && gw, DR_EINVAL, "dr_cross_bwd: full-rank needs W and gW");
    GemmArgs a = mk(h_ws, w, gx, B, d, d, d, d, d, EPI_CROSS_DX);   // gx = h @ W^T + alpha*h + g
    a.alpha = alpha; a.aux0 = h_ws; a.aux1 = g;
    if (int rc = gemm_launch(a, false, true, st)) return rc;
    return gemm_xt_g(x, h_ws, gw, B, d, d, st);
  }
  DR_REQUIRE(uk && vk && guk && gvk && xu_saved && t_ws, DR_EINVAL, "dr_cross_bwd: low-rank operands missing");
  if (int rc = gemm_xt_g(xu_saved, h_ws, gvk, B, r, d, st)) return rc;             // gV = (xU)^T h
  GemmArgs a1 = mk(h_ws, vk, t_ws, B, r, d, d, d, r, EPI_STORE);                   // t = h @ V^T
  if (int rc = gemm_launch(a1, false, true, st)) return rc;
  if (int rc = gemm_xt_g(x, t_ws, guk, B, d, r, st)) return rc;                    // gU = x^T t
  GemmArgs a2 = mk(t_ws, uk, gx, B, d, r, r, r, d, EPI_CROSS_DX);                  // gx = t @ U^T + ...
  a2.alpha = alpha; a2.aux0 = h_ws; a2.aux1 = g;
  return gemm_launch(a2, false, true, st);
}

extern "C" int dr_cross_bwd_acc(const float* x0, const float* x, const float* w, const float* uk, const float* vk,
                                float alpha, const float* u_saved, const float* xu_saved, const float* g, int64_t B,
                                int d, int r, float* h_ws, float* t_ws, float* gx0, float* gx, float* gw, float* guk,
                                float* gvk, float* gb, int x_is_x0, void* stream) {
  DR_REQUIRE(x0 && x && g && h_ws, DR_EINVAL, "dr_cross_bwd_acc: null pointer");
  DR_REQUIRE(B >= 0 && d >= 1 && r >= 0, DR_EINVAL, "dr_cross_bwd_acc: bad shape");
  DR_REQUIRE(!gx0 || u_saved, DR_EINVAL, "dr_cross_bwd_acc: gx0 requested but u_saved is NULL");
  if (x_is_x0)
    DR_REQUIRE(gx0 && x == x0, DR_EINVAL, "dr_cross_bwd_acc: x_is_x0 needs gx0 and x == x0");
  else
    DR_REQUIRE(gx, DR_EINVAL, "dr_cross_bwd_acc: gx is NULL (only the x_is_x0 form accumulates it into gx0)");
  if (r == 0)
    DR_REQUIRE(w && gw, DR_EINVAL, "dr_cross_bwd_acc: full-rank needs W and gW");
  else
    DR_REQUIRE(uk && vk && guk && gvk && xu_saved && t_ws, DR_EINVAL, "dr_cross_bwd_acc: low-rank operands missing");
  cudaStream_t st = (cudaStream_t)stream;
  if (gb) DR_CUDA_CALL(cudaMemsetAsync(gb, 0, sizeof(float) * d, st));
  if (B == 0) return DR_OK;
  {
    const int64_t rpc = rows_per_cta_for(B);
    const int64_t ctas = (B + rpc - 1) / rpc;
    const bool vec = (d & 3) == 0 && aligned16(g) && aligned16(x0) && aligned16(h_ws) &&
                     (!gx0 || (aligned16(u_saved) && aligned16(gx0)));
    if (vec) {
      using V4 = Vec<4>;
      cross_bwd_prologue_acc_kernel<4><<<(unsigned)ctas, dim3(32, 8), 0, st>>>(
          reinterpret_cast<const V4*>(g), reinterpret_cast<const V4*>(x0), reinterpret_cast<const V4*>(u_saved), B, d / 4,
          rpc, reinterpret_cast<V4*>(h_ws), reinterpret_cast<V4*>(gx0), gb);
    } else {
      using V1 = Vec<1>;
      cross_bwd_prologue_acc_kernel<1><<<(unsigned)ctas, dim3(32, 8), 0, st>>>(
          reinterpret_cast<const V1*>(g), reinterpret_cast<const V1*>(x0), reinterpret_cast<const V1*>(u_saved), B, d, rpc,
          reinterpret_cast<V1*>(h_ws), reinterpret_cast<V1*>(gx0), gb);
    }
    DR_CUDA_LAUNCH_CHECK("cross_bwd_prologue_acc");
  }
  float* dx = x_is_x0 ? gx0 : gx;                        // bottom layer of a stack: x IS x0, one gradient buffer
  const int epi = x_is_x0 ? EPI_CROSS_DX_ACC : EPI_CROSS_DX;
  if (r == 0) {
    GemmArgs a = mk(h_ws, w, dx, B, d, d, d, d, d, epi);                           // gx (+)= h @ W^T + alpha*h + g
    a.alpha = alpha; a.aux0 = h_ws; a.aux1 = g;
    if (int rc = gemm_launch(a, false, true, st)) return rc;
    return gemm_xt_g(x, h_ws, gw, B, d, d, st);
  }
  if (int rc = gemm_xt_g(xu_saved, h_ws, gvk, B, r, d, st)) return rc;             // gV = (xU)^T h
  GemmArgs a1 = mk(h_ws, vk, t_ws, B, r, d, d, d, r, EPI_STORE);                   // t = h @ V^T
  if (int rc = gemm_launch(a1, false, true, st)) return rc;
  if (int rc = gemm_xt_g(x, t_ws, guk, B, d, r, st)) return rc;                    // gU = x^T t
  GemmArgs a2 = mk(t_ws, uk, dx, B, d, r, r, r, d, epi);                           // gx (+)= t @ U^T + ...
  a2.alpha = alpha; a2.aux0 = h_ws; a2.aux1 = g;
  return gemm_launch(a2, false, true, st);
}

extern "C" int dr_scores_fwd(const float* q, const float* c, const float* p, const int64_t* cand_ids,
                             int64_t nq, int64_t nc, int D, float* scores, void* stream) {
  DR_REQUIRE(q && c && scores, DR_EINVAL, "dr_scores_fwd: null pointer");
  DR_REQUIRE(nq >= 0 && nc >= 1 && D >= 1, DR_EINVAL, "dr_scores_fwd: bad shape");
  GemmArgs a = mk(q, c, scores, nq, nc, D, D, D, nc, (p || cand_ids) ? EPI_SCORES : EPI_STORE);
  a.bias = p; a.cand_ids = cand_ids;
  return gemm_launch(a, false, true, (cudaStream_t)stream);
}

// Developer hook: plain C[M,N] = op(A) @ op(B) through the GEMM dispatcher (variant per dr_tune_set).
extern "C" int dr_debug_gemm(const float* A, const float* B, float* C, int64_t M, int64_t N, int64_t K, int transA,
                             int transB, void* stream) {
  GemmArgs a = mk(A, B, C, M, N, K, transA ? M : K, transB ? K : N, N, EPI_STORE);
  return gemm_launch(a, transA != 0, transB != 0, (cudaStream_t)stream);
}
