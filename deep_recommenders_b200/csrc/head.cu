// The skinny end of the deep tower as ONE kernel: the final Dense(1) layer, the sigmoid cross-entropy and their
// backward.  In the reference this is the tail of `tf.keras.Sequential([... Dense(u, relu) ...] + [Dense(1)])`
// (keras/models/ranking/deepfm.py:30-34; estimator dnn.py:17-29 with hidden_units + [1]), `fm + dnn` (deepfm.py:46-47) and
// `binary_crossentropy` on the sigmoid (examples/train_deepfm_on_movielens_keras.py:43).  As separate launches (Dense(1)
// forward, BCE, activation gradient + column sums, the K x 1 input-gradient and weight-gradient GEMMs) these were ~70 us of
// launch-latency-bound kernels in the C2 step for < 20 MB of traffic; fused it is one pass: read a [B,K] once, write the
// pre-activation gradient of the layer below [B,K] once.
//   logit_b = a_b . w + bias + z_add_b ;  loss = mean_b bce(logit_b, y_b) ;  g_b = (sigmoid(logit_b) - y_b) / B
//   g_prev[b,k] = g_b * w[k] * act_prev'(a[b,k])       (a = act_prev(z_prev): derivative expressed through the output)
//   gw[k] = sum_b a[b,k] g_b ;  gb = sum_b g_b ;  gb_prev[k] = sum_b g_prev[b,k]
#include "common.cuh"

namespace dr {

template <int KPL>   // elements of a row per lane (K <= 32 * KPL)
__global__ void __launch_bounds__(256) head_bce_kernel(const float* __restrict__ a, const float* __restrict__ w,
                                                        const float* __restrict__ bias, const float* __restrict__ z_add,
                                                        const float* __restrict__ y, int64_t B, int K, int prev_act,
                                                        float invB, float* __restrict__ logit_out,
                                                        float* __restrict__ prob, float* __restrict__ loss,
                                                        float* __restrict__ g_logit, float* __restrict__ g_prev,
                                                        float* __restrict__ gw, float* __restrict__ gb,
                                                        float* __restrict__ gb_prev) {
  __shared__ float s_gw[32 * KPL], s_gbp[32 * KPL], s_misc[2];
  const int lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < 32 * KPL; i += blockDim.x) { s_gw[i] = 0.f; s_gbp[i] = 0.f; }
  if (threadIdx.x < 2) s_misc[threadIdx.x] = 0.f;
  __syncthreads();
  float wv[KPL], gw_acc[KPL], gbp_acc[KPL];
#pragma unroll
  for (int j = 0; j < KPL; ++j) {
    const int k = lane + 32 * j;
    wv[j] = k < K ? __ldg(w + k) : 0.f;
    gw_acc[j] = 0.f;
    gbp_acc[j] = 0.f;
  }
  const float b0 = bias ? __ldg(bias) : 0.f;
  float loss_acc = 0.f, gb_acc = 0.f;
  const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp0; r < B; r += nwarps) {
    float av[KPL];
    float dot = 0.f;
#pragma unroll
    for (int j = 0; j < KPL; ++j) {
      const int k = lane + 32 * j;
      av[j] = k < K ? __ldg(a + r * K + k) : 0.f;
      dot = fmaf(av[j], wv[j], dot);
    }
    dot = group_sum<32>(dot);
    const float z = dot + b0;                                  // Dense(1) output (what dr_dense_fwd would write)
    const float zi = z + (z_add ? __ldg(z_add + r) : 0.f), yi = __ldg(y + r);
    const float pr = 1.f / (1.f + expf(-zi));
    const float g = (pr - yi) * invB;
    if (lane == 0) {
      loss_acc += fmaxf(zi, 0.f) - zi * yi + log1pf(expf(-fabsf(zi)));
      gb_acc += g;
      if (logit_out) logit_out[r] = z;
      if (prob) prob[r] = pr;
      if (g_logit) g_logit[r] = g;
    }
#pragma unroll
    for (int j = 0; j < KPL; ++j) {
      const int k = lane + 32 * j;
      if (k < K) {
        const float gp = g * wv[j] * act_grad_from_y(av[j], prev_act);
        if (g_prev) g_prev[r * K + k] = gp;
        gw_acc[j] = fmaf(av[j], g, gw_acc[j]);
        gbp_acc[j] += gp;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < KPL; ++j) {
    atomicAdd(&s_gw[lane + 32 * j], gw_acc[j]);
    atomicAdd(&s_gbp[lane + 32 * j], gbp_acc[j]);
  }
  if (lane == 0) { atomicAdd(&s_misc[0], loss_acc); atomicAdd(&s_misc[1], gb_acc); }
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    if (gw) red_add_f32(gw + k, s_gw[k]);
    if (gb_prev) red_add_f32(gb_prev + k, s_gbp[k]);
  }
  if (threadIdx.x == 0) {
    red_add_f32(loss, s_misc[0] * invB);
    if (gb) red_add_f32(gb, s_misc[1]);
  }
}

// The DCN tail: Dense(1) on concat[x_cross, deep] (the stacking of the reference's tests/keras/test_dcn.py:27-32 on top of
// keras/models/ranking/dcn.py:70-88, plus the deep tower), sigmoid cross-entropy and their backward, WITHOUT the concat:
// the two feature blocks are read where they lie and their gradients are written where the two backward chains read them.
//   z_b = x_cross[b,:].w[0:d] + deep[b,:].w[d:d+n] + bias ;  g_b = (sigmoid(z_b) - y_b) / B
//   g_xc[b,k] = g_b w[k] ;  g_deep[b,j] = g_b w[d+j] act'(deep[b,j]) ;  gw[k] = sum_b feat[b,k] g_b
// A row (d + n floats, 960 at d = 832, n = 128) does not fit in a warp's registers next to its two column-sum arrays the
// way head_bce_kernel keeps it, so a CTA walks the batch in tiles of 8 rows (one per warp): phase 1 stages the tile in
// shared memory while each warp reduces its row's dot product against w (shared); phase 2 turns the threads into column
// owners (thread t owns columns t, t + 256, ...), which write the gradients of the 8 rows and keep the column sums of
// gw / gb_deep in shared memory without atomics.  V as in Vec<V>.
constexpr int DCN_HEAD_ROWS = 8;
constexpr int DCN_HEAD_MAX_K = 4096;

template <int V>
__global__ void __launch_bounds__(256) dcn_head_bce_kernel(const float* __restrict__ xc, const float* __restrict__ deep,
                                                            const float* __restrict__ w, const float* __restrict__ bias,
                                                            const float* __restrict__ y, int64_t B, int d, int n, int act,
                                                            float invB, float* __restrict__ logit_out,
                                                            float* __restrict__ prob, float* __restrict__ loss,
                                                            float* __restrict__ g_logit, float* __restrict__ g_xc,
                                                            float* __restrict__ g_deep, float* __restrict__ gw,
                                                            float* __restrict__ gb, float* __restrict__ gb_deep) {
  using T = Vec<V>;
  constexpr int R = DCN_HEAD_ROWS;
  extern __shared__ __align__(16) float smem[];
  const int K = d + n, dv = d / V, Kv = K / V;
  float* s_w = smem;               // [K]
  float* s_gw = s_w + K;           // [K]     this CTA's partial sum of gw
  float* s_gbd = s_gw + K;         // [n]     ... of gb_deep
  float* s_tile = s_gbd + n;       // [R][K]  the rows of the current tile
  float* s_g = s_tile + R * K;     // [R]     their g_b
  float* s_misc = s_g + R;         // loss, gb
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = threadIdx.x; k < K; k += blockDim.x) { s_w[k] = __ldg(w + k); s_gw[k] = 0.f; }
  for (int j = threadIdx.x; j < n; j += blockDim.x) s_gbd[j] = 0.f;
  if (threadIdx.x < 2) s_misc[threadIdx.x] = 0.f;
  __syncthreads();
  const float b0 = bias ? __ldg(bias) : 0.f;
  float loss_acc = 0.f, gb_acc = 0.f;
  for (int64_t t0 = (int64_t)blockIdx.x * R; t0 < B; t0 += (int64_t)gridDim.x * R) {
    const int64_t r = t0 + warp;
    if (r < B) {
      const T* xr = reinterpret_cast<const T*>(xc + r * d);
      const T* dr = reinterpret_cast<const T*>(deep + r * n);
      const T* wv = reinterpret_cast<const T*>(s_w);
      T* trow = reinterpret_cast<T*>(s_tile + warp * K);
      float dot = 0.f;
#pragma unroll 4
      for (int c = lane; c < Kv; c += 32) {
        const T f = c < dv ? xr[c] : dr[c - dv];
        const T ww = wv[c];
        trow[c] = f;
#pragma unroll
        for (int e = 0; e < V; ++e) dot = fmaf(f.v[e], ww.v[e], dot);
      }
      dot = group_sum<32>(dot);
      if (lane == 0) {
        const float z = dot + b0, yi = __ldg(y + r);
        const float pr = 1.f / (1.f + expf(-z));
        const float g = (pr - yi) * invB;
        loss_acc += fmaxf(z, 0.f) - z * yi + log1pf(expf(-fabsf(z)));
        gb_acc += g;
        s_g[warp] = g;
        if (logit_out) logit_out[r] = z;
        if (prob) prob[r] = pr;
        if (g_logit) g_logit[r] = g;
      }
    }
    __syncthreads();
    const int rows = (int)min((int64_t)R, B - t0);
    for (int c = threadIdx.x; c < Kv; c += blockDim.x) {
      const bool is_x = c < dv;
      const T ww = reinterpret_cast<const T*>(s_w)[c];
      T gw_acc = {}, gbd_acc = {};
#pragma unroll
      for (int i = 0; i < R; ++i) {
        if (i < rows) {
          const T f = reinterpret_cast<const T*>(s_tile + i * K)[c];
          const float g = s_g[i];
          T o;
#pragma unroll
          for (int e = 0; e < V; ++e) {
            o.v[e] = g * ww.v[e] * (is_x ? 1.f : act_grad_from_y(f.v[e], act));
            gw_acc.v[e] = fmaf(f.v[e], g, gw_acc.v[e]);
            gbd_acc.v[e] += o.v[e];
          }
          if (is_x) {
            if (g_xc) reinterpret_cast<T*>(g_xc + (t0 + i) * d)[c] = o;
          } else if (g_deep) {
            reinterpret_cast<T*>(g_deep + (t0 + i) * n)[c - dv] = o;
          }
        }
      }
#pragma unroll
      for (int e = 0; e < V; ++e) {
        s_gw[c * V + e] += gw_acc.v[e];
        if (!is_x) s_gbd[(c - dv) * V + e] += gbd_acc.v[e];
      }
    }
    __syncthreads();
  }
  if (lane == 0) { atomicAdd(&s_misc[0], loss_acc); atomicAdd(&s_misc[1], gb_acc); }
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += blockDim.x)
    if (gw) red_add_f32(gw + k, s_gw[k]);
  for (int j = threadIdx.x; j < n; j += blockDim.x)
    if (gb_deep) red_add_f32(gb_deep + j, s_gbd[j]);
  if (threadIdx.x == 0) {
    red_add_f32(loss, s_misc[0] * invB);
    if (gb) red_add_f32(gb, s_misc[1]);
  }
}

}  // namespace dr

using namespace dr;

extern "C" int dr_dense_head_bce_fwd_bwd(const float* a, const float* w, const float* bias, const float* z_add,
                                         const float* y, int64_t B, int K, int prev_act, float* logit_out,
                                         float* prob_out, float* loss_out, float* g_logit, float* g_prev, float* gw,
                                         float* gb, float* gb_prev, void* stream) {
  DR_REQUIRE(a && w && y && loss_out, DR_EINVAL, "dr_dense_head_bce_fwd_bwd: null pointer");
  DR_REQUIRE(B >= 1 && K >= 1 && K <= 256, DR_EINVAL, "dr_dense_head_bce_fwd_bwd: B=%lld K=%d (need 1 <= K <= 256)",
             (long long)B, K);
  DR_REQUIRE(prev_act >= DR_ACT_NONE && prev_act <= DR_ACT_TANH, DR_EINVAL,
             "dr_dense_head_bce_fwd_bwd: unknown activation %d", prev_act);
  cudaStream_t st = (cudaStream_t)stream;
  DR_CUDA_CALL(cudaMemsetAsync(loss_out, 0, sizeof(float), st));
  if (gw) DR_CUDA_CALL(cudaMemsetAsync(gw, 0, sizeof(float) * K, st));
  if (gb) DR_CUDA_CALL(cudaMemsetAsync(gb, 0, sizeof(float), st));
  if (gb_prev) DR_CUDA_CALL(cudaMemsetAsync(gb_prev, 0, sizeof(float) * K, st));
  int64_t ctas = (B + 7) / 8;                  // 8 warps per CTA, one row per warp iteration
  if (ctas > (int64_t)num_sms() * 8) ctas = (int64_t)num_sms() * 8;
  const float invB = 1.f / (float)B;
#define DR_HEAD(KPL)                                                                                               \
  head_bce_kernel<KPL><<<(unsigned)ctas, 256, 0, st>>>(a, w, bias, z_add, y, B, K, prev_act, invB, logit_out, prob_out, \
                                                      loss_out, g_logit, g_prev, gw, gb, gb_prev)
  if (K <= 32) DR_HEAD(1);
  else if (K <= 64) DR_HEAD(2);
  else if (K <= 128) DR_HEAD(4);
  else DR_HEAD(8);
#undef DR_HEAD
  DR_CUDA_LAUNCH_CHECK("dr_dense_head_bce_fwd_bwd");
  return DR_OK;
}

extern "C" int dr_dcn_head_bce_fwd_bwd(const float* x_cross, const float* deep, const float* w, const float* bias,
                                       const float* y, int64_t B, int d, int n, int deep_act, float* logit_out,
                                       float* prob_out, float* loss_out, float* g_logit, float* g_xc, float* g_deep,
                                       float* gw, float* gb, float* gb_deep, void* stream) {
  DR_REQUIRE(x_cross && deep && w && y && loss_out, DR_EINVAL, "dr_dcn_head_bce_fwd_bwd: null pointer");
  DR_REQUIRE(B >= 1 && d >= 1 && n >= 1, DR_EINVAL, "dr_dcn_head_bce_fwd_bwd: B=%lld d=%d n=%d (need all >= 1)",
             (long long)B, d, n);
  DR_REQUIRE(deep_act >= DR_ACT_NONE && deep_act <= DR_ACT_TANH, DR_EINVAL,
             "dr_dcn_head_bce_fwd_bwd: unknown activation %d", deep_act);
  DR_REQUIRE((int64_t)d + n <= DCN_HEAD_MAX_K, DR_ENOTSUP,
             "dr_dcn_head_bce_fwd_bwd: d + n = %lld, this kernel serves heads up to %d wide", (long long)d + n,
             DCN_HEAD_MAX_K);
  cudaStream_t st = (cudaStream_t)stream;
  const int K = d + n;
  DR_CUDA_CALL(cudaMemsetAsync(loss_out, 0, sizeof(float), st));
  if (gw) DR_CUDA_CALL(cudaMemsetAsync(gw, 0, sizeof(float) * K, st));
  if (gb) DR_CUDA_CALL(cudaMemsetAsync(gb, 0, sizeof(float), st));
  if (gb_deep) DR_CUDA_CALL(cudaMemsetAsync(gb_deep, 0, sizeof(float) * n, st));
  int64_t ctas = (B + DCN_HEAD_ROWS - 1) / DCN_HEAD_ROWS;
  if (ctas > (int64_t)num_sms() * 4) ctas = (int64_t)num_sms() * 4;
  const float invB = 1.f / (float)B;
  const size_t smem = sizeof(float) * ((size_t)(2 + DCN_HEAD_ROWS) * K + n + DCN_HEAD_ROWS + 2);
  const bool vec = (d & 3) == 0 && (n & 3) == 0 && aligned16(x_cross) && aligned16(deep) && aligned16(g_xc) &&
                   aligned16(g_deep);
#define DR_DCN_HEAD(V)                                                                                              \
  do {                                                                                                              \
    DR_CUDA_CALL(cudaFuncSetAttribute(dcn_head_bce_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    dcn_head_bce_kernel<V><<<(unsigned)ctas, 256, smem, st>>>(x_cross, deep, w, bias, y, B, d, n, deep_act, invB, logit_out, \
                                                             prob_out, loss_out, g_logit, g_xc, g_deep, gw, gb, gb_deep); \
  } while (0)
  if (vec) DR_DCN_HEAD(4);
  else DR_DCN_HEAD(1);
#undef DR_DCN_HEAD
  DR_CUDA_LAUNCH_CHECK("dr_dcn_head_bce_fwd_bwd");
  return DR_OK;
}
