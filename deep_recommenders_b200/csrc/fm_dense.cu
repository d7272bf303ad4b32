// Row F standalone: FM second-order interaction on a dense [B,S,D] tensor, any S >= 1,
// D >= 1 (the reference's own tests use D=5 and D=3, so no vector-width assumption here).
//   keras/models/ranking/fm.py:28-35 ; estimator/models/feature_interaction/fm.py:22-26
// One lane group of LPR lanes per example; lane c owns dims c, c+LPR, ...; for each dim the
// slot loop keeps sum and sum-of-squares in registers.  Reads are coalesced over d.
// Also here: small element-wise helpers of the training step (SGD, BCE-with-logits).
#include "common.cuh"

namespace dr {

template <int LPR>
__global__ void __launch_bounds__(256) fm_dense_fwd_kernel(const float* __restrict__ x, int64_t B, int S,
                                                            int D, float* __restrict__ out) {
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31, c = lane % LPR, g = lane / LPR;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t ntiles = (B + G - 1) / G;
  for (int64_t tile = warp; tile < ntiles; tile += nwarps) {
    const int64_t b = tile * G + g;
    float acc = 0.f;
    if (b < B) {
      const float* xb = x + (size_t)b * S * D;
      for (int d = c; d < D; d += LPR) {
        float sum = 0.f, sq = 0.f;
        for (int s = 0; s < S; ++s) {
          const float v = __ldg(xb + (size_t)s * D + d);
          sum += v;
          sq = fmaf(v, v, sq);
        }
        acc += sum * sum - sq;
      }
    }
    acc = group_sum<LPR>(acc);
    if (c == 0 && b < B) out[b] = 0.5f * acc;
  }
}

template <int LPR>
__global__ void __launch_bounds__(256) fm_dense_bwd_kernel(const float* __restrict__ x,
                                                            const float* __restrict__ gout, int64_t B, int S,
                                                            int D, float* __restrict__ gx) {
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31, c = lane % LPR, g = lane / LPR;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t ntiles = (B + G - 1) / G;
  for (int64_t tile = warp; tile < ntiles; tile += nwarps) {
    const int64_t b = tile * G + g;
    if (b >= B) continue;
    const float gb = __ldg(gout + b);
    const float* xb = x + (size_t)b * S * D;
    float* gb_out = gx + (size_t)b * S * D;
    for (int d = c; d < D; d += LPR) {
      float sum = 0.f;
      for (int s = 0; s < S; ++s) sum += __ldg(xb + (size_t)s * D + d);
      for (int s = 0; s < S; ++s) gb_out[(size_t)s * D + d] = gb * (sum - __ldg(xb + (size_t)s * D + d));
    }
  }
}

static int lpr_scalar(int D) {
  int l = 1;
  while (l < D && l < 32) l <<= 1;
  return l;
}

template <typename K, typename... Args>
static int launch_groups(K kern, int64_t B, int LPR, cudaStream_t st, const char* name, Args... args) {
  const int G = 32 / LPR;
  const int64_t ntiles = (B + G - 1) / G;
  int64_t ctas = (ntiles + 7) / 8;
  if (ctas > num_sms() * 8) ctas = num_sms() * 8;
  kern<<<(int)ctas, 256, 0, st>>>(args...);
  DR_CUDA_LAUNCH_CHECK(name);
  return DR_OK;
}

__global__ void sgd_kernel(float* __restrict__ p, const float* __restrict__ g, int64_t n, float lr) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = fmaf(-lr, g[i], p[i]);
}

// BCE on logits (mean) + gradient.  loss accumulated with one atomic per CTA.
__global__ void __launch_bounds__(256) bce_kernel(const float* __restrict__ z, const float* __restrict__ z_add, const float* __restrict__ y,
                                                   int64_t B, float invB, float* __restrict__ prob,
                                                   float* __restrict__ loss, float* __restrict__ gz) {
  __shared__ float part[8];
  float acc = 0.f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < B; i += stride) {
    const float zi = z[i] + (z_add ? z_add[i] : 0.f), yi = y[i];
    const float pr = 1.f / (1.f + expf(-zi));
    acc += fmaxf(zi, 0.f) - zi * yi + log1pf(expf(-fabsf(zi)));
    if (prob) prob[i] = pr;
    if (gz) gz[i] = (pr - yi) * invB;
  }
  acc = group_sum<32>(acc);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += part[w];
    red_add_f32(loss, t * invB);
  }
}

}  // namespace dr

using namespace dr;

#define DR_FM_DISPATCH(KERN, ...)                                                                \
  switch (lpr_scalar(D)) {                                                                       \
    case 1: return launch_groups(KERN<1>, B, 1, st, #KERN, __VA_ARGS__);                         \
    case 2: return launch_groups(KERN<2>, B, 2, st, #KERN, __VA_ARGS__);                         \
    case 4: return launch_groups(KERN<4>, B, 4, st, #KERN, __VA_ARGS__);                         \
    case 8: return launch_groups(KERN<8>, B, 8, st, #KERN, __VA_ARGS__);                         \
    case 16: return launch_groups(KERN<16>, B, 16, st, #KERN, __VA_ARGS__);                      \
    default: return launch_groups(KERN<32>, B, 32, st, #KERN, __VA_ARGS__);                      \
  }

extern "C" int dr_fm_fwd(const float* x, int64_t B, int S, int D, float* out, void* stream) {
  DR_REQUIRE(x && out, DR_EINVAL, "dr_fm_fwd: null pointer");
  DR_REQUIRE(B >= 0 && S >= 1 && D >= 1, DR_EINVAL, "dr_fm_fwd: bad shape B=%lld S=%d D=%d", (long long)B, S, D);
  if (B == 0) return DR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  DR_FM_DISPATCH(fm_dense_fwd_kernel, x, B, S, D, out);
}

extern "C" int dr_fm_bwd(const float* x, const float* g, int64_t B, int S, int D, float* gx, void* stream) {
  DR_REQUIRE(x && g && gx, DR_EINVAL, "dr_fm_bwd: null pointer");
  DR_REQUIRE(B >= 0 && S >= 1 && D >= 1, DR_EINVAL, "dr_fm_bwd: bad shape B=%lld S=%d D=%d", (long long)B, S, D);
  if (B == 0) return DR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  DR_FM_DISPATCH(fm_dense_bwd_kernel, x, g, B, S, D, gx);
}

extern "C" int dr_sgd_step(float* p, const float* g, int64_t n, float lr, void* stream) {
  DR_REQUIRE(p && g && n >= 0, DR_EINVAL, "dr_sgd_step: bad arguments");
  if (n == 0) return DR_OK;
  int64_t ctas = (n + 255) / 256;
  if (ctas > num_sms() * 8) ctas = num_sms() * 8;
  sgd_kernel<<<(int)ctas, 256, 0, (cudaStream_t)stream>>>(p, g, n, lr);
  DR_CUDA_LAUNCH_CHECK("dr_sgd_step");
  return DR_OK;
}

extern "C" int dr_bce_logits_fwd_bwd(const float* z, const float* z_add, const float* y, int64_t B, float* prob_out,
                                     float* loss_out, float* gz, void* stream) {
  DR_REQUIRE(z && y && loss_out && B >= 1, DR_EINVAL, "dr_bce_logits_fwd_bwd: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  DR_CUDA_CALL(cudaMemsetAsync(loss_out, 0, sizeof(float), st));
  int64_t ctas = (B + 255) / 256;
  if (ctas > num_sms() * 4) ctas = num_sms() * 4;
  bce_kernel<<<(int)ctas, 256, 0, st>>>(z, z_add, y, B, 1.f / (float)B, prob_out, loss_out, gz);
  DR_CUDA_LAUNCH_CHECK("dr_bce_logits_fwd_bwd");
  return DR_OK;
}
