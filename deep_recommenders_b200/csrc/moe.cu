// Multi-gate mixture of experts: the gate softmax of every task and the expert mixture in one pass.
//   estimator/models/multi_task_learning/mixture_of_experts.py:46-53 (gating_network), :69 (tf.stack of the experts),
//   :73-78 (per gate: softmax, [B,1,E] @ [B,E,H], squeeze).  The backward is TensorFlow autodiff there.
//
// Layouts (no copies between the surrounding GEMMs):
//   experts [B, E*H]  expert e is column block e*H .. (e+1)*H   (what the grouped expert tower writes)
//   logits  [B, T*E]  task t's gate logits are column block t*E  (the single gating GEMM's output)
//   gates   [B, T*E]  saved softmax;  out [B, T*H]  task t's mixture is column block t*H (the grouped task towers' input)
// Forward:  gates[b,t,:] = softmax(logits[b,t,:])  (max subtracted, expf, divided by the sum, as tf.nn.softmax)
//           out[b,t,h]   = sum_e gates[b,t,e] * experts[b,e,h]       (e ascending, fmaf, starting from -0.0)
// Backward: g_experts[b,e,h] = sum_t gates[b,t,e] * g_out[b,t,h]                    (t ascending, fmaf)
//           dg[b,t,e]        = sum_h g_out[b,t,h] * experts[b,e,h]
//           g_logits[b,t,e]  = gates[b,t,e] * (dg[b,t,e] - sum_e' gates[b,t,e'] * dg[b,t,e'])
// Ownership: one warp owns a row b.  Lane e computes gate e of a task; the lanes stride over h.  The sums over h and e'
// are per-lane partials in a fixed order and a fixed xor butterfly, so every output element has one owner, there are no
// atomics, and reruns are bit-identical.  experts is read once from memory per pass (the backward's E passes over the
// row re-read g_out from L1, not the expert stack).
// Arithmetic: fp32 FFMA.
#include "common.cuh"

#include <math.h>

namespace dr {

namespace {

constexpr int MOE_WARPS = 8;
constexpr int MOE_MAX_E = 32;
constexpr int MOE_MAX_T = 16;

__device__ __forceinline__ float moe_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float moe_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// TT = T rounded up to a power of two: the per-lane task accumulators stay in registers.
template <int TT>
__global__ void __launch_bounds__(MOE_WARPS * 32) moe_mix_fwd_kernel(const float* __restrict__ experts,
                                                                     const float* __restrict__ logits, int64_t B, int E,
                                                                     int T, int H, float* __restrict__ gates,
                                                                     float* __restrict__ out) {
  __shared__ float s_gate[MOE_WARPS][MOE_MAX_T * MOE_MAX_E];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* sg = s_gate[warp];
  const int64_t EH = (int64_t)E * H, TH = (int64_t)T * H, TE = (int64_t)T * E;
  for (int64_t b = (int64_t)blockIdx.x * MOE_WARPS + warp; b < B; b += (int64_t)gridDim.x * MOE_WARPS) {
    for (int t = 0; t < T; ++t) {
      const float l = lane < E ? __ldg(logits + b * TE + t * E + lane) : -INFINITY;
      const float m = moe_warp_max(l);
      const float x = lane < E ? expf(l - m) : 0.f;
      const float s = moe_warp_sum(x);
      if (lane < E) {
        const float g = x / s;
        sg[t * E + lane] = g;
        gates[b * TE + t * E + lane] = g;
      }
    }
    __syncwarp();
    const float* ex = experts + b * EH;
    float* o = out + b * TH;
    for (int h = lane; h < H; h += 32) {
      // the sums start from -0.0: fmaf(g, v, -0.0) is exactly g * v, signed zeros included (from +0.0 a -0.0 product
      // would come out +0.0), so E = 1 returns the expert bit for bit
      float acc[TT];
#pragma unroll
      for (int t = 0; t < TT; ++t) acc[t] = -0.f;
      for (int e = 0; e < E; ++e) {
        const float v = __ldg(ex + (int64_t)e * H + h);
#pragma unroll
        for (int t = 0; t < TT; ++t)
          if (t < T) acc[t] = fmaf(sg[t * E + e], v, acc[t]);
      }
#pragma unroll
      for (int t = 0; t < TT; ++t)
        if (t < T) o[(int64_t)t * H + h] = acc[t];
    }
    __syncwarp();
  }
}

template <int TT>
__global__ void __launch_bounds__(MOE_WARPS * 32) moe_mix_bwd_kernel(const float* __restrict__ experts,
                                                                     const float* __restrict__ gates,
                                                                     const float* __restrict__ g_out, int64_t B, int E,
                                                                     int T, int H, float* __restrict__ g_experts,
                                                                     float* __restrict__ g_logits) {
  __shared__ float s_gate[MOE_WARPS][MOE_MAX_T * MOE_MAX_E];
  __shared__ float s_dg[MOE_WARPS][MOE_MAX_T * MOE_MAX_E];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* sg = s_gate[warp];
  float* sd = s_dg[warp];
  const int64_t EH = (int64_t)E * H, TH = (int64_t)T * H, TE = (int64_t)T * E;
  for (int64_t b = (int64_t)blockIdx.x * MOE_WARPS + warp; b < B; b += (int64_t)gridDim.x * MOE_WARPS) {
    for (int i = lane; i < TE; i += 32) sg[i] = __ldg(gates + b * TE + i);
    __syncwarp();
    const float* ex = experts + b * EH;
    const float* go = g_out + b * TH;
    float* gex = g_experts + b * EH;
    for (int e = 0; e < E; ++e) {
      float part[TT];
#pragma unroll
      for (int t = 0; t < TT; ++t) part[t] = 0.f;
      for (int h = lane; h < H; h += 32) {
        const float v = __ldg(ex + (int64_t)e * H + h);
        float acc = 0.f;
#pragma unroll
        for (int t = 0; t < TT; ++t)
          if (t < T) {
            const float gv = __ldg(go + (int64_t)t * H + h);
            acc = fmaf(sg[t * E + e], gv, acc);
            part[t] = fmaf(gv, v, part[t]);
          }
        gex[(int64_t)e * H + h] = acc;
      }
#pragma unroll
      for (int t = 0; t < TT; ++t)
        if (t < T) {
          const float d = moe_warp_sum(part[t]);
          if (lane == 0) sd[t * E + e] = d;
        }
    }
    __syncwarp();
    for (int t = 0; t < T; ++t) {
      const float g = lane < E ? sg[t * E + lane] : 0.f;
      const float d = lane < E ? sd[t * E + lane] : 0.f;
      const float s = moe_warp_sum(g * d);
      if (lane < E) g_logits[b * TE + t * E + lane] = g * (d - s);
    }
    __syncwarp();
  }
}

int moe_grid(int64_t B) {
  int64_t ctas = (B + MOE_WARPS - 1) / MOE_WARPS;
  const int64_t cap = (int64_t)num_sms() * 16;
  return (int)(ctas < cap ? ctas : cap);
}

int moe_check(int64_t B, int E, int T, int H, const char* what) {
  DR_REQUIRE(B >= 0 && E >= 1 && T >= 1 && H >= 1, DR_EINVAL, "%s: bad shape B=%lld E=%d T=%d H=%d", what,
             (long long)B, E, T, H);
  DR_REQUIRE(E <= MOE_MAX_E && T <= MOE_MAX_T, DR_ENOTSUP, "%s: served for 1 <= E <= %d and 1 <= T <= %d, got E=%d T=%d",
             what, MOE_MAX_E, MOE_MAX_T, E, T);
  DR_REQUIRE((int64_t)E * H < ((int64_t)1 << 31) && (int64_t)T * H < ((int64_t)1 << 31), DR_ENOTSUP,
             "%s: E*H and T*H must stay below 2^31, got E=%d T=%d H=%d", what, E, T, H);
  return DR_OK;
}

}  // namespace

}  // namespace dr

using namespace dr;

#define MOE_DISPATCH(KERNEL, T, ...)                                                    \
  do {                                                                                 \
    if ((T) <= 1) KERNEL<1><<<grid, MOE_WARPS * 32, 0, st>>>(__VA_ARGS__);             \
    else if ((T) <= 2) KERNEL<2><<<grid, MOE_WARPS * 32, 0, st>>>(__VA_ARGS__);        \
    else if ((T) <= 4) KERNEL<4><<<grid, MOE_WARPS * 32, 0, st>>>(__VA_ARGS__);        \
    else if ((T) <= 8) KERNEL<8><<<grid, MOE_WARPS * 32, 0, st>>>(__VA_ARGS__);        \
    else KERNEL<16><<<grid, MOE_WARPS * 32, 0, st>>>(__VA_ARGS__);                     \
  } while (0)

extern "C" int dr_moe_mix_fwd(const float* experts, const float* logits, int64_t B, int E, int T, int H, float* gates,
                              float* out, void* stream) {
  DR_REQUIRE(experts && logits && gates && out, DR_EINVAL, "dr_moe_mix_fwd: null pointer");
  if (int rc = moe_check(B, E, T, H, "dr_moe_mix_fwd")) return rc;
  if (B == 0) return DR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = moe_grid(B);
  MOE_DISPATCH(moe_mix_fwd_kernel, T, experts, logits, B, E, T, H, gates, out);
  DR_CUDA_LAUNCH_CHECK("moe_mix_fwd");
  return DR_OK;
}

extern "C" int dr_moe_mix_bwd(const float* experts, const float* gates, const float* g_out, int64_t B, int E, int T,
                              int H, float* g_experts, float* g_logits, void* stream) {
  DR_REQUIRE(experts && gates && g_out && g_experts && g_logits, DR_EINVAL, "dr_moe_mix_bwd: null pointer");
  if (int rc = moe_check(B, E, T, H, "dr_moe_mix_bwd")) return rc;
  if (B == 0) return DR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = moe_grid(B);
  MOE_DISPATCH(moe_mix_bwd_kernel, T, experts, gates, g_out, B, E, T, H, g_experts, g_logits);
  DR_CUDA_LAUNCH_CHECK("moe_mix_bwd");
  return DR_OK;
}
