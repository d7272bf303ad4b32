// SURVEY.md 8(f) #1 -- Adam, the optimizer both reference examples train with
// (examples/train_deepfm_on_movielens_keras.py:44 tf.keras.optimizers.Adam(); examples/train_fm_on_movielens_estimator.py:51
// tf.train.AdamOptimizer(0.01)).  TensorFlow applies Adam DENSELY even to IndexedSlices gradients: m and v of
// every row decay every step and every row of the variable moves (optimizer_v2/adam.py _resource_apply_sparse,
// training/adam.py _apply_sparse_shared: `m_t = assign(m, m * beta1)` over the whole variable, then a
// scatter_add of the touched rows).  dr_adam_step is that dense update in one pass over the parameter arena;
// the row-sparse gradients are accumulated beforehand by dr_embed_fm_bwd / dr_scatter_add with scale = 1.
// HBM-bound: 4 reads + 3 (or 4, zero_grad) writes of n floats per step.
#include "adam.cuh"

namespace dr {

__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, float* __restrict__ g,
                                                    float* __restrict__ m, float* __restrict__ v, int64_t n,
                                                    float lr_t, float omb1, float omb2, float eps, int zero_grad,
                                                    int vec_ok, const float* __restrict__ lr_t_dev) {
  if (lr_t_dev) lr_t = __ldg(lr_t_dev);   // bias-corrected rate written by dr_adam_advance (CUDA-graph friendly)
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n4 = vec_ok ? n / 4 : 0;
  for (int64_t i = tid; i < n4; i += stride) {
    float4 pp = reinterpret_cast<float4*>(p)[i];
    const float4 gg = reinterpret_cast<const float4*>(g)[i];
    float4 mm = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    adam_functor4(pp, gg, mm, vv, lr_t, omb1, omb2, eps);
    reinterpret_cast<float4*>(p)[i] = pp;
    reinterpret_cast<float4*>(m)[i] = mm;
    reinterpret_cast<float4*>(v)[i] = vv;
    if (zero_grad) reinterpret_cast<float4*>(g)[i] = f4_zero();
  }
  for (int64_t i = n4 * 4 + tid; i < n; i += stride) {
    float pp = p[i], mm = m[i], vv = v[i];
    adam_functor(pp, g[i], mm, vv, lr_t, omb1, omb2, eps);
    p[i] = pp; m[i] = mm; v[i] = vv;
    if (zero_grad) g[i] = 0.f;
  }
}

}  // namespace dr

using namespace dr;

extern "C" int dr_adam_step(float* p, float* g, float* m, float* v, int64_t n, float lr_t, float beta1, float beta2,
                            float eps, int zero_grad, const float* lr_t_dev, void* stream) {
  DR_REQUIRE(n >= 0, DR_EINVAL, "dr_adam_step: n=%lld < 0", (long long)n);
  if (n == 0) return DR_OK;
  DR_REQUIRE(p && g && m && v, DR_EINVAL, "dr_adam_step: null pointer");
  if (int rc = check_adam_hparams("dr_adam_step", beta1, beta2, eps)) return rc;
  const int vec_ok = aligned16(p) && aligned16(g) && aligned16(m) && aligned16(v);
  int64_t ctas = capped_grid(n / 4, 256, 8);
  if (ctas < 1) ctas = 1;
  adam_kernel<<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(p, g, m, v, n, lr_t, 1.f - beta1, 1.f - beta2, eps,
                                                                 zero_grad, vec_ok, lr_t_dev);
  DR_CUDA_LAUNCH_CHECK("dr_adam_step");
  return DR_OK;
}

// ---- dr_adam_step over a list of tensors in one launch -------------------------------------------------------------
// tf.keras Adam updates every variable of a model each step; a launch per variable makes a model with many small
// variables (the Transformer) launch-bound.  The tensor table and its work list travel by value in the kernel's argument
// block (no host-to-device copy, so the entry can be captured in a CUDA graph): CTA b works on chunk b - chunk0[i] of
// tensor i, the last i with chunk0[i] <= b.  Kept under the classic 4 KB argument limit: 64 tensors per launch.
namespace dr {
constexpr int kMultiTensors = 64;
constexpr int kMultiChunk = 16384;      // floats per CTA: a multiple of 4, so a 16-B aligned tensor's chunks stay aligned

struct AdamMultiArgs {
  float* p[kMultiTensors];
  float* g[kMultiTensors];
  float* m[kMultiTensors];
  float* v[kMultiTensors];
  int64_t n[kMultiTensors];
  int32_t chunk0[kMultiTensors + 1];   // first CTA of tensor i; chunk0[count] = the grid
  uint64_t vec;                        // bit i: tensor i's four pointers are 16-B aligned (float4 path)
  int count;
};

__global__ void __launch_bounds__(256) adam_multi_kernel(const __grid_constant__ AdamMultiArgs a, float lr_t,
                                                          float omb1, float omb2, float eps,
                                                          const float* __restrict__ lr_t_dev) {
  if (lr_t_dev) lr_t = __ldg(lr_t_dev);
  const int b = blockIdx.x;
  int i = 0, hi = a.count - 1;
  while (i < hi) {
    const int mid = (i + hi + 1) >> 1;
    if (a.chunk0[mid] <= b) i = mid;
    else hi = mid - 1;
  }
  float* __restrict__ p = a.p[i];
  const float* __restrict__ g = a.g[i];
  float* __restrict__ m = a.m[i];
  float* __restrict__ v = a.v[i];
  const int64_t begin = (int64_t)(b - a.chunk0[i]) * kMultiChunk;
  const int64_t end = min(begin + kMultiChunk, a.n[i]);
  const int64_t end4 = ((a.vec >> i) & 1) ? (end & ~(int64_t)3) : begin;
  for (int64_t j = begin + 4 * threadIdx.x; j < end4; j += 4 * blockDim.x) {
    float4 pp = *reinterpret_cast<const float4*>(p + j);
    const float4 gg = *reinterpret_cast<const float4*>(g + j);
    float4 mm = *reinterpret_cast<const float4*>(m + j);
    float4 vv = *reinterpret_cast<const float4*>(v + j);
    adam_functor4(pp, gg, mm, vv, lr_t, omb1, omb2, eps);
    stg4(p + j, pp);
    stg4(m + j, mm);
    stg4(v + j, vv);
  }
  for (int64_t j = end4 + threadIdx.x; j < end; j += blockDim.x) {
    float pp = p[j], mm = m[j], vv = v[j];
    adam_functor(pp, g[j], mm, vv, lr_t, omb1, omb2, eps);
    p[j] = pp; m[j] = mm; v[j] = vv;
  }
}
}  // namespace dr

extern "C" int dr_adam_step_multi(int n_tensors, float* const* p, float* const* g, float* const* m, float* const* v,
                                  const int64_t* n, float lr_t, float beta1, float beta2, float eps,
                                  const float* lr_t_dev, void* stream) {
  DR_REQUIRE(n_tensors >= 0, DR_EINVAL, "dr_adam_step_multi: n_tensors=%d < 0", n_tensors);
  if (n_tensors == 0) return DR_OK;
  DR_REQUIRE(p && g && m && v && n, DR_EINVAL, "dr_adam_step_multi: null pointer array");
  if (int rc = check_adam_hparams("dr_adam_step_multi", beta1, beta2, eps)) return rc;
  for (int i = 0; i < n_tensors; ++i) {      // every tensor is checked before the first launch
    DR_REQUIRE(n[i] >= 0, DR_EINVAL, "dr_adam_step_multi: n[%d]=%lld < 0", i, (long long)n[i]);
    DR_REQUIRE(n[i] == 0 || (p[i] && g[i] && m[i] && v[i]), DR_EINVAL, "dr_adam_step_multi: null pointer in tensor %d",
               i);
    DR_REQUIRE(n[i] / kMultiChunk < INT32_MAX, DR_EINVAL, "dr_adam_step_multi: n[%d]=%lld too large", i,
               (long long)n[i]);
  }
  AdamMultiArgs a;
  a.count = 0;
  a.vec = 0;
  int32_t grid = 0;
  auto launch = [&]() -> int {
    a.chunk0[a.count] = grid;
    adam_multi_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>(a, lr_t, 1.f - beta1, 1.f - beta2, eps,
                                                                        lr_t_dev);
    DR_CUDA_LAUNCH_CHECK("dr_adam_step_multi");
    a.count = 0;
    a.vec = 0;
    grid = 0;
    return DR_OK;
  };
  for (int i = 0; i < n_tensors; ++i) {
    if (n[i] == 0) continue;
    const int32_t chunks = (int32_t)((n[i] + kMultiChunk - 1) / kMultiChunk);
    if (a.count == kMultiTensors || grid > INT32_MAX - chunks)
      if (int rc = launch()) return rc;
    const int k = a.count++;
    a.p[k] = p[i]; a.g[k] = g[i]; a.m[k] = m[i]; a.v[k] = v[i];
    a.n[k] = n[i];
    a.chunk0[k] = grid;
    if (aligned16(p[i]) && aligned16(g[i]) && aligned16(m[i]) && aligned16(v[i])) a.vec |= 1ull << k;
    grid += chunks;
  }
  return a.count ? launch() : DR_OK;
}

// ---- step counter on the device: t += 1, lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t) -------------------------------
// Keras optimizer_v2 Adam._prepare_local: local_step = iterations + 1, beta powers in the variable dtype.  Keeping
// t and lr_t in device memory lets the whole train step (incl. the optimizer) replay as one CUDA graph.
namespace dr {
__global__ void adam_advance_kernel(int64_t* step, float lr, float b1, float b2, float* lr_t) {
  const int64_t t = *step + 1;
  *step = t;
  const double p1 = pow((double)b1, (double)t), p2 = pow((double)b2, (double)t);
  *lr_t = (float)((double)lr * sqrt(1.0 - p2) / (1.0 - p1));
}

// ---- row-sparse ("lazy") Adam over the rows one batch touched -----------------------------------------------------
// Inputs: the gradient arena g already holds the batch's row gradients summed over duplicate ids (dr_embed_fm_bwd with
// scale = 1 into g); every other row of g is zero.  One lane group per lookup (b, s): its leader claims the row by
// stamping it with the current step (atomicExch on stamp[row]); exactly one group per distinct row wins, applies the
// ApplyAdam functor to the row's 16-B chunks of (p, m, v) and clears the row of g, so g is all-zero again afterwards.
// Rows the batch did not touch keep p, m, v (tfa LazyAdam semantics; tf.keras Adam = dr_adam_step over the arena).
// HBM-bound: per distinct row 4 line reads + 4 line writes, plus one 4-B atomic per lookup.
template <int LPR, typename IdT>
__global__ void __launch_bounds__(256) lazy_adam_rows_kernel(const IdT* __restrict__ ids, int64_t n_lookups, int S,
                                                              const int64_t* __restrict__ rows,
                                                              const int64_t* __restrict__ slot_offsets,
                                                              float* __restrict__ p, float* __restrict__ g,
                                                              float* __restrict__ m, float* __restrict__ v,
                                                              int64_t row_stride, int D, int lin_in_row,
                                                              float* __restrict__ lin_p, float* __restrict__ lin_g,
                                                              float* __restrict__ lin_m, float* __restrict__ lin_v,
                                                              int32_t* __restrict__ stamp,
                                                              const int64_t* __restrict__ step_dev,
                                                              const float* __restrict__ lr_t_dev, float omb1,
                                                              float omb2, float eps) {
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31, c = lane % LPR, grp = lane / LPR;
  const int32_t step = (int32_t)(__ldg(step_dev) & 0x7fffffff);
  const float lr_t = __ldg(lr_t_dev);
  const bool chunk_ok = c * 4 < D;
  const bool lin_lane = lin_in_row && c * 4 == D;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t base = warp * G; base < n_lookups; base += nwarps * G) {
    const int64_t L = base + grp;
    int64_t row = -1;
    if (L < n_lookups) {
      const int s = (int)(L % S);
      const int64_t id = (int64_t)__ldg(ids + L);
      if ((uint64_t)id < (uint64_t)__ldg(rows + s)) row = __ldg(slot_offsets + s) + id;
    }
    int won = 0;
    if (c == 0 && row >= 0) won = atomicExch(stamp + row, step) != step;
    won = __shfl_sync(0xffffffffu, won, grp * LPR);   // every lane of the warp takes part (trip count is warp-uniform)
    if (won && (chunk_ok || lin_lane)) {
      const size_t o = (size_t)row * row_stride + c * 4;
      float4 pp = ldg4(p + o), mm = ldg4(m + o), vv = ldg4(v + o);
      const float4 gg = ldg4(g + o);
      adam_functor(pp.x, gg.x, mm.x, vv.x, lr_t, omb1, omb2, eps);
      if (!lin_lane) {   // the [w | pad] chunk only carries one parameter
        adam_functor(pp.y, gg.y, mm.y, vv.y, lr_t, omb1, omb2, eps);
        adam_functor(pp.z, gg.z, mm.z, vv.z, lr_t, omb1, omb2, eps);
        adam_functor(pp.w, gg.w, mm.w, vv.w, lr_t, omb1, omb2, eps);
      }
      stg4(p + o, pp); stg4(m + o, mm); stg4(v + o, vv); stg4(g + o, f4_zero());
    }
    if (won && lin_p && c == 0) {   // split layout: first-order weights live in their own arrays
      float pp = lin_p[row], mm = lin_m[row], vv = lin_v[row];
      adam_functor(pp, lin_g[row], mm, vv, lr_t, omb1, omb2, eps);
      lin_p[row] = pp; lin_m[row] = mm; lin_v[row] = vv; lin_g[row] = 0.f;
    }
  }
}
}  // namespace dr

extern "C" int dr_adam_advance(int64_t* step_dev, float lr, float beta1, float beta2, float* lr_t_dev, void* stream) {
  DR_REQUIRE(step_dev && lr_t_dev, DR_EINVAL, "dr_adam_advance: null pointer");
  if (int rc = check_adam_hparams("dr_adam_advance", beta1, beta2, 0.f)) return rc;
  adam_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(step_dev, lr, beta1, beta2, lr_t_dev);
  DR_CUDA_LAUNCH_CHECK("dr_adam_advance");
  return DR_OK;
}

extern "C" int dr_lazy_adam_rows(const void* ids, int id_bytes, int64_t B, int S, int D, const int64_t* rows,
                                 const int64_t* slot_offsets, float* p, float* g, float* m, float* v,
                                 int64_t row_stride, int flags, float* lin_p, float* lin_g, float* lin_m,
                                 float* lin_v, int32_t* stamp, const int64_t* step_dev, const float* lr_t_dev,
                                 float beta1, float beta2, float eps, void* stream) {
  DR_REQUIRE(B >= 0 && S >= 1 && S <= 4096, DR_EINVAL, "dr_lazy_adam_rows: B=%lld S=%d", (long long)B, S);
  DR_REQUIRE(D >= 4 && D <= 128 && D % 4 == 0, DR_EINVAL, "dr_lazy_adam_rows: D=%d unsupported", D);
  DR_REQUIRE(id_bytes == 8 || id_bytes == 4, DR_EINVAL, "dr_lazy_adam_rows: id_bytes=%d (need 4 or 8)", id_bytes);
  if (B == 0) return DR_OK;
  DR_REQUIRE(ids && rows && slot_offsets && p && g && m && v && stamp && step_dev && lr_t_dev, DR_EINVAL,
             "dr_lazy_adam_rows: null pointer");
  const int lin_in_row = (flags & DR_EMBED_LIN_IN_ROW) ? 1 : 0;
  DR_REQUIRE(row_stride >= D + (lin_in_row ? 4 : 0) && row_stride % 4 == 0 && (!lin_in_row || D <= 124), DR_EINVAL,
             "dr_lazy_adam_rows: bad row_stride=%lld for D=%d", (long long)row_stride, D);
  DR_REQUIRE(!lin_p || (lin_g && lin_m && lin_v), DR_EINVAL, "dr_lazy_adam_rows: lin_p given without lin_g/m/v");
  DR_REQUIRE(!(lin_p && lin_in_row), DR_EINVAL, "dr_lazy_adam_rows: first-order arrays AND DR_EMBED_LIN_IN_ROW");
  DR_REQUIRE(aligned16(p) && aligned16(g) && aligned16(m) && aligned16(v), DR_EALIGN,
             "dr_lazy_adam_rows: an arena base is not 16-B aligned");
  if (int rc = check_adam_hparams("dr_lazy_adam_rows", beta1, beta2, eps)) return rc;
  const int lpr = lanes_per_row(D / 4 + lin_in_row);     // the [w | pad] chunk takes a lane of its own
  const int64_t n = B * S;
  const int64_t ctas = capped_grid(n, 256 / lpr, 8);
  return with_lpr_id(lpr, id_bytes, [&](auto L, auto id) {
    using IdT = decltype(id);
    lazy_adam_rows_kernel<L, IdT><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(
        (const IdT*)ids, n, S, rows, slot_offsets, p, g, m, v, row_stride, D, lin_in_row, lin_p, lin_g, lin_m, lin_v,
        stamp, step_dev, lr_t_dev, 1.f - beta1, 1.f - beta2, eps);
    DR_CUDA_LAUNCH_CHECK("dr_lazy_adam_rows");
    return DR_OK;
  });
}
