// SURVEY.md 8(f) #3 -- the small kernels around the top-k selection of the retrieval indexes and the
// FactorizedTopK metric (keras/models/retrieval/factorized_top_k.py):
//   _take_long_axis :26-41     out[i, j] = arr[i, indices[i, j]]
//   tf.gather(identifiers, indices)  (:211, :230, :334)  the same with one shared row of identifiers
//   _exclude :58-62            adjusted = scores - isin(identifiers, exclude) * 1e5
//   FactorizedTopK.update_state :487-501   positive score = rowwise q . c ; TopKCategoricalAccuracy over
//                              [positive | top-k scores] with the true class in column 0
// All HBM-bound single passes; the scores themselves come from dr_scores_fwd, the selection from dr_topk_rows.
#include "common.cuh"

namespace dr {

template <typename T>
__global__ void __launch_bounds__(256) take_long_axis_kernel(const T* __restrict__ arr, int64_t nq, int64_t ncols,
                                                              int64_t ld, const int32_t* __restrict__ idx, int k,
                                                              T* __restrict__ out) {
  const int64_t total = nq * k, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < total; f += stride) {
    const int64_t i = f / k;
    const int64_t j = (int64_t)__ldg(idx + f);
    T v = T(0);
    if (j >= 0 && j < ncols) v = __ldg(arr + (size_t)i * ld + j);   // ld == 0: one shared row (tf.gather on a vector)
    out[f] = v;
  }
}

// isin over a short exclusion list per row (e entries, typically the user's history of a few ids)
__global__ void __launch_bounds__(256) exclude_adjust_kernel(const float* __restrict__ scores,
                                                              const int64_t* __restrict__ identifiers,
                                                              const int64_t* __restrict__ exclude, int64_t nq,
                                                              int64_t n, int64_t e, float penalty,
                                                              float* __restrict__ out) {
  const int64_t total = nq * n, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < total; f += stride) {
    const int64_t i = f / n;
    const int64_t id = __ldg(identifiers + f);
    const int64_t* ex = exclude + (size_t)i * e;
    bool isin = false;
    for (int64_t t = 0; t < e; ++t) isin |= (__ldg(ex + t) == id);
    out[f] = __ldg(scores + f) - (isin ? 1.f : 0.f) * penalty;
  }
}

// out[i] = sum_d a[i, d] * b[i, d], one warp per row, fixed reduction order (lane-strided partials, butterfly)
__global__ void __launch_bounds__(256) rowwise_dot_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                           int64_t n, int D, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= n) return;
  float acc = 0.f;
  for (int d = lane; d < D; d += 32) acc = fmaf(__ldg(a + (size_t)row * D + d), __ldg(b + (size_t)row * D + d), acc);
  acc = group_sum<32>(acc);
  if (lane == 0) out[row] = acc;
}

// rank[i] = #{ j : pred[i, j] > pred[i, col] }  -- tf.math.in_top_k(pred, col, k) == rank < k (ties count as inside)
__global__ void __launch_bounds__(256) column_rank_kernel(const float* __restrict__ positive,
                                                           const float* __restrict__ others, int64_t nq, int64_t n,
                                                           int64_t ld, int32_t* __restrict__ rank) {
  const int lane = threadIdx.x & 31;
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= nq) return;
  const float t = __ldg(positive + row);
  int c = 0;
  for (int64_t j = lane; j < n; j += 32) c += __ldg(others + (size_t)row * ld + j) > t ? 1 : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) rank[row] = c;
}

static inline unsigned flat_grid(int64_t n) {
  int64_t ctas = (n + 255) / 256;
  if (ctas > num_sms() * 8) ctas = num_sms() * 8;
  return (unsigned)(ctas < 1 ? 1 : ctas);
}

}  // namespace dr

using namespace dr;

extern "C" int dr_take_long_axis(const void* arr, int elem_bytes, int64_t nq, int64_t ncols, int64_t ld,
                                 const int32_t* indices, int k, void* out, void* stream) {
  DR_REQUIRE(nq >= 0 && ncols >= 1 && k >= 1 && (ld == 0 || ld >= ncols), DR_EINVAL,
             "dr_take_long_axis: nq=%lld ncols=%lld ld=%lld k=%d", (long long)nq, (long long)ncols, (long long)ld, k);
  DR_REQUIRE(elem_bytes == 4 || elem_bytes == 8, DR_EINVAL, "dr_take_long_axis: elem_bytes=%d (need 4 or 8)", elem_bytes);
  if (nq == 0) return DR_OK;
  DR_REQUIRE(arr && indices && out, DR_EINVAL, "dr_take_long_axis: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (elem_bytes == 4)
    take_long_axis_kernel<uint32_t><<<flat_grid(nq * k), 256, 0, st>>>((const uint32_t*)arr, nq, ncols, ld, indices, k,
                                                                     (uint32_t*)out);
  else
    take_long_axis_kernel<unsigned long long><<<flat_grid(nq * k), 256, 0, st>>>(
        (const unsigned long long*)arr, nq, ncols, ld, indices, k, (unsigned long long*)out);
  DR_CUDA_LAUNCH_CHECK("dr_take_long_axis");
  return DR_OK;
}

extern "C" int dr_exclude_adjust(const float* scores, const int64_t* identifiers, const int64_t* exclude, int64_t nq,
                                 int64_t n, int64_t e, float penalty, float* adjusted, void* stream) {
  DR_REQUIRE(nq >= 0 && n >= 1 && e >= 0, DR_EINVAL, "dr_exclude_adjust: nq=%lld n=%lld e=%lld", (long long)nq,
             (long long)n, (long long)e);
  if (nq == 0) return DR_OK;
  DR_REQUIRE(scores && identifiers && adjusted && (exclude || e == 0), DR_EINVAL, "dr_exclude_adjust: null pointer");
  exclude_adjust_kernel<<<flat_grid(nq * n), 256, 0, (cudaStream_t)stream>>>(scores, identifiers, exclude, nq, n, e,
                                                                             penalty, adjusted);
  DR_CUDA_LAUNCH_CHECK("dr_exclude_adjust");
  return DR_OK;
}

extern "C" int dr_rowwise_dot(const float* a, const float* b, int64_t n, int D, float* out, void* stream) {
  DR_REQUIRE(n >= 0 && D >= 1, DR_EINVAL, "dr_rowwise_dot: n=%lld D=%d", (long long)n, D);
  if (n == 0) return DR_OK;
  DR_REQUIRE(a && b && out, DR_EINVAL, "dr_rowwise_dot: null pointer");
  rowwise_dot_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, b, n, D, out);
  DR_CUDA_LAUNCH_CHECK("dr_rowwise_dot");
  return DR_OK;
}

extern "C" int dr_column_rank(const float* positive, const float* others, int64_t nq, int64_t n, int64_t ld,
                              int32_t* rank, void* stream) {
  DR_REQUIRE(nq >= 0 && n >= 0 && ld >= n, DR_EINVAL, "dr_column_rank: nq=%lld n=%lld ld=%lld", (long long)nq,
             (long long)n, (long long)ld);
  if (nq == 0) return DR_OK;
  DR_REQUIRE(positive && rank && (others || n == 0), DR_EINVAL, "dr_column_rank: null pointer");
  column_rank_kernel<<<(unsigned)((nq * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(positive, others, nq, n, ld,
                                                                                         rank);
  DR_CUDA_LAUNCH_CHECK("dr_column_rank");
  return DR_OK;
}
