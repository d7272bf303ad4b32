// The wide half of Wide & Deep: tf.feature_column.linear_model over indicator and crossed columns
// (reference estimator/models/ranking/wide_and_deep.py:31-33) and the FTRL-Proximal update TensorFlow's
// FtrlOptimizer applies to it (examples/train_wdl_on_movielens_estimator.py:65-69).
//
// State: one 16-B record {w, z, n, g} per wide row -- the weight, FTRL's linear and accumulator slots, and the row's
// gradient for the current batch -- so the forward read, the gradient atomic and the update of a row all hit the
// same 32-B sector.  Record total_rows is the bias.  Slot s owns rows [slot_offsets[s], slot_offsets[s] + rows[s]).
//
//   forward   logit[b] = bias + sum over the lookups of b of w[row]   (OOV / out-of-range ids contribute nothing;
//             duplicates in a bag count, as an indicator column's multi-hot counts them)
//   backward  g[row] += g_logit[b] per lookup, g_bias += sum_b g_logit[b]   (float atomics: last bits vary by order)
//   ftrl      every touched row applies TensorFlow's ApplyFtrl functor (learning_rate_power = -0.5) exactly once
//             with its batch gradient, and its g is left at zero.
//
// Why the row-sparse update equals TensorFlow's dense one: linear_model treats an indicator column as a dense column,
// so ApplyFtrl rewrites every row every step.  For a row with g = 0: n' = n, z gains g - 0 * w = 0, and w is recomputed
// from the unchanged (z, n).  That leaves the row bit-identical provided w already is the function of (z, n) the last
// update wrote, which holds from the zero initialisation on (w = z = 0 gives w = 0 for any n).  A user-supplied initial
// w breaks the condition: TensorFlow would overwrite it on the first step, this kernel only on the row's first touch.
//
// A row is claimed by atomicExch(&g, 0): the lookup that receives the (nonzero) sum applies the update, the others
// receive 0 and skip it -- a zero sum is the dense no-op.  No stamp array is needed.
#include "common.cuh"

namespace dr {

struct WideBags {
  int n;
  int slot[DR_WIDE_MAX_BAGS];
  const int64_t* ids[DR_WIDE_MAX_BAGS];
  const int64_t* splits[DR_WIDE_MAX_BAGS];
};

enum WideMode { kWideFwd = 0, kWideBwd = 1, kWideFtrl = 2 };

struct FtrlParams {
  float lr, l1, l2x2;
};

// TensorFlow's ApplyFtrl functor (training_ops.cc) with learning_rate_power = -0.5, in its order of operations.
__device__ __forceinline__ void ftrl_apply(float& w, float& z, float& n, float g, const FtrlParams& p) {
  const float n_new = n + g * g;
  const float sq_new = sqrtf(n_new);
  z += g - (sq_new - sqrtf(n)) / p.lr * w;
  const float x = (z > 0.f ? p.l1 : (z < 0.f ? -p.l1 : 0.f)) - z;
  const float y = sq_new / p.lr + p.l2x2;
  w = fabsf(z) > p.l1 ? x / y : 0.f;
  n = n_new;
}

__device__ __forceinline__ void ftrl_record(float* rec, const FtrlParams& p) {
  const float g = atomicExch(rec + 3, 0.f);
  if (g != 0.f) {
    float4 r = __ldcg(reinterpret_cast<const float4*>(rec));
    ftrl_apply(r.x, r.y, r.z, g, p);
    r.w = 0.f;
    __stcg(reinterpret_cast<float4*>(rec), r);
  }
}

template <int MODE>
__device__ __forceinline__ void wide_lookup(float* state, int64_t row, float g, const FtrlParams& p, float& acc) {
  float* rec = state + 4 * row;
  if (MODE == kWideFwd) acc += __ldg(rec);
  else if (MODE == kWideBwd) red_add_f32(rec + 3, g);
  else ftrl_record(rec, p);
}

// A group of LPE lanes per example: lanes stride over the single-valued slots, then over each bag of the example.
// The minimum of 4 blocks per SM lets ptxas use up to 64 registers; with the default bound it spills a few at 32.
template <int MODE, int LPE>
__global__ void __launch_bounds__(256, 4) wide_kernel(float* __restrict__ state, int64_t total_rows,
                                                    const int64_t* __restrict__ rows,
                                                    const int64_t* __restrict__ slot_offsets,
                                                    const int64_t* __restrict__ ids, int64_t B, int S,
                                                    const WideBags bags, const float* __restrict__ g_logit,
                                                    float* __restrict__ logit, FtrlParams p) {
  constexpr int G = 32 / LPE;
  const int lane = threadIdx.x & 31, c = lane % LPE, grp = lane / LPE;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  float bias_g = 0.f;
  if (MODE == kWideFtrl && blockIdx.x == 0 && threadIdx.x == 0) ftrl_record(state + 4 * total_rows, p);
  for (int64_t base = warp * G; base < B; base += nwarps * G) {   // trip count is warp-uniform
    const int64_t b = base + grp;
    float acc = 0.f;
    if (b < B) {
      const float g = MODE == kWideBwd ? __ldg(g_logit + b) : 0.f;
      if (MODE == kWideBwd && c == 0) bias_g += g;
      for (int s = c; s < S; s += LPE) {
        bool bag = false;
#pragma unroll
        for (int i = 0; i < DR_WIDE_MAX_BAGS; ++i) bag |= i < bags.n && bags.slot[i] == s;
        const int64_t id = __ldg(ids + b * S + s);
        if (!bag && (uint64_t)id < (uint64_t)__ldg(rows + s))
          wide_lookup<MODE>(state, __ldg(slot_offsets + s) + id, g, p, acc);
      }
#pragma unroll 1
      for (int i = 0; i < bags.n; ++i) {
        const int s = bags.slot[i];
        const int64_t n_rows = __ldg(rows + s), off = __ldg(slot_offsets + s);
        const int64_t e = __ldg(bags.splits[i] + b + 1);
        for (int64_t j = __ldg(bags.splits[i] + b) + c; j < e; j += LPE) {
          const int64_t id = __ldg(bags.ids[i] + j);
          if ((uint64_t)id < (uint64_t)n_rows) wide_lookup<MODE>(state, off + id, g, p, acc);
        }
      }
    }
    if (MODE == kWideFwd) {
      acc = group_sum<LPE>(acc);
      if (b < B && c == 0) logit[b] = __ldg(state + 4 * total_rows) + acc;
    }
  }
  if (MODE == kWideBwd) {   // one atomic per block for the bias gradient
    __shared__ float part[8];
    bias_g = group_sum<32>(bias_g);
    if (lane == 0) part[threadIdx.x >> 5] = bias_g;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += part[w];
      if (t != 0.f) atomicAdd(state + 4 * total_rows + 3, t);
    }
  }
}

template <int MODE>
static int wide_launch(float* state, int64_t total_rows, const int64_t* rows, const int64_t* slot_offsets,
                       const int64_t* ids, int64_t B, int S, int n_bags, const int* bag_slots,
                       const int64_t* const* bag_ids, const int64_t* const* bag_splits, const float* g_logit,
                       float* logit, FtrlParams p, const char* who, void* stream) {
  DR_REQUIRE(B >= 0 && S >= 1 && S <= 4096 && total_rows >= 0, DR_EINVAL, "%s: B=%lld S=%d total_rows=%lld", who,
             (long long)B, S, (long long)total_rows);
  DR_REQUIRE(n_bags >= 0 && n_bags <= DR_WIDE_MAX_BAGS, DR_EINVAL, "%s: n_bags=%d (at most %d)", who, n_bags,
             DR_WIDE_MAX_BAGS);
  DR_REQUIRE(state && rows && slot_offsets && ids, DR_EINVAL, "%s: null pointer", who);
  DR_REQUIRE(aligned16(state), DR_EINVAL, "%s: the state arena is not 16-B aligned", who);
  WideBags bags{};
  bags.n = n_bags;
  if (n_bags) DR_REQUIRE(bag_slots && bag_ids && bag_splits, DR_EINVAL, "%s: null bag arrays", who);
  for (int i = 0; i < n_bags; ++i) {
    DR_REQUIRE(bag_slots[i] >= 0 && bag_slots[i] < S && bag_splits[i] && (bag_ids[i] || B == 0), DR_EINVAL,
               "%s: bag %d: slot %d outside [0, %d) or null arrays", who, i, bag_slots[i], S);
    bags.slot[i] = bag_slots[i];
    bags.ids[i] = bag_ids[i];
    bags.splits[i] = bag_splits[i];
  }
  if (B == 0 && MODE != kWideFtrl) return DR_OK;
  int lpe = 4;
  while (lpe < S && lpe < 32) lpe <<= 1;
  int64_t ctas = capped_grid(B, 256 / lpe, 8);
  if (ctas < 1) ctas = 1;   // dr_wide_ftrl at B = 0 still updates the bias record
  return with_lpr<32, 4>(lpe, [&](auto L) {
    wide_kernel<MODE, L><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(state, total_rows, rows, slot_offsets, ids, B,
                                                                          S, bags, g_logit, logit, p);
    DR_CUDA_LAUNCH_CHECK(who);
    return DR_OK;
  });
}

}  // namespace dr

using namespace dr;

extern "C" int dr_wide_fwd(const float* state, int64_t total_rows, const int64_t* rows, const int64_t* slot_offsets,
                           const int64_t* ids, int64_t B, int S, int n_bags, const int* bag_slots,
                           const int64_t* const* bag_ids, const int64_t* const* bag_splits, float* logit,
                           void* stream) {
  DR_REQUIRE(logit || B == 0, DR_EINVAL, "dr_wide_fwd: null logit");
  return wide_launch<kWideFwd>(const_cast<float*>(state), total_rows, rows, slot_offsets, ids, B, S, n_bags, bag_slots,
                               bag_ids, bag_splits, nullptr, logit, FtrlParams{1.f, 0.f, 0.f}, "dr_wide_fwd", stream);
}

extern "C" int dr_wide_bwd(float* state, int64_t total_rows, const int64_t* rows, const int64_t* slot_offsets,
                           const int64_t* ids, int64_t B, int S, int n_bags, const int* bag_slots,
                           const int64_t* const* bag_ids, const int64_t* const* bag_splits, const float* g_logit,
                           void* stream) {
  DR_REQUIRE(g_logit || B == 0, DR_EINVAL, "dr_wide_bwd: null g_logit");
  return wide_launch<kWideBwd>(state, total_rows, rows, slot_offsets, ids, B, S, n_bags, bag_slots, bag_ids,
                               bag_splits, g_logit, nullptr, FtrlParams{1.f, 0.f, 0.f}, "dr_wide_bwd", stream);
}

extern "C" int dr_wide_ftrl(float* state, int64_t total_rows, const int64_t* rows, const int64_t* slot_offsets,
                            const int64_t* ids, int64_t B, int S, int n_bags, const int* bag_slots,
                            const int64_t* const* bag_ids, const int64_t* const* bag_splits, float lr, float l1,
                            float l2, void* stream) {
  DR_REQUIRE(lr > 0.f && l1 >= 0.f && l2 >= 0.f, DR_EINVAL, "dr_wide_ftrl: lr=%g l1=%g l2=%g (need lr > 0, l1, l2 >= 0)",
             (double)lr, (double)l1, (double)l2);
  return wide_launch<kWideFtrl>(state, total_rows, rows, slot_offsets, ids, B, S, n_bags, bag_slots, bag_ids,
                                bag_splits, nullptr, nullptr, FtrlParams{lr, l1, 2.f * l2}, "dr_wide_ftrl", stream);
}
