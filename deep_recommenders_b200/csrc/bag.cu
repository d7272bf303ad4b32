// SURVEY.md 8(f) #2 -- multi-valued categorical slot ("Genres" is a VarLenFeature: movielens.py:122).
//   embedding_column(c, D)  ->  safe_embedding_lookup_sparse(ids, combiner="mean"): ids < 0 (out-of-vocabulary)
//                               are pruned, the rest averaged; a bag with no valid id gives the zero vector.
//   indicator_column(c)     ->  multi-hot COUNT vector, so the first-order term is sum_j w[id_j]  (combiner
//                               "sum", D = 1).
// Ragged layout: ids [nnz] (int64 / int32) + row_splits [B+1] (int64), bag b = ids[row_splits[b], row_splits[b+1]).
// HBM-bound like the single-valued gather: a lane group owns one bag, each lane one 16-B chunk of the row
// (scalar lanes when D % 4 != 0), ids are broadcast loads, rows are LDG.128 that do not allocate in L1.
#include "common.cuh"

namespace dr {

// TF divides the weighted sum by sum(w) (mean) or sqrt(sum(w^2)) (sqrtn), w = 1: keep a true division.
__device__ __forceinline__ float bag_den(int combiner, int cnt) {
  if (combiner == DR_COMBINER_MEAN) return (float)cnt;
  if (combiner == DR_COMBINER_SQRTN) return sqrtf((float)cnt);
  return 1.f;
}

template <typename IdT, int VEC>
__global__ void __launch_bounds__(256) embed_bag_fwd_kernel(const float* __restrict__ table, int64_t rows,
                                                             int64_t row_stride, const IdT* __restrict__ ids,
                                                             const int64_t* __restrict__ splits, int64_t B, int D,
                                                             int combiner, int group, float* __restrict__ out, int64_t out_stride) {
  const int chunks = D / VEC;
  const int bags_per_block = blockDim.x / group;
  const int g = threadIdx.x / group, c0 = threadIdx.x % group;
  for (int64_t b = (int64_t)blockIdx.x * bags_per_block + g; b < B; b += (int64_t)gridDim.x * bags_per_block) {
    const int64_t beg = __ldg(splits + b), end = __ldg(splits + b + 1);
    for (int c = c0; c < chunks; c += group) {
      float acc[VEC];
#pragma unroll
      for (int e = 0; e < VEC; ++e) acc[e] = 0.f;
      int cnt = 0;
      for (int64_t j = beg; j < end; ++j) {
        const int64_t id = (int64_t)__ldg(ids + j);
        if (id < 0 || id >= rows) continue;
        ++cnt;
        const float* src = table + (size_t)id * row_stride + (size_t)c * VEC;
        if (VEC == 4) {
          const float4 r = ldg_nc_na(src);
          acc[0] += r.x; acc[1 % VEC] += r.y; acc[2 % VEC] += r.z; acc[3 % VEC] += r.w;
        } else {
          acc[0] += __ldg(src);
        }
      }
      const float den = cnt > 0 ? bag_den(combiner, cnt) : 1.f;   // cnt == 0: acc is all zeros
      float* dst = out + (size_t)b * out_stride + (size_t)c * VEC;
      if (VEC == 4) stg4(dst, make_float4(acc[0] / den, acc[1 % VEC] / den, acc[2 % VEC] / den, acc[3 % VEC] / den));
      else dst[0] = acc[0] / den;
    }
  }
}

// grad_table[id_j] += scale * g_out[b] / den(b)   for every valid id of bag b (duplicates accumulate).
template <typename IdT, int VEC>
__global__ void __launch_bounds__(256) embed_bag_bwd_kernel(const IdT* __restrict__ ids,
                                                             const int64_t* __restrict__ splits, int64_t B, int D,
                                                             int combiner, int group, const float* __restrict__ g_out,
                                                             int64_t g_stride, int64_t rows, int64_t row_stride,
                                                             float* __restrict__ grad_table, float scale) {
  const int chunks = D / VEC;
  const int bags_per_block = blockDim.x / group;
  const int g = threadIdx.x / group, c0 = threadIdx.x % group;
  for (int64_t b = (int64_t)blockIdx.x * bags_per_block + g; b < B; b += (int64_t)gridDim.x * bags_per_block) {
    const int64_t beg = __ldg(splits + b), end = __ldg(splits + b + 1);
    int cnt = 0;
    for (int64_t j = beg; j < end; ++j) {
      const int64_t id = (int64_t)__ldg(ids + j);
      cnt += (id >= 0 && id < rows) ? 1 : 0;
    }
    if (cnt == 0) continue;
    const float den = bag_den(combiner, cnt);
    for (int c = c0; c < chunks; c += group) {
      const float* gsrc = g_out + (size_t)b * g_stride + (size_t)c * VEC;
      float4 gv = f4_zero();
      if (VEC == 4) {
        gv = ldg4(gsrc);
        gv = make_float4(gv.x / den * scale, gv.y / den * scale, gv.z / den * scale, gv.w / den * scale);
      } else {
        gv.x = __ldg(gsrc) / den * scale;
      }
      for (int64_t j = beg; j < end; ++j) {
        const int64_t id = (int64_t)__ldg(ids + j);
        if (id < 0 || id >= rows) continue;
        float* dst = grad_table + (size_t)id * row_stride + (size_t)c * VEC;
        if (VEC == 4) red_add_v4(dst, gv);
        else red_add_f32(dst, gv.x);
      }
    }
  }
}

static inline int bag_group(int chunks) {
  int g = 1;
  while (g < chunks && g < 32) g <<= 1;
  return g;
}

}  // namespace dr

using namespace dr;

static int bag_check(const char* fn, const void* ids, int id_bytes, const int64_t* splits, int64_t B, int D,
                     int combiner, int64_t rows, int64_t row_stride) {
  DR_REQUIRE(B >= 0, DR_EINVAL, "%s: B=%lld < 0", fn, (long long)B);
  DR_REQUIRE(D >= 1 && D <= 1024, DR_EINVAL, "%s: D=%d outside [1,1024]", fn, D);
  DR_REQUIRE(rows >= 1 && row_stride >= D, DR_EINVAL, "%s: rows=%lld row_stride=%lld (need >= D=%d)", fn,
             (long long)rows, (long long)row_stride, D);
  DR_REQUIRE(id_bytes == 8 || id_bytes == 4, DR_EINVAL, "%s: id_bytes=%d (need 4 or 8)", fn, id_bytes);
  DR_REQUIRE(combiner == DR_COMBINER_SUM || combiner == DR_COMBINER_MEAN || combiner == DR_COMBINER_SQRTN,
             DR_EINVAL, "%s: combiner=%d", fn, combiner);
  if (B > 0) DR_REQUIRE(splits && ids, DR_EINVAL, "%s: null ids / row_splits", fn);
  return DR_OK;
}

extern "C" int dr_embed_bag_fwd(const float* table, int64_t rows, int64_t row_stride, const void* ids, int id_bytes,
                                const int64_t* row_splits, int64_t B, int D, int combiner, float* out,
                                int64_t out_stride, void* stream) {
  if (int rc = bag_check("dr_embed_bag_fwd", ids, id_bytes, row_splits, B, D, combiner, rows, row_stride)) return rc;
  if (B == 0) return DR_OK;
  DR_REQUIRE(table && out, DR_EINVAL, "dr_embed_bag_fwd: null table / out");
  DR_REQUIRE(out_stride >= D, DR_EINVAL, "dr_embed_bag_fwd: out_stride=%lld < D=%d", (long long)out_stride, D);
  const bool vec = (D % 4 == 0) && (row_stride % 4 == 0) && (out_stride % 4 == 0) && aligned16(table) && aligned16(out);
  const int group = bag_group(vec ? D / 4 : D);
  const int64_t ctas = capped_grid(B, 256 / group, 16);
  return with_id_type(id_bytes, [&](auto id) {
    using IdT = decltype(id);
    auto k = vec ? embed_bag_fwd_kernel<IdT, 4> : embed_bag_fwd_kernel<IdT, 1>;
    k<<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(table, rows, row_stride, (const IdT*)ids, row_splits, B, D,
                                                        combiner, group, out, out_stride);
    DR_CUDA_LAUNCH_CHECK("embed_bag_fwd");
    return DR_OK;
  });
}

extern "C" int dr_embed_bag_bwd(const void* ids, int id_bytes, const int64_t* row_splits, int64_t B, int D,
                                int combiner, const float* g_out, int64_t g_stride, int64_t rows,
                                int64_t row_stride, float* grad_table, float scale, void* stream) {
  if (int rc = bag_check("dr_embed_bag_bwd", ids, id_bytes, row_splits, B, D, combiner, rows, row_stride)) return rc;
  if (B == 0) return DR_OK;
  DR_REQUIRE(g_out && grad_table, DR_EINVAL, "dr_embed_bag_bwd: null g_out / grad_table");
  DR_REQUIRE(g_stride >= D, DR_EINVAL, "dr_embed_bag_bwd: g_stride=%lld < D=%d", (long long)g_stride, D);
  const bool vec = (D % 4 == 0) && (row_stride % 4 == 0) && (g_stride % 4 == 0) && aligned16(grad_table) && aligned16(g_out);
  const int group = bag_group(vec ? D / 4 : D);
  const int64_t ctas = capped_grid(B, 256 / group, 16);
  return with_id_type(id_bytes, [&](auto id) {
    using IdT = decltype(id);
    auto k = vec ? embed_bag_bwd_kernel<IdT, 4> : embed_bag_bwd_kernel<IdT, 1>;
    k<<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>((const IdT*)ids, row_splits, B, D, combiner, group, g_out,
                                                        g_stride, rows, row_stride, grad_table, scale);
    DR_CUDA_LAUNCH_CHECK("embed_bag_bwd");
    return DR_OK;
  });
}
