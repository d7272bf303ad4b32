// The input row of FNN's tower (reference estimator/models/ranking/fnn.py:53-82), concat([bias, w_1 .. w_S, e_1 .. e_S])
// with one first-order scalar w_s and one embedding e_s per field, gathered in ONE pass over the embedding arena.
//
// Row layout, P = round_up(1 + S, 4), ld = P + S*D:
//   column 0                 the FM bias (read on the device: no host sync)
//   columns 1 .. S           w_s
//   columns 1+S .. P-1       zero
//   columns [P + s*D, P + (s+1)*D)   e_s
// The pad sits between the scalars and the embeddings so that every embedding segment starts 16-B aligned (vector
// stores) and ld is a multiple of 4, which the tensor-core GEMM of the tower's first layer needs for its operand
// (gemm_tc_eligible).  The first layer's kernel carries zero rows at the pad columns.
//
// Mapping: a lane group of LPR lanes (the power of two >= D/4) owns one lookup (example b, slot s): lane c reads
// the 16-B chunk c of the row, lane 0 also the first-order weight -- in the fused layout (DR_EMBED_LIN_IN_ROW) a
// scalar load of float D of the same 128-B line, issued right behind its chunk load, in the split layout a load from
// lin_ptrs[s].  Lookups are numbered i = b*S + s, so a warp's lookups are consecutive ids of the [B, S] matrix and
// consecutive output segments.  The lookup of slot 0 also writes the bias and the zero pad of its row.
// An id that is negative or >= rows[s] gives a zero embedding and a zero w (as dr_embed_fm_fwd).
//
// Backward: the same mapping reads g_x's embedding chunk and w column of every lookup and scatter-adds scale * g into
// the looked-up row (vector red.global.add) and its first-order weight (scalar red).  Column 0 and the pad are not
// read: the bias is a constant of the model.  Float atomics: the last bits depend on the order of duplicate ids.
#include "common.cuh"

namespace dr {

struct FnnParams {
  const float* const* table_ptrs;
  const float* const* lin_ptrs;
  const int64_t* rows;
  const void* ids;
  const float* bias;
  float* out;                        // forward: [B, ld]
  const float* g_x;                  // backward: [B, ld]
  float* const* grad_table_ptrs;
  float* const* grad_lin_ptrs;
  float scale;
  uint32_t n;                        // B * S lookups (< 2^31)
  int S, D, P;
  int64_t ld, row_stride, lin_stride;
  int lin_in_row;
};

template <int LPR, typename IdT, int U>
__global__ void __launch_bounds__(256) fnn_input_fwd_kernel(const FnnParams p) {
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31, c = lane % LPR, grp = lane / LPR;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const uint32_t S = (uint32_t)p.S;
  const int D = p.D, P = p.P;
  const bool chunk_ok = c * 4 < D;
  const IdT* __restrict__ ids = reinterpret_cast<const IdT*>(p.ids);
  const float bias = __ldg(p.bias);

  for (int64_t t0 = warp * (G * U); t0 < p.n; t0 += nwarps * (G * U)) {   // trip count is warp-uniform
    float4 v[U];
    float w[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = t0 + u * G + grp;
      v[u] = f4_zero();
      w[u] = 0.f;
      if (i < p.n) {
        const uint32_t s = (uint32_t)i % S;
        const int64_t id = (int64_t)__ldg(ids + i);
        if ((uint64_t)id < (uint64_t)__ldg(p.rows + s)) {
          const float* rowp = p.table_ptrs[s] + (size_t)id * p.row_stride;
          if (chunk_ok) v[u] = ldg_nc_na(rowp + c * 4);
          if (c == 0)
            w[u] = p.lin_in_row ? ldg_nc_na_f32(rowp + D) : __ldg(p.lin_ptrs[s] + (size_t)id * p.lin_stride);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = t0 + u * G + grp;
      if (i < p.n) {
        const uint32_t b = (uint32_t)i / S, s = (uint32_t)i - b * S;
        float* orow = p.out + (size_t)b * p.ld;
        if (chunk_ok) stg4(orow + P + (size_t)s * D + c * 4, v[u]);
        if (c == 0) {
          orow[1 + s] = w[u];
          if (s == 0) {
            orow[0] = bias;
            for (int j = 1 + (int)S; j < P; ++j) orow[j] = 0.f;
          }
        }
      }
    }
  }
}

template <int LPR, typename IdT, int U>
__global__ void __launch_bounds__(256) fnn_input_bwd_kernel(const FnnParams p) {
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31, c = lane % LPR, grp = lane / LPR;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const uint32_t S = (uint32_t)p.S;
  const int D = p.D, P = p.P;
  const bool chunk_ok = c * 4 < D;
  const IdT* __restrict__ ids = reinterpret_cast<const IdT*>(p.ids);
  const float sc = p.scale;

  for (int64_t t0 = warp * (G * U); t0 < p.n; t0 += nwarps * (G * U)) {
    float4 g[U];
    float gw[U];
    int64_t id[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = t0 + u * G + grp;
      g[u] = f4_zero();
      gw[u] = 0.f;
      id[u] = -1;
      if (i < p.n) {
        const uint32_t b = (uint32_t)i / S, s = (uint32_t)i - b * S;
        const int64_t r = (int64_t)__ldg(ids + i);
        if ((uint64_t)r < (uint64_t)__ldg(p.rows + s)) {
          id[u] = r;
          const float* grow = p.g_x + (size_t)b * p.ld;
          if (chunk_ok) g[u] = __ldg(reinterpret_cast<const float4*>(grow + P + (size_t)s * D + c * 4));
          if (c == 0) gw[u] = __ldg(grow + 1 + s);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (id[u] < 0) continue;
      const uint32_t s = (uint32_t)(t0 + u * G + grp) % S;
      float* rowp = p.grad_table_ptrs[s] + (size_t)id[u] * p.row_stride;
      if (chunk_ok) red_add_v4(rowp + c * 4, make_float4(sc * g[u].x, sc * g[u].y, sc * g[u].z, sc * g[u].w));
      if (c == 0)
        red_add_f32(p.lin_in_row ? rowp + D : p.grad_lin_ptrs[s] + (size_t)id[u] * p.lin_stride, sc * gw[u]);
    }
  }
}

template <bool BWD, int LPR, typename IdT>
static int fnn_launch(const FnnParams& p, cudaStream_t st) {
  constexpr int U = LPR <= 8 ? 8 : 4;
  constexpr int kThreads = 256, G = 32 / LPR;
  const int64_t tiles = ((int64_t)p.n + G * U - 1) / (G * U);
  const int64_t ctas = capped_grid(tiles, kThreads / 32, 2048 / kThreads);
  if (BWD) {
    fnn_input_bwd_kernel<LPR, IdT, U><<<(unsigned)ctas, kThreads, 0, st>>>(p);
    DR_CUDA_LAUNCH_CHECK("fnn_input_bwd");
  } else {
    fnn_input_fwd_kernel<LPR, IdT, U><<<(unsigned)ctas, kThreads, 0, st>>>(p);
    DR_CUDA_LAUNCH_CHECK("fnn_input_fwd");
  }
  return DR_OK;
}

// The checks both entries share; fills the geometry of p.
static int fnn_check(const char* fn, const float* const* table_ptrs, const float* const* lin_ptrs,
                     const int64_t* rows, const void* ids, int id_bytes, int64_t row_stride, int64_t lin_stride,
                     int flags, int64_t B, int S, int D, int64_t ld, const float* x, FnnParams& p) {
  DR_REQUIRE(table_ptrs && rows && ids && x, DR_EINVAL, "%s: null table pointers / rows / ids / row buffer", fn);
  if (int rc = check_lookup_dims(fn, B, S, D, id_bytes, ",")) return rc;
  const int P = (1 + S + 3) / 4 * 4;
  DR_REQUIRE(ld == P + (int64_t)S * D, DR_EINVAL, "%s: ld=%lld, the row layout needs P + S*D = %lld", fn,
             (long long)ld, (long long)(P + (int64_t)S * D));
  const int lin_in_row = (flags & DR_EMBED_LIN_IN_ROW) ? 1 : 0;
  DR_REQUIRE(flags == (flags & DR_EMBED_LIN_IN_ROW), DR_EINVAL, "%s: flags=%d (only DR_EMBED_LIN_IN_ROW)", fn, flags);
  if (row_stride == 0) row_stride = D;
  if (lin_stride == 0) lin_stride = 1;
  DR_REQUIRE(row_stride >= D && row_stride % 4 == 0, DR_EINVAL,
             "%s: row_stride=%lld must be >= D and a multiple of 4", fn, (long long)row_stride);
  DR_REQUIRE(!lin_in_row || (row_stride >= D + 4 && D <= 124), DR_EINVAL,
             "%s: DR_EMBED_LIN_IN_ROW needs row_stride >= D+4 and D <= 124", fn);
  DR_REQUIRE(lin_in_row || (lin_ptrs && lin_stride >= 1), DR_EINVAL,
             "%s: the split layout needs lin_ptrs and lin_stride >= 1", fn);
  DR_REQUIRE(aligned16(x), DR_EALIGN, "%s: the [B, ld] row buffer is not 16-B aligned", fn);
  DR_REQUIRE(B * (int64_t)S < ((int64_t)1 << 31), DR_ENOTSUP, "%s: B*S=%lld >= 2^31 lookups", fn,
             (long long)(B * (int64_t)S));
  p.table_ptrs = table_ptrs; p.lin_ptrs = lin_ptrs; p.rows = rows; p.ids = ids;
  p.n = (uint32_t)(B * S); p.S = S; p.D = D; p.P = P;
  p.ld = ld; p.row_stride = row_stride; p.lin_stride = lin_stride; p.lin_in_row = lin_in_row;
  return DR_OK;
}

}  // namespace dr

using namespace dr;

extern "C" int dr_fnn_input_fwd(const float* const* table_ptrs, const float* const* lin_ptrs, const int64_t* rows,
                                const void* ids, int id_bytes, int64_t row_stride, int64_t lin_stride, int flags,
                                const float* bias, int64_t B, int S, int D, int64_t ld, float* out, void* stream) {
  FnnParams p{};
  if (int rc = fnn_check("dr_fnn_input_fwd", table_ptrs, lin_ptrs, rows, ids, id_bytes, row_stride, lin_stride, flags,
                         B, S, D, ld, out, p))
    return rc;
  DR_REQUIRE(bias, DR_EINVAL, "dr_fnn_input_fwd: null bias");
  if (B == 0) return DR_OK;
  p.bias = bias; p.out = out;
  return with_lpr_id(lanes_per_row(D / 4), id_bytes, [&](auto L, auto id) {
    return fnn_launch<false, L, decltype(id)>(p, (cudaStream_t)stream);
  });
}

extern "C" int dr_fnn_input_bwd(const void* ids, int id_bytes, const int64_t* rows, const float* g_x, int64_t B,
                                int S, int D, int64_t ld, int64_t row_stride, int64_t lin_stride, int flags,
                                float* const* grad_table_ptrs, float* const* grad_lin_ptrs, float scale,
                                void* stream) {
  FnnParams p{};
  if (int rc = fnn_check("dr_fnn_input_bwd", grad_table_ptrs, grad_lin_ptrs, rows, ids, id_bytes, row_stride,
                         lin_stride, flags, B, S, D, ld, g_x, p))
    return rc;
  if (B == 0) return DR_OK;
  p.g_x = g_x; p.grad_table_ptrs = grad_table_ptrs; p.grad_lin_ptrs = grad_lin_ptrs; p.scale = scale;
  return with_lpr_id(lanes_per_row(D / 4), id_bytes, [&](auto L, auto id) {
    return fnn_launch<true, L, decltype(id)>(p, (cudaStream_t)stream);
  });
}
