// Sparse (CSR) times dense product with a fused bias / activation / residual epilogue: the GCN layer's aggregation.
//   keras/models/retrieval/gcn.py:45-55 (tf.sparse.sparse_dense_matmul(adj, features), then the Dense and the residual
//   add).  The backward is the same product with A^T (a transposed CSR the caller builds once per adjacency).
//
// y[r, :] = act(sum_{p in row r} values[p] * x[indices[p], :] + bias)   out = y + residual   (both optional)
// Ownership: a group of G lanes (G a power of two, <= 32) owns one output row; narrow rows pack 32 / G rows into a
// warp.  The group loads G (index, value) pairs at a time, one per lane, and broadcasts each with a shuffle.  Lanes span
// the columns, V = 4 floats per access (16-byte loads) when every row is 16-byte aligned, else V = 1; a lane holds NC
// such chunks, so one pass over the row's pairs covers G*V*NC columns, and wider rows take several passes.
// Summation: fp32 fmaf in ascending position within the row, one owner per output element: no atomics, and reruns
// are bit-identical.  A column index outside [0, n_cols) is skipped before any load.
#include "common.cuh"

#include <math.h>

namespace dr {

namespace {

constexpr int SPMM_THREADS = 256;
constexpr int SPMM_SOFTMAX_MAX_F = 1024;

template <int V>
__device__ __forceinline__ void spmm_load(const float* p, float (&v)[V]) {
  if constexpr (V == 4) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
    v[0] = __ldg(p);
  }
}

template <int V>
__device__ __forceinline__ void spmm_store(float* p, const float (&v)[V]) {
  if constexpr (V == 4) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    p[0] = v[0];
  }
}

template <int G>
__device__ __forceinline__ float spmm_group_max(float v, unsigned mask) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(mask, v, o, G));
  return v;
}

template <int G>
__device__ __forceinline__ float spmm_group_sum(float v, unsigned mask) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(mask, v, o, G);
  return v;
}

template <int G, int V, int NC>
__global__ void __launch_bounds__(SPMM_THREADS) spmm_csr_kernel(const int* __restrict__ indptr,
                                                                const int* __restrict__ indices,
                                                                const float* __restrict__ values, int n_rows,
                                                                int n_cols, const float* __restrict__ x, int F,
                                                                const float* __restrict__ bias,
                                                                const float* __restrict__ residual, int act,
                                                                float* __restrict__ y, float* __restrict__ out) {
  const int gl = threadIdx.x & (G - 1);
  const int row = blockIdx.x * (SPMM_THREADS / G) + threadIdx.x / G;
  if (row >= n_rows) return;                     // whole groups leave together: the shuffles below see full groups
  const unsigned gmask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << ((threadIdx.x & 31) & ~(G - 1)));
  const int p0 = __ldg(indptr + row), p1 = __ldg(indptr + row + 1);
  constexpr int TILE = G * V * NC;
  for (int c0 = 0; c0 < F; c0 += TILE) {
    float acc[NC][V];
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int e = 0; e < V; ++e) acc[c][e] = 0.f;
    for (int p = p0; p < p1; p += G) {
      int j = -1;
      float a = 0.f;
      if (p + gl < p1) {
        j = __ldg(indices + p + gl);
        a = __ldg(values + p + gl);
      }
      const int cnt = min(G, p1 - p);
      int k = 0;
      // two pairs per step: both rows' loads are issued before either's FMAs, which still run in position order
      for (; k + 1 < cnt; k += 2) {
        const int j0 = G == 1 ? j : __shfl_sync(gmask, j, k, G);
        const float a0 = G == 1 ? a : __shfl_sync(gmask, a, k, G);
        const int j1 = __shfl_sync(gmask, j, k + 1, G);
        const float a1 = __shfl_sync(gmask, a, k + 1, G);
        const bool ok0 = (unsigned)j0 < (unsigned)n_cols, ok1 = (unsigned)j1 < (unsigned)n_cols;
        float v0[NC][V], v1[NC][V];
#pragma unroll
        for (int c = 0; c < NC; ++c) {
          const int col = c0 + (c * G + gl) * V;
          if (ok0 && col < F) spmm_load<V>(x + (int64_t)j0 * F + col, v0[c]);
          if (ok1 && col < F) spmm_load<V>(x + (int64_t)j1 * F + col, v1[c]);
        }
#pragma unroll
        for (int c = 0; c < NC; ++c) {
          const int col = c0 + (c * G + gl) * V;
          if (col < F) {
#pragma unroll
            for (int e = 0; e < V; ++e) {
              if (ok0) acc[c][e] = fmaf(a0, v0[c][e], acc[c][e]);
              if (ok1) acc[c][e] = fmaf(a1, v1[c][e], acc[c][e]);
            }
          }
        }
      }
      if (k < cnt) {
        const int j0 = G == 1 ? j : __shfl_sync(gmask, j, k, G);
        const float a0 = G == 1 ? a : __shfl_sync(gmask, a, k, G);
        if ((unsigned)j0 < (unsigned)n_cols) {
#pragma unroll
          for (int c = 0; c < NC; ++c) {
            const int col = c0 + (c * G + gl) * V;
            if (col < F) {
              float v0[V];
              spmm_load<V>(x + (int64_t)j0 * F + col, v0);
#pragma unroll
              for (int e = 0; e < V; ++e) acc[c][e] = fmaf(a0, v0[e], acc[c][e]);
            }
          }
        }
      }
    }
    // epilogue: z = acc + bias, y = act(z) (softmax: the host guarantees one pass covers the row), out = y + residual
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const int col = c0 + (c * G + gl) * V;
      if (bias && col < F)
#pragma unroll
        for (int e = 0; e < V; ++e) acc[c][e] += __ldg(bias + col + e);
    }
    if (act == DR_ACT_SOFTMAX) {
      float m = -INFINITY;
#pragma unroll
      for (int c = 0; c < NC; ++c)
        if (c0 + (c * G + gl) * V < F)
#pragma unroll
          for (int e = 0; e < V; ++e) m = fmaxf(m, acc[c][e]);
      m = spmm_group_max<G>(m, gmask);
      float s = 0.f;
#pragma unroll
      for (int c = 0; c < NC; ++c)
        if (c0 + (c * G + gl) * V < F)
#pragma unroll
          for (int e = 0; e < V; ++e) {
            acc[c][e] = expf(acc[c][e] - m);
            s += acc[c][e];
          }
      s = spmm_group_sum<G>(s, gmask);
#pragma unroll
      for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int e = 0; e < V; ++e) acc[c][e] = acc[c][e] / s;
    } else {
#pragma unroll
      for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int e = 0; e < V; ++e) acc[c][e] = act_apply(acc[c][e], act);
    }
    const int64_t base = (int64_t)row * F;
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const int col = c0 + (c * G + gl) * V;
      if (col < F) {
        spmm_store<V>(y + base + col, acc[c]);
        if (residual) {
          float r[V];
          spmm_load<V>(residual + base + col, r);
#pragma unroll
          for (int e = 0; e < V; ++e) r[e] += acc[c][e];
          spmm_store<V>(out + base + col, r);
        }
      }
    }
  }
}

template <int G, int V, int NC>
int spmm_launch(const int* indptr, const int* indices, const float* values, int n_rows, int n_cols, const float* x,
                int F, const float* bias, const float* residual, int act, float* y, float* out, cudaStream_t st) {
  constexpr int rows_per_cta = SPMM_THREADS / G;
  const unsigned grid = (unsigned)((n_rows + rows_per_cta - 1) / rows_per_cta);
  spmm_csr_kernel<G, V, NC><<<grid, SPMM_THREADS, 0, st>>>(indptr, indices, values, n_rows, n_cols, x, F, bias,
                                                           residual, act, y, out);
  DR_CUDA_LAUNCH_CHECK("spmm_csr");
  return DR_OK;
}

// Lanes per row: the fewest (power of two) that cover the row in V-wide chunks, at most 32.  A 32-lane owner holds NC
// chunks per lane: enough to cover the row in one pass when the softmax needs that, else at most 8 (the pass repeats).
template <int V>
int spmm_dispatch(const int* indptr, const int* indices, const float* values, int n_rows, int n_cols, const float* x,
                  int F, const float* bias, const float* residual, int act, float* y, float* out, cudaStream_t st) {
  const int units = (F + V - 1) / V;
#define SPMM_ARGS indptr, indices, values, n_rows, n_cols, x, F, bias, residual, act, y, out, st
  if (units <= 1) return spmm_launch<1, V, 1>(SPMM_ARGS);
  if (units <= 2) return spmm_launch<2, V, 1>(SPMM_ARGS);
  if (units <= 4) return spmm_launch<4, V, 1>(SPMM_ARGS);
  if (units <= 8) return spmm_launch<8, V, 1>(SPMM_ARGS);
  if (units <= 16) return spmm_launch<16, V, 1>(SPMM_ARGS);
  const int per_lane = (units + 31) / 32;
  if (per_lane <= 1) return spmm_launch<32, V, 1>(SPMM_ARGS);
  if (per_lane <= 2) return spmm_launch<32, V, 2>(SPMM_ARGS);
  if (per_lane <= 4) return spmm_launch<32, V, 4>(SPMM_ARGS);
  if (per_lane <= 8 || act != DR_ACT_SOFTMAX) return spmm_launch<32, V, 8>(SPMM_ARGS);
  if constexpr (V == 1) {
    if (per_lane <= 16) return spmm_launch<32, 1, 16>(SPMM_ARGS);
    return spmm_launch<32, 1, 32>(SPMM_ARGS);
  }
#undef SPMM_ARGS
  set_error("dr_spmm_csr_fwd: no softmax kernel for F=%d", F);   // unreachable: F <= 1024 is checked first
  return DR_ENOTSUP;
}

}  // namespace

}  // namespace dr

using namespace dr;

extern "C" int dr_spmm_csr_fwd(const int* indptr, const int* indices, const float* values, int64_t n_rows,
                               int64_t n_cols, int64_t nnz, const float* x, int F, const float* bias,
                               const float* residual, int act, float* y, float* out, void* stream) {
  DR_REQUIRE(n_rows >= 0 && n_cols >= 0 && nnz >= 0 && F >= 1, DR_EINVAL,
             "dr_spmm_csr_fwd: bad shape n_rows=%lld n_cols=%lld nnz=%lld F=%d", (long long)n_rows, (long long)n_cols,
             (long long)nnz, F);
  const int64_t lim = (int64_t)1 << 31;
  DR_REQUIRE(n_rows < lim && n_cols < lim && nnz < lim, DR_ENOTSUP,
             "dr_spmm_csr_fwd: served for n_rows, n_cols, nnz < 2^31, got %lld, %lld, %lld", (long long)n_rows,
             (long long)n_cols, (long long)nnz);
  DR_REQUIRE((act >= DR_ACT_NONE && act <= DR_ACT_TANH) || act == DR_ACT_SOFTMAX, DR_EINVAL,
             "dr_spmm_csr_fwd: unknown activation %d", act);
  DR_REQUIRE(act != DR_ACT_SOFTMAX || F <= SPMM_SOFTMAX_MAX_F, DR_ENOTSUP,
             "dr_spmm_csr_fwd: the softmax epilogue is served for F <= %d, got F=%d", SPMM_SOFTMAX_MAX_F, F);
  DR_REQUIRE(!residual || out, DR_EINVAL, "dr_spmm_csr_fwd: a residual needs out");
  if (n_rows == 0) return DR_OK;
  DR_REQUIRE(indptr && y && (nnz == 0 || (indices && values)) && (nnz == 0 || n_cols == 0 || x), DR_EINVAL,
             "dr_spmm_csr_fwd: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const bool vec = (F & 3) == 0 && (!x || aligned16(x)) && aligned16(y) &&
                   (!residual || (aligned16(residual) && aligned16(out)));
  if (vec)
    return spmm_dispatch<4>(indptr, indices, values, (int)n_rows, (int)n_cols, x, F, bias, residual, act, y, out, st);
  return spmm_dispatch<1>(indptr, indices, values, (int)n_rows, (int)n_cols, x, F, bias, residual, act, y, out, st);
}
