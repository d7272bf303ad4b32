// Variant 0 of the fp32 GEMM core: FFMA register-tiled kernel (see gemm.cuh).
#include "gemm.cuh"
#include <float.h>

namespace dr {

int g_tune_gemm_variant = 2;   // library default = the shipped core (wgmma 3xTF32, split in kernel; needs no workspace); 0 = FFMA, 1 = pre-split planes
int g_tune_gemm_splitk = 0;   // 0 = heuristic

__device__ __forceinline__ float4 load4_guard(const float* __restrict__ base, int64_t r, int64_t c,
                                              int64_t ld, int64_t R, int64_t Cn, bool vec_ok) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (r >= R || c >= Cn) return v;
  const float* p = base + r * ld + c;
  if (vec_ok && c + 3 < Cn) return *reinterpret_cast<const float4*>(p);
  v.x = __ldg(p);
  if (c + 1 < Cn) v.y = __ldg(p + 1);
  if (c + 2 < Cn) v.z = __ldg(p + 2);
  if (c + 3 < Cn) v.w = __ldg(p + 3);
  return v;
}

__device__ __forceinline__ float epi_scalar(const GemmArgs& a, float acc, int64_t m, int64_t n) {
  const int64_t off = m * a.ldc + n;
  switch (a.epi) {
    case EPI_BIAS_ACT: return act_apply(acc + (a.bias ? __ldg(a.bias + n) : 0.f), a.act);
    case EPI_ACTGRAD: return acc * act_grad_from_y(__ldg(a.aux0 + off), a.act);
    case EPI_CROSS: {
      const float x = __ldg(a.aux1 + off);
      float u = acc + (a.bias ? __ldg(a.bias + n) : 0.f);
      if (a.alpha != 0.f) u = u + a.alpha * x;
      if (a.out2) a.out2[off] = u;
      return __ldg(a.aux0 + off) * u + x;
    }
    case EPI_CROSS_DX: {
      float v = acc + __ldg(a.aux1 + off);
      if (a.alpha != 0.f) v += a.alpha * __ldg(a.aux0 + off);
      return v;
    }
    case EPI_SCORES: {
      float v = acc;
      if (a.bias) v = v - logf(__ldg(a.bias + n));
      if (a.cand_ids && m + a.row0 != n && m + a.row0 < a.N && __ldg(a.cand_ids + n) == __ldg(a.cand_ids + m + a.row0))
        v = v + (-FLT_MAX / 100.0f);
      return v;
    }
    default: return acc;
  }
}

// ACC (EPI_CROSS_DX_ACC) is a compile-time form with kernels of its own (sgemm_acc_kernel), so that the kernels of every
// other epilogue compile exactly as they do without it.
template <int BM, int BN, int BK, int TM, int TN, bool TA, bool TB, bool ACC>
__device__ __forceinline__ void sgemm_body(const GemmArgs& a) {
  constexpr int NT = 256;
  constexpr int TX = BN / TN, TY = BM / TM;
  static_assert(TX * TY == NT, "thread tile mismatch");
  constexpr int VM = TM >= 4 ? 4 : TM, NVM = TM / VM;
  constexpr int VN = TN >= 4 ? 4 : TN, NVN = TN / VN;
  constexpr int LDA_S = BM + 4, LDB_S = BN + 4;
  __shared__ __align__(16) float As[2][BK][LDA_S];
  __shared__ __align__(16) float Bs[2][BK][LDB_S];

  const int t = threadIdx.x;
  const int tx = t % TX, ty = t / TX;
  const int64_t m0 = (int64_t)blockIdx.x * BM;
  const int64_t n0 = (int64_t)blockIdx.y * BN;

  // split-K range (multiples of BK)
  const int64_t ktiles = (a.K + BK - 1) / BK;
  const int64_t per = (ktiles + a.splitk - 1) / a.splitk;
  const int64_t kt0 = (int64_t)blockIdx.z * per;
  const int64_t kt1 = min(ktiles, kt0 + per);
  if (kt0 >= kt1) return;

  const bool vecA = ((a.lda & 3) == 0) && aligned16(a.A);
  const bool vecB = ((a.ldb & 3) == 0) && aligned16(a.B);

  constexpr int FA = BM * BK / 4;             // float4 per A tile
  constexpr int FB = BK * BN / 4;
  constexpr int LA = (FA + NT - 1) / NT;
  constexpr int LB = (FB + NT - 1) / NT;
  float4 ra[LA], rb[LB];

  auto gload = [&](int64_t kt) {
    const int64_t k0 = kt * BK;
#pragma unroll
    for (int i = 0; i < LA; ++i) {
      const int f = t + i * NT;
      if (FA % NT == 0 || f < FA) {
        if (!TA) {
          const int row = f / (BK / 4), kq = f % (BK / 4);
          ra[i] = load4_guard(a.A, m0 + row, k0 + kq * 4, a.lda, a.M, a.K, vecA);
        } else {
          const int kk = f / (BM / 4), mq = f % (BM / 4);
          ra[i] = load4_guard(a.A, k0 + kk, m0 + mq * 4, a.lda, a.K, a.M, vecA);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < LB; ++i) {
      const int f = t + i * NT;
      if (FB % NT == 0 || f < FB) {
        if (!TB) {
          const int kk = f / (BN / 4), nq = f % (BN / 4);
          rb[i] = load4_guard(a.B, k0 + kk, n0 + nq * 4, a.ldb, a.K, a.N, vecB);
        } else {
          const int n = f / (BK / 4), kq = f % (BK / 4);
          rb[i] = load4_guard(a.B, n0 + n, k0 + kq * 4, a.ldb, a.N, a.K, vecB);
        }
      }
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < LA; ++i) {
      const int f = t + i * NT;
      if (FA % NT == 0 || f < FA) {
        if (!TA) {
          const int row = f / (BK / 4), kq = f % (BK / 4);
          As[buf][kq * 4 + 0][row] = ra[i].x;
          As[buf][kq * 4 + 1][row] = ra[i].y;
          As[buf][kq * 4 + 2][row] = ra[i].z;
          As[buf][kq * 4 + 3][row] = ra[i].w;
        } else {
          const int kk = f / (BM / 4), mq = f % (BM / 4);
          *reinterpret_cast<float4*>(&As[buf][kk][mq * 4]) = ra[i];
        }
      }
    }
#pragma unroll
    for (int i = 0; i < LB; ++i) {
      const int f = t + i * NT;
      if (FB % NT == 0 || f < FB) {
        if (!TB) {
          const int kk = f / (BN / 4), nq = f % (BN / 4);
          *reinterpret_cast<float4*>(&Bs[buf][kk][nq * 4]) = rb[i];
        } else {
          const int n = f / (BK / 4), kq = f % (BK / 4);
          Bs[buf][kq * 4 + 0][n] = rb[i].x;
          Bs[buf][kq * 4 + 1][n] = rb[i].y;
          Bs[buf][kq * 4 + 2][n] = rb[i].z;
          Bs[buf][kq * 4 + 3][n] = rb[i].w;
        }
      }
    }
  };

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  gload(kt0);
  sstore(0);
  __syncthreads();

  int buf = 0;
  for (int64_t kt = kt0; kt < kt1; ++kt) {
    const bool more = (kt + 1) < kt1;
    if (more) gload(kt + 1);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float av[TM], bv[TN];
#pragma unroll
      for (int v = 0; v < NVM; ++v) {
        const float* p = &As[buf][kk][v * (BM / NVM) + ty * VM];
        if (VM == 4) {
          const float4 q = *reinterpret_cast<const float4*>(p);
          av[v * VM + 0] = q.x; av[v * VM + 1] = q.y; av[v * VM + 2] = q.z; av[v * VM + 3] = q.w;
        } else {
#pragma unroll
          for (int e = 0; e < VM; ++e) av[v * VM + e] = p[e];
        }
      }
#pragma unroll
      for (int v = 0; v < NVN; ++v) {
        const float* p = &Bs[buf][kk][v * (BN / NVN) + tx * VN];
        if (VN == 4) {
          const float4 q = *reinterpret_cast<const float4*>(p);
          bv[v * VN + 0] = q.x; bv[v * VN + 1] = q.y; bv[v * VN + 2] = q.z; bv[v * VN + 3] = q.w;
        } else {
#pragma unroll
          for (int e = 0; e < VN; ++e) bv[v * VN + e] = p[e];
        }
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (more) {
      sstore(buf ^ 1);
      __syncthreads();
      buf ^= 1;
    }
  }

  // ---- epilogue -------------------------------------------------------------------------
  const bool vecC = ((a.ldc & 3) == 0) && aligned16(a.C) && (a.epi == EPI_STORE || a.epi == EPI_BIAS_ACT);
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int64_t m = m0 + (i / VM) * (BM / NVM) + ty * VM + (i % VM);
    if (m >= a.M) continue;
#pragma unroll
    for (int v = 0; v < NVN; ++v) {
      const int64_t n = n0 + v * (BN / NVN) + tx * VN;
      if (n >= a.N) continue;
      if constexpr (ACC) {
#pragma unroll
        for (int e = 0; e < VN; ++e)
          if (n + e < a.N) {
            const int64_t off = m * a.ldc + n + e;
            a.C[off] += acc[i][v * VN + e] + a.alpha * __ldg(a.aux0 + off) + __ldg(a.aux1 + off);
          }
      } else if (a.epi == EPI_ATOMIC) {
#pragma unroll
        for (int e = 0; e < VN; ++e)
          if (n + e < a.N) red_add_f32(a.C + m * a.ldc + n + e, acc[i][v * VN + e]);
      } else if (VN == 4 && vecC && n + 3 < a.N) {
        float4 o;
        o.x = epi_scalar(a, acc[i][v * VN + 0], m, n + 0);
        o.y = epi_scalar(a, acc[i][v * VN + 1], m, n + 1);
        o.z = epi_scalar(a, acc[i][v * VN + 2], m, n + 2);
        o.w = epi_scalar(a, acc[i][v * VN + 3], m, n + 3);
        *reinterpret_cast<float4*>(a.C + m * a.ldc + n) = o;
      } else {
#pragma unroll
        for (int e = 0; e < VN; ++e)
          if (n + e < a.N) a.C[m * a.ldc + n + e] = epi_scalar(a, acc[i][v * VN + e], m, n + e);
      }
    }
  }
}

template <int BM, int BN, int BK, int TM, int TN, bool TA, bool TB>
__global__ void __launch_bounds__(256) sgemm_kernel(const GemmArgs a) {
  sgemm_body<BM, BN, BK, TM, TN, TA, TB, false>(a);
}

// EPI_CROSS_DX_ACC: the only GEMM that accumulates into C is the Cross input gradient h @ W^T (A as stored, B transposed).
template <int BM, int BN, int BK, int TM, int TN>
__global__ void __launch_bounds__(256) sgemm_acc_kernel(const GemmArgs a) {
  sgemm_body<BM, BN, BK, TM, TN, false, true, true>(a);
}

template <int BM, int BN, int BK, int TM, int TN>
static int launch_cfg(const GemmArgs& a, bool ta, bool tb, cudaStream_t st) {
  dim3 grid((unsigned)((a.M + BM - 1) / BM), (unsigned)((a.N + BN - 1) / BN), (unsigned)a.splitk);
  if (a.epi == EPI_CROSS_DX_ACC) {
    DR_REQUIRE(!ta && tb, DR_ENOTSUP, "gemm: the accumulating Cross epilogue serves A as stored, B transposed only");
    sgemm_acc_kernel<BM, BN, BK, TM, TN><<<grid, 256, 0, st>>>(a);
  } else if (!ta && !tb) sgemm_kernel<BM, BN, BK, TM, TN, false, false><<<grid, 256, 0, st>>>(a);
  else if (!ta && tb) sgemm_kernel<BM, BN, BK, TM, TN, false, true><<<grid, 256, 0, st>>>(a);
  else if (ta && !tb) sgemm_kernel<BM, BN, BK, TM, TN, true, false><<<grid, 256, 0, st>>>(a);
  else sgemm_kernel<BM, BN, BK, TM, TN, true, true><<<grid, 256, 0, st>>>(a);
  DR_CUDA_LAUNCH_CHECK("sgemm");
  return DR_OK;
}

int gemm_launch(const GemmArgs& a0, bool ta, bool tb, cudaStream_t st) {
  GemmArgs a = a0;
  DR_REQUIRE(a.A && a.B && a.C, DR_EINVAL, "gemm: null operand");
  DR_REQUIRE(a.M >= 0 && a.N >= 1 && a.K >= 1, DR_EINVAL, "gemm: bad shape M=%lld N=%lld K=%lld",
             (long long)a.M, (long long)a.N, (long long)a.K);
  if (a.M == 0) return DR_OK;
  if (a.splitk < 1) a.splitk = 1;
  DR_REQUIRE(a.splitk == 1 || a.epi == EPI_ATOMIC, DR_EINVAL, "gemm: split-K needs the atomic epilogue");
  DR_REQUIRE((a.N + 15) / 16 <= 65535, DR_EINVAL, "gemm: N=%lld too large for grid.y", (long long)a.N);
  if (gemm_tc_eligible(a, ta, tb)) return gemm_tc_launch(a, ta, tb, st);
  const int64_t ktiles = (a.K + 15) / 16;
  if (a.splitk > ktiles) a.splitk = (int)ktiles;
  if (a.N > 64) return launch_cfg<128, 128, 16, 8, 8>(a, ta, tb, st);
  if (a.N > 16) return launch_cfg<128, 32, 16, 8, 2>(a, ta, tb, st);
  return launch_cfg<256, 16, 16, 8, 2>(a, ta, tb, st);
}

}  // namespace dr
