// fp32 GEMM core shared by the Dense tower (row D), the Cross layer (row X) and the score
// matrix (row R).  C[M,N] = epilogue( sum_k A(m,k) * B(k,n) ).
//
// Precision: the parity bar is 1e-5 relative in fp32 (BASELINE.json north_star), which a
// single-pass TF32/BF16 tensor-core product cannot meet (SURVEY.md section 7, hard part 2).
// Variant 0 (this file) is an FFMA register-tiled kernel: 128x128x16 CTA tile, 8x8 per
// thread, global->register->shared double buffering.  Variant 1 (gemm_tc.cu, when built) is
// the wgmma 3xTF32 path; both share the epilogues below.
#pragma once
#include "common.cuh"

namespace dr {

enum Epi : int {
  EPI_STORE = 0,      // C = acc
  EPI_BIAS_ACT = 1,   // C = act(acc + bias[n])
  EPI_ATOMIC = 2,     // C += acc   (split-K; C pre-zeroed)
  EPI_ACTGRAD = 3,    // C = acc * act'(aux0[m,n])            aux0 = layer output y
  EPI_CROSS = 4,      // u = acc + bias[n] + alpha*aux1[m,n]; out2 = u; C = aux0*u + aux1  (aux0=x0, aux1=x)
  EPI_CROSS_DX = 5,   // C = acc + alpha*aux0[m,n] + aux1[m,n]    (aux0 = h, aux1 = g)
  EPI_SCORES = 6,     // C = acc - log(p[n]) + dup(m,n)*MIN_FLOAT  (bias = p or null, ids in aux ptr)
  EPI_CROSS_DX_ACC = 7,   // C += acc + alpha*aux0[m,n] + aux1[m,n]   (EPI_CROSS_DX accumulated into C; splitk == 1, so each
                          // element has one owner: a plain load-add-store, no reduction traffic, deterministic)
};

struct GemmArgs {
  const float* A;   // !TA: [M,K] row-major (lda) ; TA: stored [K,M] (lda)
  const float* B;   // !TB: [K,N] row-major (ldb) ; TB: stored [N,K] (ldb)
  float* C;         // [M,N] row-major (ldc)
  int64_t M, N, K;
  int64_t lda, ldb, ldc;
  int epi;
  int act;
  float alpha;
  const float* bias;
  const float* aux0;
  const float* aux1;
  float* out2;
  const int64_t* cand_ids;   // EPI_SCORES
  int64_t row0;              // EPI_SCORES: query row m of this call is global query m + row0 (its positive = candidate m + row0)
  int splitk;                // >= 1
  int stages;                // 0 = default depth of the raw operand ring (3); 2 = two stages (32 KB less shared memory)
  int share;                 // 1 = the GEMM runs beside a memory-bound kernel on another stream: same as stages = 2
};

extern int g_tune_gemm_variant;
extern int g_tune_gemm_splitk;

// C = A * B with the given storage flags; picks the tile shape from N. Returns DR_* / cudaError.
int gemm_launch(const GemmArgs& a, bool transA, bool transB, cudaStream_t st);

// wgmma 3xTF32 variants (gemm_tc.cu): g_tune_gemm_variant == 2 splits in the kernel; == 1 needs an aligned shape
// and a registered workspace (dr_set_workspace) that can hold the hi/lo operand planes.
bool gemm_tc_eligible(const GemmArgs& a, bool transA, bool transB);
int gemm_tc_launch(const GemmArgs& a, bool transA, bool transB, cudaStream_t st);

}  // namespace dr
