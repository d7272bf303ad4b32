// xDeepFM's Compressed Interaction Network layer (CIN), forward and backward.
//   keras/models/ranking/xdeepfm.py:71-96 (CIN.call); the backward is TensorFlow autodiff there.
//
// The reference materialises the outer product Z[b, d, i*h+j] = x0[b,i,d] * x[b,j,d] and runs a width-1 conv1d over it.
// Here every product is a GEMM whose K operand is generated on chip and never reaches global memory:
//   Khatri-Rao GEMM   out[b,k,d] = sum_{a,c} W[a*sa + c*sc + k*sk] * P[b,a,d] * Q[b,c,d]
//     forward  P = x0 (m), Q = x (h),  out = y   (M = H):  sa = h*H, sc = H,   sk = 1
//     gx0      P = x  (h), Q = G (H),  out = gx0 (M = m):  sa = H,   sc = 1,   sk = h*H
//     gx       P = x0 (m), Q = G (H),  out = gx  (M = h):  sa = h*H, sc = 1,   sk = H
//   W is read in place through the three strides (no permuted copy).  One CTA owns BM outputs x 128 columns, where a
//   column is one (example, d) pair and a tile holds whole examples (128 / D of them), so the sum pooling over d is a
//   fixed-order reduction inside the CTA.
//   weight gradient   gW[i*h+j, k] = sum_{b,d} x0[b,i,d] * x[b,j,d] * G[b,k,d]: the same tile loop with G as the A
//   operand and the x0 (x) x pair products as the generated B operand, split over the B*D columns with red.global.add.
// Arithmetic: fp32 FFMA, 16 x 16 threads with an (BM/16) x 8 register tile, K steps of 16 staged in shared memory
// through a register prefetch (two buffers, one barrier per step).
#include "common.cuh"

namespace dr {

namespace {

constexpr int CIN_BN = 128;       // columns per CTA tile
constexpr int CIN_BK = 16;        // contraction step
constexpr int CIN_THREADS = 256;
constexpr int CIN_MAX_FIELDS = 1024;
constexpr int CIN_MAX_D = CIN_BN;

// n / d and n % d for n < 2^32 with one 64-bit multiply: the estimate from ceil(2^32 / d) is q or q + 1.
struct FastDiv {
  uint32_t d;
  uint64_t m;
};
static FastDiv make_fastdiv(uint32_t d) { return FastDiv{d, ((1ull << 32) + d - 1) / d}; }
__device__ __forceinline__ void divmod(const FastDiv& f, uint32_t n, int& q, int& r) {
  uint32_t e = (uint32_t)(((uint64_t)n * f.m) >> 32);
  int rr = (int)(n - e * f.d);
  if (rr < 0) { --e; rr += (int)f.d; }
  q = (int)e;
  r = rr;
}

template <int BM>
struct CinSmem {
  static constexpr int LDA = BM + 4;           // padded: the k-fastest staging stores hit distinct banks
  static constexpr int LDB = CIN_BN + 4;
  union {
    struct {
      float a[2][CIN_BK][LDA];
      float b[2][CIN_BK][LDB];
    } k;
    float y[64][CIN_BN + 1];                   // epilogue: 64 output rows of the tile at a time
  };
};

// acc[TM][8] += A[kk][rows] x B[kk][cols] over one staged step.  Thread (ty, tx) owns rows ty*4 + 64*ii + e and
// columns tx*4 + 64*jj + f, read as float4 (conflict-free: a quarter warp reads 128 contiguous bytes).
template <int BM>
__device__ __forceinline__ void tile_fma(const float (*As)[BM + 4], const float (*Bs)[CIN_BN + 4],
                                         float (&acc)[BM / 16][8], int ty, int tx) {
  constexpr int TM = BM / 16;
#pragma unroll
  for (int kk = 0; kk < CIN_BK; ++kk) {
    float a[TM], b[8];
#pragma unroll
    for (int ii = 0; ii < TM / 4; ++ii) {
      const float4 v = *reinterpret_cast<const float4*>(&As[kk][ty * 4 + 64 * ii]);
      a[ii * 4 + 0] = v.x; a[ii * 4 + 1] = v.y; a[ii * 4 + 2] = v.z; a[ii * 4 + 3] = v.w;
    }
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      const float4 v = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4 + 64 * jj]);
      b[jj * 4 + 0] = v.x; b[jj * 4 + 1] = v.y; b[jj * 4 + 2] = v.z; b[jj * 4 + 3] = v.w;
    }
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
  }
}

struct KrArgs {
  const float* P;
  const float* Q;
  const float* W;
  const float* bias;    // [M] or NULL
  float* out;           // [B, M, D]
  float* pooled;        // [B, M] or NULL
  int64_t B;
  int p, q, D, M, ept;  // ept = examples per tile = 128 / D
  int sa, sc, sk;
  int act;
  int accumulate;       // 1: out += result (plain load-add-store: every element has one owner)
  FastDiv div_q, div_d;
};

}  // namespace

// Khatri-Rao GEMM (forward and both input gradients).  grid = (ceil(B / ept), ceil(M / BM)).
template <int BM>
__global__ void __launch_bounds__(CIN_THREADS, 2) cin_kr_gemm_kernel(const KrArgs g) {
  constexpr int TM = BM / 16;
  __shared__ __align__(16) CinSmem<BM> sm;
  const int t = threadIdx.x, ty = t >> 4, tx = t & 15;
  const int64_t b0 = (int64_t)blockIdx.x * g.ept;
  const int k0 = blockIdx.y * BM;
  const int K = g.p * g.q;
  const int nsteps = (K + CIN_BK - 1) / CIN_BK;

  // generated operand: this thread always stages column j of the tile, rows kz0 + 2s of each step
  const int j = t & (CIN_BN - 1), kz0 = t >> 7;
  int e_loc, d_loc;
  divmod(g.div_d, (uint32_t)j, e_loc, d_loc);
  const bool col_ok = e_loc < g.ept && b0 + e_loc < g.B;
  const float* Pb = g.P + (col_ok ? ((b0 + e_loc) * g.p * g.D + d_loc) : 0);
  const float* Qb = g.Q + (col_ok ? ((b0 + e_loc) * g.q * g.D + d_loc) : 0);
  // weight operand: output-fastest when sk == 1 (forward), contraction-fastest otherwise
  const bool w_kfast = g.sk == 1;
  constexpr int WPT = BM * CIN_BK / CIN_THREADS;   // == TM
  const int wr0 = w_kfast ? (t % BM) : (t >> 4);
  const int wk0 = w_kfast ? (t / BM) : (t & 15);

  float zr[8], wr[WPT];
  auto load_step = [&](int step) {
    int kg = step * CIN_BK + kz0, a, c;
    divmod(g.div_q, (uint32_t)kg, a, c);
#pragma unroll
    for (int s = 0; s < 8; ++s) {
      zr[s] = (col_ok && kg < K) ? __ldg(Pb + a * g.D) * __ldg(Qb + c * g.D) : 0.f;
      kg += 2; c += 2;
      while (c >= g.q) { c -= g.q; ++a; }
    }
#pragma unroll
    for (int s = 0; s < WPT; ++s) {
      const int kk = w_kfast ? wk0 + (CIN_THREADS / BM) * s : wk0;
      const int r = w_kfast ? wr0 : wr0 + 16 * s;
      const int kw = step * CIN_BK + kk;
      float v = 0.f;
      if (kw < K && k0 + r < g.M) {
        int aw, cw;
        divmod(g.div_q, (uint32_t)kw, aw, cw);
        v = __ldg(g.W + (int64_t)aw * g.sa + (int64_t)cw * g.sc + (int64_t)(k0 + r) * g.sk);
      }
      wr[s] = v;
    }
  };
  auto store_step = [&](int buf) {
#pragma unroll
    for (int s = 0; s < 8; ++s) sm.k.b[buf][kz0 + 2 * s][j] = zr[s];
#pragma unroll
    for (int s = 0; s < WPT; ++s) {
      const int kk = w_kfast ? wk0 + (CIN_THREADS / BM) * s : wk0;
      const int r = w_kfast ? wr0 : wr0 + 16 * s;
      sm.k.a[buf][kk][r] = wr[s];
    }
  };

  float acc[TM][8];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) acc[i][jj] = 0.f;

  load_step(0);
  store_step(0);
  __syncthreads();
  for (int step = 0; step < nsteps; ++step) {
    const int buf = step & 1;
    if (step + 1 < nsteps) load_step(step + 1);
    tile_fma<BM>(sm.k.a[buf], sm.k.b[buf], acc, ty, tx);
    if (step + 1 < nsteps) store_step(buf ^ 1);
    __syncthreads();
  }

  // epilogue: 64 rows at a time through shared memory, then stores in output order ([b][k][d] contiguous runs)
#pragma unroll
  for (int ii = 0; ii < TM / 4; ++ii) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int row = ty * 4 + e;
      const int k = k0 + 64 * ii + row;
      const float bv = (g.bias && k < g.M) ? __ldg(g.bias + k) : 0.f;
#pragma unroll
      for (int jj = 0; jj < 2; ++jj)
#pragma unroll
        for (int f = 0; f < 4; ++f) {
          float v = acc[ii * 4 + e][jj * 4 + f];
          if (!g.accumulate) v = act_apply(v + bv, g.act);
          sm.y[row][tx * 4 + 64 * jj + f] = v;
        }
    }
    __syncthreads();
    const int rows = min(64, g.M - (k0 + 64 * ii));
    const int64_t nex = min((int64_t)g.ept, g.B - b0);
    const int per_ex = rows * g.D;
    const int total = (int)nex * per_ex;
    for (int f = t; f < total; f += CIN_THREADS) {
      const int ex = f / per_ex, rem = f - ex * per_ex;
      int r, d;
      divmod(g.div_d, (uint32_t)rem, r, d);
      const int64_t o = ((b0 + ex) * g.M + k0 + 64 * ii + r) * g.D + d;
      const float v = sm.y[r][ex * g.D + d];
      g.out[o] = g.accumulate ? g.out[o] + v : v;
    }
    if (g.pooled) {
      for (int f = t; f < (int)nex * rows; f += CIN_THREADS) {
        const int ex = f / rows, r = f - ex * rows;
        float s = 0.f;
        for (int d = 0; d < g.D; ++d) s += sm.y[r][ex * g.D + d];
        g.pooled[(b0 + ex) * g.M + k0 + 64 * ii + r] = s;
      }
    }
    __syncthreads();
  }
}

// gW[i*h+j, k] = sum over this CTA's column range of G[n,k] * x0[n,i] * x[n,j], reduced into gW with red.global.add.
// grid = (ceil(m*h / 128), ceil(H / BM), splits); a CTA covers `steps_per_split` steps of 16 columns (b, d).
template <int BM>
__global__ void __launch_bounds__(CIN_THREADS, 2) cin_wgrad_kernel(const float* __restrict__ x0,
                                                                   const float* __restrict__ x,
                                                                   const float* __restrict__ G, int m, int h, int D,
                                                                   int H, uint32_t ncols, int steps_per_split,
                                                                   FastDiv div_d, FastDiv div_h,
                                                                   float* __restrict__ gw) {
  constexpr int TM = BM / 16;
  __shared__ __align__(16) CinSmem<BM> sm;
  const int t = threadIdx.x, ty = t >> 4, tx = t & 15;
  const int pair0 = blockIdx.x * CIN_BN;
  const int k0 = blockIdx.y * BM;
  const int npairs = m * h;
  const int total_steps = (int)((ncols + CIN_BK - 1) / CIN_BK);
  const int step0 = blockIdx.z * steps_per_split;
  const int step1 = min(total_steps, step0 + steps_per_split);
  if (step0 >= step1) return;

  // every staged element of this thread belongs to column kk of the step: one divmod per step
  const int kk = t & 15, rs = t >> 4;
  int i_first, j_first;            // field pair of this thread's first staged row; the others follow 16 pairs apart
  divmod(div_h, (uint32_t)(pair0 + rs), i_first, j_first);
  float ar[TM], br[8];
  auto load_step = [&](int step) {
    const uint32_t n = (uint32_t)step * CIN_BK + kk;
    const bool ok = n < ncols;
    int b = 0, d = 0;
    if (ok) divmod(div_d, n, b, d);
    const float* gb = G + ((int64_t)b * H * D + d);
    const float* x0b = x0 + ((int64_t)b * m * D + d);
    const float* xb = x + ((int64_t)b * h * D + d);
#pragma unroll
    for (int s = 0; s < TM; ++s) {
      const int k = k0 + rs + 16 * s;
      ar[s] = (ok && k < H) ? __ldg(gb + (int64_t)k * D) : 0.f;
    }
    int i = i_first, jf = j_first;
#pragma unroll
    for (int s = 0; s < 8; ++s) {
      br[s] = (ok && i < m) ? __ldg(x0b + i * D) * __ldg(xb + jf * D) : 0.f;
      jf += 16;
      while (jf >= h) { jf -= h; ++i; }
    }
  };
  auto store_step = [&](int buf) {
#pragma unroll
    for (int s = 0; s < TM; ++s) sm.k.a[buf][kk][rs + 16 * s] = ar[s];
#pragma unroll
    for (int s = 0; s < 8; ++s) sm.k.b[buf][kk][rs + 16 * s] = br[s];
  };

  float acc[TM][8];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) acc[i][jj] = 0.f;

  load_step(step0);
  store_step(0);
  __syncthreads();
  for (int step = step0; step < step1; ++step) {
    const int buf = (step - step0) & 1;
    if (step + 1 < step1) load_step(step + 1);
    tile_fma<BM>(sm.k.a[buf], sm.k.b[buf], acc, ty, tx);
    if (step + 1 < step1) store_step(buf ^ 1);
    __syncthreads();
  }
#pragma unroll
  for (int ii = 0; ii < TM / 4; ++ii)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int k = k0 + ty * 4 + 64 * ii + e;
      if (k >= H) continue;
#pragma unroll
      for (int jj = 0; jj < 2; ++jj)
#pragma unroll
        for (int f = 0; f < 4; ++f) {
          const int pr = pair0 + tx * 4 + 64 * jj + f;
          if (pr < npairs) red_add_f32(gw + (int64_t)pr * H + k, acc[ii * 4 + e][jj * 4 + f]);
        }
    }
}

// G[b,k,d] = (gy[b,k,d] + gpool[b,k]) * act'(y[b,k,d]) and gb[k] += sum_{b,d} G.  One warp per (b, k) row of D values
// at a time; per-CTA column sums of gb in shared memory.
__global__ void __launch_bounds__(256) cin_grad_prologue_kernel(const float* __restrict__ y, const float* __restrict__ gy,
                                                                const float* __restrict__ gpool, int64_t rows, int H,
                                                                int D, int act, float* __restrict__ G,
                                                                float* __restrict__ gb) {
  extern __shared__ float s_gb[];
  if (gb)
    for (int k = threadIdx.x; k < H; k += blockDim.x) s_gb[k] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < rows; r += nwarps) {
    const float gp = gpool ? __ldg(gpool + r) : 0.f;
    float part = 0.f;
    for (int d = lane; d < D; d += 32) {
      const int64_t o = r * D + d;
      float v = (gy ? gy[o] : 0.f) + gp;
      if (act != DR_ACT_NONE) v *= act_grad_from_y(__ldg(y + o), act);
      G[o] = v;
      part += v;
    }
    if (gb) {
      part = group_sum<32>(part);
      if (lane == 0) atomicAdd(&s_gb[(int)(r % H)], part);
    }
  }
  if (!gb) return;
  __syncthreads();
  for (int k = threadIdx.x; k < H; k += blockDim.x) red_add_f32(gb + k, s_gb[k]);
}

static int launch_kr(const float* P, const float* Q, const float* W, const float* bias, float* out, float* pooled,
                     int64_t B, int p, int q, int D, int M, int sa, int sc, int sk, int act, int accumulate,
                     cudaStream_t st) {
  KrArgs a{};
  a.P = P; a.Q = Q; a.W = W; a.bias = bias; a.out = out; a.pooled = pooled;
  a.B = B; a.p = p; a.q = q; a.D = D; a.M = M; a.ept = CIN_BN / D;
  a.sa = sa; a.sc = sc; a.sk = sk; a.act = act; a.accumulate = accumulate;
  a.div_q = make_fastdiv((uint32_t)q);
  a.div_d = make_fastdiv((uint32_t)D);
  const int64_t ctiles = (B + a.ept - 1) / a.ept;
  if (M > 64) {
    cin_kr_gemm_kernel<128><<<dim3((unsigned)ctiles, (unsigned)((M + 127) / 128)), CIN_THREADS, 0, st>>>(a);
  } else {
    cin_kr_gemm_kernel<64><<<dim3((unsigned)ctiles, 1), CIN_THREADS, 0, st>>>(a);
  }
  DR_CUDA_LAUNCH_CHECK("cin_kr_gemm");
  return DR_OK;
}

static int check_shape(const char* who, int64_t B, int m, int h, int D, int H) {
  DR_REQUIRE(B >= 0 && m >= 1 && h >= 1 && D >= 1 && H >= 1, DR_EINVAL,
             "%s: bad shape B=%lld m=%d h=%d D=%d H=%d", who, (long long)B, m, h, D, H);
  DR_REQUIRE(m <= CIN_MAX_FIELDS && h <= CIN_MAX_FIELDS && H <= CIN_MAX_FIELDS && D <= CIN_MAX_D, DR_ENOTSUP,
             "%s: m=%d h=%d H=%d D=%d above the served caps (m, h, H <= %d, D <= %d)", who, m, h, H, D,
             CIN_MAX_FIELDS, CIN_MAX_D);
  DR_REQUIRE(B * D < (int64_t)1 << 31, DR_ENOTSUP, "%s: B*D = %lld columns above the served cap 2^31", who,
             (long long)(B * D));
  return DR_OK;
}

}  // namespace dr

using namespace dr;

extern "C" int dr_cin_fwd(const float* x0, const float* x, const float* w, const float* bias, int64_t B, int m, int h,
                          int D, int H, int act, float* y, float* pooled, void* stream) {
  DR_REQUIRE(w && (B == 0 || (x0 && x && y)), DR_EINVAL, "dr_cin_fwd: null pointer");   // B = 0: empty tensors
  DR_REQUIRE(act >= DR_ACT_NONE && act <= DR_ACT_TANH, DR_EINVAL, "dr_cin_fwd: unknown activation %d", act);
  if (int rc = check_shape("dr_cin_fwd", B, m, h, D, H)) return rc;
  if (B == 0) return DR_OK;
  return launch_kr(x0, x, w, bias, y, pooled, B, m, h, D, H, h * H, H, 1, act, 0, (cudaStream_t)stream);
}

extern "C" int dr_cin_bwd(const float* x0, const float* x, const float* w, const float* y, const float* gy,
                          const float* gpool, int64_t B, int m, int h, int D, int H, int act, int x_is_x0, float* g_ws,
                          float* gx0, float* gx, float* gw, float* gb, void* stream) {
  DR_REQUIRE(w && gw && (B == 0 || (x0 && x && y && g_ws && gx0)), DR_EINVAL, "dr_cin_bwd: null pointer");
  DR_REQUIRE(B == 0 || gy || gpool, DR_EINVAL, "dr_cin_bwd: gy and gpool are both NULL");
  DR_REQUIRE(act >= DR_ACT_NONE && act <= DR_ACT_TANH, DR_EINVAL, "dr_cin_bwd: unknown activation %d", act);
  if (x_is_x0) {
    DR_REQUIRE(!gx && x == x0 && h == m, DR_EINVAL, "dr_cin_bwd: x_is_x0 needs x == x0, h == m and gx == NULL");
  } else {
    DR_REQUIRE(B == 0 || gx, DR_EINVAL, "dr_cin_bwd: gx is NULL (only the x_is_x0 form accumulates it into gx0)");
  }
  if (int rc = check_shape("dr_cin_bwd", B, m, h, D, H)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  DR_CUDA_CALL(cudaMemsetAsync(gw, 0, sizeof(float) * (size_t)m * h * H, st));
  if (gb) DR_CUDA_CALL(cudaMemsetAsync(gb, 0, sizeof(float) * H, st));
  if (B == 0) return DR_OK;
  {
    const int64_t rows = B * H;
    int64_t ctas = (rows + 7) / 8;
    if (ctas > (int64_t)num_sms() * 8) ctas = (int64_t)num_sms() * 8;
    cin_grad_prologue_kernel<<<(unsigned)ctas, 256, gb ? sizeof(float) * H : 0, st>>>(y, gy, gpool, rows, H, D, act,
                                                                                     g_ws, gb);
    DR_CUDA_LAUNCH_CHECK("cin_grad_prologue");
  }
  // gx0[b,i,d] = sum_{j,k} W[i,j,k] x[b,j,d] G[b,k,d] ;  gx[b,j,d] = sum_{i,k} W[i,j,k] x0[b,i,d] G[b,k,d]
  if (int rc = launch_kr(x, g_ws, w, nullptr, gx0, nullptr, B, h, H, D, m, H, 1, h * H, DR_ACT_NONE, 0, st)) return rc;
  if (int rc = launch_kr(x0, g_ws, w, nullptr, x_is_x0 ? gx0 : gx, nullptr, B, m, H, D, h, h * H, 1, H, DR_ACT_NONE,
                         x_is_x0, st))
    return rc;
  {
    const uint32_t ncols = (uint32_t)(B * D);
    const int64_t steps = (ncols + CIN_BK - 1) / CIN_BK;
    const int bm = H > 64 ? 128 : 64;
    const int64_t tiles = (int64_t)((m * h + CIN_BN - 1) / CIN_BN) * ((H + bm - 1) / bm);
    // enough CTAs for ~4 waves of 2 CTAs per SM, each split at least 64 steps (1024 columns) long
    int64_t splits = ((int64_t)num_sms() * 8 + tiles - 1) / tiles;
    if (splits > steps / 64) splits = steps / 64;
    if (splits < 1) splits = 1;
    const int per = (int)((steps + splits - 1) / splits);
    splits = (steps + per - 1) / per;
    const dim3 grid((unsigned)((m * h + CIN_BN - 1) / CIN_BN), (unsigned)((H + bm - 1) / bm), (unsigned)splits);
    const FastDiv dd = make_fastdiv((uint32_t)D), dh = make_fastdiv((uint32_t)h);
    if (bm == 128)
      cin_wgrad_kernel<128><<<grid, CIN_THREADS, 0, st>>>(x0, x, g_ws, m, h, D, H, ncols, per, dd, dh, gw);
    else
      cin_wgrad_kernel<64><<<grid, CIN_THREADS, 0, st>>>(x0, x, g_ws, m, h, D, H, ncols, per, dd, dh, gw);
    DR_CUDA_LAUNCH_CHECK("cin_wgrad");
  }
  return DR_OK;
}
