// TensorFlow's Adam as the optimizer kernels of optim.cu and embed_adam.cu share it: the ApplyAdam functor, the replay
// of the steps a row sat out, one lane's share of a row's replay and update, and the host-side check of their
// hyperparameters.
#pragma once
#include "common.cuh"

namespace dr {

__device__ __forceinline__ void adam_functor(float& p, float g, float& m, float& v, float lr_t, float omb1, float omb2,
                                             float eps) {
  // training_ops ApplyAdam: m += (g - m)(1 - b1); v += (g*g - v)(1 - b2); var -= lr_t * m / (sqrt(v) + eps)
  m += (g - m) * omb1;
  v += (g * g - v) * omb2;
  p -= (m * lr_t) / (sqrtf(v) + eps);
}

__device__ __forceinline__ void adam_functor4(float4& p, float4 g, float4& m, float4& v, float lr_t, float omb1,
                                              float omb2, float eps) {
  adam_functor(p.x, g.x, m.x, v.x, lr_t, omb1, omb2, eps);
  adam_functor(p.y, g.y, m.y, v.y, lr_t, omb1, omb2, eps);
  adam_functor(p.z, g.z, m.z, v.z, lr_t, omb1, omb2, eps);
  adam_functor(p.w, g.w, m.w, v.w, lr_t, omb1, omb2, eps);
}

__host__ __device__ inline int adam_state_stride(int D) { return (3 * D + 5 + 31) / 32 * 32; }   // + count + step stamp

__device__ __forceinline__ float4 ld_cg4(const float* p) {
  float4 r;
  asm volatile("ld.global.cg.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ float ld_cg1(const float* p) {
  float r;
  asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(r) : "l"(p) : "memory");
  return r;
}

// How a kernel reads a row's Adam state: through L2 (LdCg) where other lanes of the same kernel have just added into
// the block or moved its count, with plain loads (LdPlain) where nothing else in the kernel writes it.  s1(st, o, k)
// reads st[o + k].
struct LdPlain {
  static __device__ __forceinline__ float4 v4(const float* p) { return *reinterpret_cast<const float4*>(p); }
  static __device__ __forceinline__ float s1(const float* st, int o, int k) { return st[o + k]; }
};
struct LdCg {
  static __device__ __forceinline__ float4 v4(const float* p) { return ld_cg4(p); }
  static __device__ __forceinline__ float s1(const float* st, int o, int k) { return ld_cg1(st + o + k); }
};

// ---- exact tf.keras Adam for rows that were NOT touched for a while (EXACT mode) ---------------------------------------
// TensorFlow's Adam is dense: in a step that does not touch a row, m <- m - m(1-b1), v <- v - v(1-b2) and the row still
// moves by -lr_j m / (sqrt(v) + eps).  The row-sparse form replays those skipped steps when the row is next touched (or
// flushed): per-row stamp = last step whose update the row has seen; lr_j comes from the history dr_adam_advance_hist
// keeps (ring of `hist_len` bias-corrected rates), or is recomputed when the step fell out of the ring.  Steps beyond
// kCatchUpMax after the stamp cannot move the row any more (m has decayed by 0.9^2048, far below fp32's range relative to
// v): they only decay v, in closed form.
constexpr int kCatchUpMax = 2048;
struct AdamHist {
  const float* lr_hist;
  int hist_len;
  float lr, b1, b2;
};
__device__ __forceinline__ float adam_lr_at(const AdamHist& h, int64_t j, int64_t t_now) {
  if (h.lr_hist && t_now - j < h.hist_len) return __ldg(h.lr_hist + (j % h.hist_len));
  return h.lr * sqrtf(1.f - powf(h.b2, (float)j)) / (1.f - powf(h.b1, (float)j));
}
// N elements of one lane: replay steps (stamp, upto] with zero gradient
template <int N>
__device__ __forceinline__ void adam_catch_up(float (&p)[N], float (&m)[N], float (&v)[N], int64_t stamp, int64_t upto,
                                              int64_t t_now, const AdamHist& h, float omb1, float omb2, float eps) {
  if (stamp <= 0 || upto <= stamp) return;                    // never updated (m = v = 0): nothing to replay
  const int64_t gap = upto - stamp;
  const int n = (int)(gap < kCatchUpMax ? gap : kCatchUpMax);
  for (int k = 1; k <= n; ++k) {
    const float lr_j = adam_lr_at(h, stamp + k, t_now);
#pragma unroll
    for (int e = 0; e < N; ++e) {
      m[e] = fmaf(-m[e], omb1, m[e]);
      v[e] = fmaf(-v[e], omb2, v[e]);
      p[e] -= __fdividef(m[e] * lr_j, sqrtf(v[e]) + eps);
    }
  }
  if (gap > n) {
    const float dm = powf(1.f - omb1, (float)(gap - n)), dv = powf(1.f - omb2, (float)(gap - n));
#pragma unroll
    for (int e = 0; e < N; ++e) { m[e] *= dm; v[e] *= dv; }
  }
}

__device__ __forceinline__ void adam_catch_up4(float4& p, float4& m, float4& v, int64_t stamp, int64_t upto,
                                               int64_t t_now, const AdamHist& h, float omb1, float omb2, float eps) {
  float pa[4] = {p.x, p.y, p.z, p.w}, ma[4] = {m.x, m.y, m.z, m.w}, va[4] = {v.x, v.y, v.z, v.w};
  adam_catch_up<4>(pa, ma, va, stamp, upto, t_now, h, omb1, omb2, eps);
  p = make_float4(pa[0], pa[1], pa[2], pa[3]);
  m = make_float4(ma[0], ma[1], ma[2], ma[3]);
  v = make_float4(va[0], va[1], va[2], va[3]);
}

__device__ __forceinline__ void adam_catch_up1(float& p, float& m, float& v, int64_t stamp, int64_t upto,
                                               int64_t t_now, const AdamHist& h, float omb1, float omb2, float eps) {
  float pa[1] = {p}, ma[1] = {m}, va[1] = {v};
  adam_catch_up<1>(pa, ma, va, stamp, upto, t_now, h, omb1, omb2, eps);
  p = pa[0]; m = ma[0]; v = va[0];
}

// ---- one lane's share of a row: its 16-B chunk of the table row (p) and of the state block's m and v, or the row's
// first-order weight (*w) and its gradient and moments st[o_s + 0, 1, 2].  The table row is read with plain loads.
// The helpers form each address and order each load as the kernels did when these steps were written out in them: the
// kernels compile to the same machine code as before, and a change to either shows up as a SASS difference. ----------
// replay steps (stamp, upto]; the state is read through `Ld`, the lane's words are st[o_m + k, ...) and p[k, ...)
template <class Ld>
__device__ __forceinline__ void adam_replay_chunk(float* st, int o_m, int o_v, float* p, int k, int64_t stamp,
                                                  int64_t upto, int64_t t_now, const AdamHist& h, float omb1, float omb2,
                                                  float eps) {
  float4 mm = Ld::v4(st + o_m + k), vv = Ld::v4(st + o_v + k);
  float4 pp = *reinterpret_cast<const float4*>(p + k);
  adam_catch_up4(pp, mm, vv, stamp, upto, t_now, h, omb1, omb2, eps);
  stg4(p + k, pp);
  stg4(st + o_m + k, mm);
  stg4(st + o_v + k, vv);
}
template <class Ld>
__device__ __forceinline__ void adam_replay_weight(float* w, float* st, int o_s, int64_t stamp, int64_t upto,
                                                   int64_t t_now, const AdamHist& h, float omb1, float omb2, float eps) {
  float pw = *w, mw = Ld::s1(st, o_s, 1), vw = Ld::s1(st, o_s, 2);
  adam_catch_up1(pw, mw, vw, stamp, upto, t_now, h, omb1, omb2, eps);
  *w = pw; st[o_s + 1] = mw; st[o_s + 2] = vw;
}
// replay steps (stamp, upto], then take this step from the accumulated gradient g and clear it; the state is read
// through L2 (its gradient is the other lanes' red.add)
__device__ __forceinline__ void adam_replay_step_chunk(float* g, float* m, float* v, float* p, int64_t stamp,
                                                       int64_t upto, int64_t t_now, const AdamHist& h, float lr_t,
                                                       float omb1, float omb2, float eps) {
  const float4 gg = ld_cg4(g);
  float4 mm = ld_cg4(m), vv = ld_cg4(v);
  float4 pp = *reinterpret_cast<const float4*>(p);
  adam_catch_up4(pp, mm, vv, stamp, upto, t_now, h, omb1, omb2, eps);
  adam_functor4(pp, gg, mm, vv, lr_t, omb1, omb2, eps);
  stg4(p, pp);
  stg4(m, mm);
  stg4(v, vv);
  stg4(g, f4_zero());
}
__device__ __forceinline__ void adam_replay_step_weight(float* w, float* st, int o_s, int64_t stamp, int64_t upto,
                                                        int64_t t_now, const AdamHist& h, float lr_t, float omb1,
                                                        float omb2, float eps) {
  float pw = *w, mw = ld_cg1(st + o_s + 1), vw = ld_cg1(st + o_s + 2);
  adam_catch_up1(pw, mw, vw, stamp, upto, t_now, h, omb1, omb2, eps);
  adam_functor(pw, ld_cg1(st + o_s), mw, vw, lr_t, omb1, omb2, eps);
  *w = pw; st[o_s + 1] = mw; st[o_s + 2] = vw;
  st[o_s] = 0.f;
}

// ---- host side of the entries -----------------------------------------------------------------------------------------
static inline int check_adam_hparams(const char* fn, float beta1, float beta2, float eps) {
  DR_REQUIRE(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f && eps >= 0.f, DR_EINVAL,
             "%s: beta1=%g beta2=%g eps=%g out of range", fn, (double)beta1, (double)beta2, (double)eps);
  return DR_OK;
}

}  // namespace dr
