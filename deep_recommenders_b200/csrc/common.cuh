// Shared host/device helpers for libdeeprec_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <type_traits>
#include "deeprec_b200.h"

#ifndef __CUDA_ARCH_LIST__
#define __CUDA_ARCH_LIST__ 900
#endif

namespace dr {

// SMs of the current device (132 on an H100 SXM, fewer on a PCIe card or a MIG slice): sizes every persistent grid and
// split-K heuristic.  Queried once per process (api.cu).
int num_sms();

// Largest world the row-sharded entries address (peer-base tables of this many pointers live in shared memory).
constexpr int kMaxShardWorld = 64;

// ---- error plumbing -------------------------------------------------------------------
void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define DR_REQUIRE(cond, code, ...)              \
  do {                                           \
    if (!(cond)) {                               \
      dr::set_error(__VA_ARGS__);                \
      return (code);                             \
    }                                            \
  } while (0)

#define DR_CUDA_LAUNCH_CHECK(name)                                            \
  do {                                                                        \
    cudaError_t e__ = cudaGetLastError();                                     \
    if (e__ != cudaSuccess) {                                                 \
      dr::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));  \
      return (int)e__;                                                        \
    }                                                                         \
    dr::count_launch();                                                       \
  } while (0)

#define DR_CUDA_CALL(expr)                                                    \
  do {                                                                        \
    cudaError_t e__ = (expr);                                                 \
    if (e__ != cudaSuccess) {                                                 \
      dr::set_error("%s failed: %s", #expr, cudaGetErrorString(e__));         \
      return (int)e__;                                                        \
    }                                                                         \
  } while (0)

__host__ __device__ static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ---- host side of the entries: argument checks and launch dispatch ------------------------------------------------------
// The shape and id-width checks of the lookup entries, in this order.  `d_join` joins the two conditions of the D
// message: the embedding entries print " and", the FNN entries ",".
static inline int check_lookup_dims(const char* fn, int64_t B, int S, int D, int id_bytes, const char* d_join = " and") {
  DR_REQUIRE(B >= 0, DR_EINVAL, "%s: B=%lld < 0", fn, (long long)B);
  DR_REQUIRE(S >= 1 && S <= 4096, DR_EINVAL, "%s: S=%d outside [1,4096]", fn, S);
  DR_REQUIRE(D >= 4 && D <= 128 && (D % 4) == 0, DR_EINVAL,
             "%s: D=%d unsupported (need D %% 4 == 0%s 4 <= D <= 128)", fn, D, d_join);
  DR_REQUIRE(id_bytes == 8 || id_bytes == 4, DR_EINVAL, "%s: id_bytes=%d (need 4 or 8)", fn, id_bytes);
  return DR_OK;
}

// Lanes per row for `chunks` 16-B chunks: the next power of two.
static inline int lanes_per_row(int chunks) {
  int lpr = 1;
  while (lpr < chunks) lpr <<= 1;
  return lpr;
}

// ceil(items / per_cta) CTAs, at most ctas_per_sm per SM
static inline int64_t capped_grid(int64_t items, int64_t per_cta, int ctas_per_sm) {
  const int64_t ctas = (items + per_cta - 1) / per_cta, cap = (int64_t)num_sms() * ctas_per_sm;
  return ctas > cap ? cap : ctas;
}

// A kernel launched with more than 48 KB of dynamic shared memory has to be allowed that much first.
template <typename Kernel>
static inline int allow_dynamic_smem(Kernel* k, size_t smem) {
  if (smem > 48 * 1024) DR_CUDA_CALL(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return DR_OK;
}

// f(std::integral_constant<int, LPR>{}) for lpr in {MIN, 2 MIN, ..., MAX}; any other lpr runs as MAX.  Returns f's code,
// and instantiates f for those lane counts only.
template <int MAX = 32, int MIN = 1, typename F>
inline int with_lpr(int lpr, F&& f) {
  if constexpr (MIN >= MAX) return f(std::integral_constant<int, MAX>{});
  else if (lpr == MIN) return f(std::integral_constant<int, MIN>{});
  else return with_lpr<MAX, 2 * MIN>(lpr, f);
}
// f(IdT{}) with IdT = int64_t for id_bytes 8, int32_t otherwise
template <typename F>
inline int with_id_type(int id_bytes, F&& f) {
  if (id_bytes == 8) return f(int64_t{});
  return f(int32_t{});
}
template <int MAX = 32, typename F>
inline int with_lpr_id(int lpr, int id_bytes, F&& f) {
  return with_lpr<MAX>(lpr, [&](auto L) { return with_id_type(id_bytes, [&](auto id) { return f(L, id); }); });
}

// ---- device helpers -------------------------------------------------------------------
#ifdef __CUDACC__

// 128-bit read-only load that does not allocate in L1 (random rows are touched once).
__device__ __forceinline__ float4 ldg_nc_na(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ float ldg_nc_na_f32(const float* p) {
  float r;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}
// L2 eviction-priority hints (experiment, knob embed_l2_hints): the random table rows are dead after one use
// (evict_first), the stacked output is re-read by the next kernel (evict_last), the backward's atomically updated lines
// should drain to HBM early instead of staying dirty in L2 until the next kernel's stores push them out.
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ float4 ldg_nc_na_hint(const float* p, uint64_t pol) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ float ldg_nc_na_f32_hint(const float* p, uint64_t pol) {
  float r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(r) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ void stg4_hint(float* p, float4 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void red_add_v4_hint(float* p, float4 v, uint64_t pol) {
  asm volatile("red.global.add.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void red_add_f32_hint(float* p, float v, uint64_t pol) {
  asm volatile("red.global.add.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(p), "f"(v), "l"(pol) : "memory");
}
// 128-bit load through the normal (L1-allocating) path.
__device__ __forceinline__ float4 ldg4(const float* p) { return *reinterpret_cast<const float4*>(p); }

// streaming 128-bit store (write-once data that the next kernel reads from L2/HBM).
__device__ __forceinline__ void stg4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// 128-bit vector reduction into global memory (sm_90+): one REDG.E.ADD.F32x4 per 16 B.
__device__ __forceinline__ void red_add_v4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}
__device__ __forceinline__ void red_add_f32(float* p, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

template <int W>
__device__ __forceinline__ float group_sum(float v) {
  // butterfly over the W (power of two, <= 32) lanes of an aligned lane group
#pragma unroll
  for (int o = W / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float4 f4_zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ float4 f4_add(float4 a, float4 b) {
  return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}
__device__ __forceinline__ float4 f4_shfl_down(float4 v, int delta) {
  return make_float4(__shfl_down_sync(0xffffffffu, v.x, delta), __shfl_down_sync(0xffffffffu, v.y, delta),
                     __shfl_down_sync(0xffffffffu, v.z, delta), __shfl_down_sync(0xffffffffu, v.w, delta));
}

// V consecutive floats moved as one access: V = 4 is a 128-bit load / store (16-B aligned address), V = 1 the scalar
// form of the same kernel for shapes that are not a multiple of 4 wide.
template <int V>
struct alignas(4 * V) Vec {
  float v[V];
};

__device__ __forceinline__ float act_apply(float v, int act) {
  switch (act) {
    case DR_ACT_RELU: return fmaxf(v, 0.f);
    case DR_ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    case DR_ACT_TANH: return tanhf(v);
    default: return v;
  }
}
// derivative expressed through the OUTPUT y = act(z)
__device__ __forceinline__ float act_grad_from_y(float y, int act) {
  switch (act) {
    case DR_ACT_RELU: return y > 0.f ? 1.f : 0.f;
    case DR_ACT_SIGMOID: return y * (1.f - y);
    case DR_ACT_TANH: return 1.f - y * y;
    default: return 1.f;
  }
}
#endif  // __CUDACC__

}  // namespace dr
