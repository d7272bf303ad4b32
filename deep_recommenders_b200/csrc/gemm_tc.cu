// The tensor-core form of the fp32 GEMM core: Hopper warpgroup MMA (wgmma) with 3xTF32 split products.
//
//   C[M,N] = epilogue( A @ B ),   A = Ah + Al, B = Bh + Bl   (Ah = fp32 with the low 13 mantissa
//   bits cleared = exactly representable in TF32, Al = A - Ah exactly),
//   A @ B ~= Al@Bh + Ah@Bl + Ah@Bh      (the dropped Al@Bl term is ~2^-22 relative)
// which restores fp32-level accuracy (the parity bar is 1e-5 relative, out of reach of single-pass
// TF32/BF16) at 3 tensor-core products per k-step.
//
// Structure (one 128 x BN output tile per work item, persistent grid, 416 threads, sm_90a only):
//   warps 0-7   two consumer warpgroups, 64 rows of the tile each: wgmma.mma_async.m64n{BN}k8.tf32 (accumulator in
//               registers) x 4 k-steps x 3 products per k-block, then the fused epilogue (gemm.cuh Epi modes).  The
//               modes whose only output is C write the warpgroup's 64 x BN results into a shared-memory staging tile
//               that one thread stores with TMA (a TMA reduce-add for split-K), so the warpgroup goes on to the next
//               tile's MMAs while the tile drains; the others, and C that TMA cannot address, store float2 / issue
//               split-K reductions straight from the accumulator registers.  Variant 2: each thread loads its
//               A-fragment elements from the raw A tile, splits them in registers and passes them to wgmma as a
//               register fragment; B comes from the plane ring.  Variant 1: both operands from the plane ring.
//   warps 8-11  splitters (variant 2): turn every staged raw fp32 B tile into its hi and lo planes in the layout wgmma
//               reads
//   warp 12     TMA producer: cp.async.bulk.tensor into the raw ring, completion on "full" mbarriers (expect_tx)
// wgmma reads 32-bit B operands from shared memory K-major only (canonical SWIZZLE_128B layout, 32 tf32 = 128 B per
// row).  A B operand stored K-major (row-major [N, K]) is staged by TMA in exactly that layout and split chunk by chunk;
// one stored MN-major ([K, N] row-major: the weight of a forward layer, gZ in a weight gradient) is staged as stored and
// TRANSPOSED by the same splitter pass, which has to touch every element anyway.  A is staged as stored (K-major in
// SWIZZLE_128B, MN-major unswizzled) and read element by element by the consumers, so either layout needs no transpose.
// Two rings decouple the stages: raw tiles (TMA -> splitters and consumers), B planes (splitters -> wgmma), each with
// full / empty mbarriers; fence.proxy.async orders the splitters' generic stores before wgmma's reads.
// Variant 1 (g_tune_gemm_variant == 1, PRESPLIT): the hi/lo planes of both operands are produced K-major in
// caller-provided workspace (dr_set_workspace) by split_tf32_kernel / split_tf32_transpose_kernel and TMA loads them
// straight into the plane ring; variant 2 (the default) needs no workspace and no pre-pass.
// Weight planes (gemm_tc_wplanes_kernel, variant 2 with the plane cache on, A K-major, B small against A): B's K-major
// hi/lo planes are split once per step into the workspace and TMA loads them beside the raw A tile into one ring
// [A raw | Bh | Bl]; A is split in registers as in variant 2.  No splitter warps, no plane ring: 288 threads, and a stage
// is released once its k-block's MMAs have retired.  A tile whose valid width is at most 32 or 64 columns runs
// m64n32k8 / m64n64k8 MMAs into the leading accumulators.
// In every kernel a consumer warpgroup whose 64 rows all lie past M issues no loads, MMAs or epilogue for that tile.
#include "gemm.cuh"
#include <cuda.h>
#include <float.h>
#include <string.h>

namespace dr {

// ---- workspace registered by the host (dr_set_workspace) ----------------------------------------
int g_tune_gemm_bn = 0;     // 0 = auto; 32 / 64 / 128 cap the tile width (wider requests run 128: the accumulator of a
                            // 64 x 256 warpgroup tile would take 128 registers per thread)
int g_tune_tc_min_n = 32;   // outputs narrower than this stay on the FFMA kernel
int g_tune_tc_l2_promo = 256;
static void* g_ws_ptr = nullptr;
static size_t g_ws_bytes = 0;

// Plane cache (dr_gemm_plane_cache, variant 1): inside a train step every tensor is split into its TF32 hi/lo
// planes ONCE per layout and the planes are shared by all the GEMMs that read it (x: forward and dW; gz: dX and
// dW; W: forward and dX).  Off by default: without it every GEMM call splits its own operands.  An entry is keyed by
// the whole view it was split from (pointer, layout, rows, K, pitch): one pointer read as [128, 64] and as [64, 128],
// or with K = 33 and K = 36 (same plane pitch), has other planes.
struct PlaneEntry { const float* src; bool transposed; int64_t rows, K, ld; float* hi; float* lo; int64_t pitch; };
static PlaneEntry g_planes[64];
static int g_nplanes = 0;
static bool g_cache_on = false;
static size_t g_bump = 0;     // floats used at the front of the workspace

constexpr int TC_BM = 128;
constexpr int TC_BK = 32;          // 32 tf32 = 128 bytes = one SWIZZLE_128B row
constexpr int TC_CONSUMERS = 256;  // two warpgroups
constexpr int TC_SPLITTERS = 128;
constexpr int TC_THREADS = TC_CONSUMERS + TC_SPLITTERS + 32;
constexpr int TC_WP_THREADS = TC_CONSUMERS + 32;   // weight-plane kernel: consumers + TMA warp
constexpr int TC_PLANE_STAGES = 2;
constexpr int TC_RAW_STAGES = 3;                   // raw ring depth of the splitter kernels (2 when shared)
constexpr int TC_MAX_RAW_STAGES = 4;
constexpr int TC_WP_STAGES = 4;                    // ring depth of the weight-plane kernel

// ---- small PTX wrappers ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}"
      ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// Shared -> global TMA store of one box, or its element-wise add into global memory; one bulk group per call site.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tm, const void* smem_src, int c0, int c1, bool add) {
  if (add)
    asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(tm), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1) : "memory");
  else
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(tm), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void named_barrier_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// wgmma shared-memory matrix descriptor of a K-major SWIZZLE_128B operand: rows of 128 B, 8-row swizzle groups 1024 B
// apart (stride byte offset); the leading byte offset is not used by swizzled K-major layouts.  The tile base is
// 1024-B aligned, so the base-offset field stays 0; a k-step of 8 tf32 advances the start address by 32 B.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024u >> 4) << 32;
  d |= (uint64_t)1 << 62;   // SWIZZLE_128B
  return d;
}

// D[64 x N] += A[64 x 8] * B[8 x N], tf32 operands from shared memory, fp32 accumulator fragment in registers
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t da, uint64_t db);
template <>
__device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
      "}, %16, %17, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(1));
}
template <>
__device__ __forceinline__ void wgmma_tf32<64>(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(1));
}
template <>
__device__ __forceinline__ void wgmma_tf32<128>(float (&d)[64], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(1));
}

// D[64 x N] += A[64 x 8] * B[8 x N] with A from registers: the thread's four elements of the .tf32 m64nNk8 A fragment
// (warp w of the warpgroup owns rows 16 w .. 16 w + 15; a[0] is row lane / 4, column lane % 4 of the k-step, a[1] row
// lane / 4 + 8, a[2] and a[3] the same rows at column lane % 4 + 4), B from shared memory by descriptor.
template <int N>
__device__ __forceinline__ void wgmma_tf32_ra(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t db);
template <>
__device__ __forceinline__ void wgmma_tf32_ra<32>(float (&d)[16], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
      "}, {%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(1));
}
template <>
__device__ __forceinline__ void wgmma_tf32_ra<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(1));
}
template <>
__device__ __forceinline__ void wgmma_tf32_ra<128>(float (&d)[64], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(1));
}

__global__ void __launch_bounds__(256) split_tf32_kernel(const float* __restrict__ x, int64_t n4,
                                                          float* __restrict__ hi, float* __restrict__ lo) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    float4 h, l;
    h.x = __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u); l.x = v.x - h.x;
    h.y = __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u); l.y = v.y - h.y;
    h.z = __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u); l.z = v.z - h.z;
    h.w = __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u); l.w = v.w - h.w;
    reinterpret_cast<float4*>(hi)[i] = h;
    reinterpret_cast<float4*>(lo)[i] = l;
  }
}

// x [R, C] row-major (pitch ldx)  ->  hi, lo [C, R] row-major (pitch ldo): transposed hi/lo planes,
// so that every tensor-core operand is K-major (the operand layout validated on hardware).
__global__ void __launch_bounds__(256) split_tf32_transpose_kernel(const float* __restrict__ x, int64_t R,
                                                                    int64_t C, int64_t ldx, int64_t ldo,
                                                                    float* __restrict__ hi, float* __restrict__ lo) {
  __shared__ float tile[32][33];
  const int tx = threadIdx.x, ty = threadIdx.y;   // (32, 8)
  const int64_t tiles_c = (C + 31) / 32, tiles_r = (R + 31) / 32;
  for (int64_t t = blockIdx.x; t < tiles_c * tiles_r; t += gridDim.x) {
    const int64_t r0 = (t / tiles_c) * 32, c0 = (t % tiles_c) * 32;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t r = r0 + ty + 8 * i, c = c0 + tx;
      tile[ty + 8 * i][tx] = (r < R && c < C) ? __ldg(x + r * ldx + c) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t c = c0 + ty + 8 * i, r = r0 + tx;
      if (c < C && r < R) {
        const float v = tile[tx][ty + 8 * i];
        const float h = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
        hi[c * ldo + r] = h;
        lo[c * ldo + r] = v - h;
      }
    }
    __syncthreads();
  }
}

// Splitter pass over one staged B tile of ROWS x 32 floats: hi = top 19 bits, lo = v - hi (exact), both written in
// the K-major SWIZZLE_128B layout (16-B chunk c of row r at r * 128 + ((c ^ (r & 7)) << 4)).
//   K-major raw tile: TMA staged it in that very layout, so the pass is elementwise on 16-B chunks;
//   MN-major raw tile: [32 k-rows][ROWS] as stored; a thread gathers 4 consecutive k of one row (the lanes of a warp read
//   32 consecutive floats of one k-row: conflict free) and writes one chunk (8 lanes cover all 32 banks: conflict free).
template <int ROWS, bool MN>
__device__ __forceinline__ void split_tile(const uint8_t* raw, uint8_t* hi, uint8_t* lo, int tid) {
  constexpr int CHUNKS = ROWS * 8;
#pragma unroll 4
  for (int idx = tid; idx < CHUNKS; idx += TC_SPLITTERS) {
    float4 v;
    uint32_t off;
    if (!MN) {
      off = (uint32_t)idx * 16u;
      v = *reinterpret_cast<const float4*>(raw + off);
    } else {
      const int r = idx % ROWS, c = idx / ROWS;
      const float* src = reinterpret_cast<const float*>(raw) + (4 * c) * ROWS + r;
      v = make_float4(src[0], src[ROWS], src[2 * ROWS], src[3 * ROWS]);
      off = (uint32_t)r * 128u + (uint32_t)((c ^ (r & 7)) << 4);
    }
    float4 h, l;
    h.x = __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u); l.x = v.x - h.x;
    h.y = __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u); l.y = v.y - h.y;
    h.z = __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u); l.z = v.z - h.z;
    h.w = __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u); l.w = v.w - h.w;
    *reinterpret_cast<float4*>(hi + off) = h;
    *reinterpret_cast<float4*>(lo + off) = l;
  }
}

// Work item = (m tile, n tile, k split).  Items are strided over the persistent grid.
struct TcItem {
  int64_t m0, n0;
  int kb0, nkb;
};
__device__ __forceinline__ TcItem tc_decode(int64_t item, int64_t n_tiles, int64_t m_tiles, int64_t kblocks,
                                            int64_t per, int BN) {
  TcItem t;
  const int64_t nt = item % n_tiles;
  const int64_t mt = (item / n_tiles) % m_tiles;
  const int64_t z = item / (n_tiles * m_tiles);
  t.m0 = mt * TC_BM;
  t.n0 = nt * BN;
  t.kb0 = (int)(z * per);
  const int64_t kb1 = min(kblocks, (z + 1) * per);
  t.nkb = (int)(kb1 - z * per);
  return t;
}

// Two adjacent columns n, n + 1 (n even) of a row-major operand: one 8-B access when VEC (base 8-B aligned, even pitch),
// else two scalar ones, the second only when `two` (n + 1 < N).
template <bool VEC>
__device__ __forceinline__ float2 ld_pair(const float* p, const bool two) {
  if constexpr (VEC) return __ldg(reinterpret_cast<const float2*>(p));
  else return make_float2(__ldg(p), two ? __ldg(p + 1) : 0.f);
}
template <bool VEC>
__device__ __forceinline__ void st_pair(float* p, const float2 v, const bool two) {
  if constexpr (VEC) {
    *reinterpret_cast<float2*>(p) = v;
  } else {
    p[0] = v.x;
    if (two) p[1] = v.y;
  }
}

// Staging tile of one consumer warpgroup: its 64 x BN results as BN / 32 boxes of 64 rows x 32 floats, each box in the
// TMA SWIZZLE_128B layout (16-B chunk c of row r at r * 128 + ((c ^ (r & 7)) << 4)), 8 KB apart; the base is 1024-B
// aligned.  `stg_frag_addr`: address of the thread's float2 at d[4 j + 2 h], from `stg` = the tile's row 16 w of warp w
// of the warpgroup.  A warp's store of one (h, j) covers 8 rows (lane / 4, so r & 7 = lane / 4) x 8 columns: lane pairs (lane % 4 = 0, 1 and 2, 3) fill chunks 2 (j % 4) and
// 2 (j % 4) + 1 of their row, XORed with r & 7.  Rows r and r ^ 1 land on the same chunk pair and the other three pairs
// of rows on the three other pairs, so every bank takes exactly two of the 256 bytes: two wavefronts, the least for a
// 256-B store.
__device__ __forceinline__ uint32_t stg_frag_addr(const uint32_t stg, const int lane, const int h, const int j) {
  const uint32_t r = (uint32_t)(lane >> 2) + 8u * (uint32_t)h;
  const uint32_t chunk = (uint32_t)(2 * (j & 3) + ((lane >> 1) & 1)) ^ (uint32_t)(lane >> 2);
  return stg + (uint32_t)(j >> 2) * 8192u + r * 128u + (chunk << 4) + (uint32_t)(lane & 1) * 8u;
}

// Fused epilogue of one warpgroup's 64 x BN accumulator in one epilogue mode EPI (and activation ACT), both fixed at
// compile time, so the whole fragment is straight-line code.  Fragment layout of wgmma's D: warp w of the warpgroup owns
// rows 16 w .. 16 w + 15; d[4 j + {0, 1}] are columns 8 j + 2 (lane % 4) + {0, 1} of row lane / 4, d[4 j + {2, 3}] the
// same columns of row lane / 4 + 8.  Four lanes write one whole 32-B sector of a row.
// The fragment is walked in groups of G column pairs: the group's bias pair (shared by both rows) and aux pairs are all
// loaded before any arithmetic on it, so their latencies overlap; G is small enough that the loads fit beside the
// accumulators without spilling.  Each element's arithmetic is that of the FFMA kernel's epi_scalar (gemm.cu), operation
// for operation, so both kernels round alike.
// STAGED: the results go to the warpgroup's staging tile at shared address `stg` instead of global memory (EPI_ATOMIC:
// the bare accumulators, which a TMA reduce-add then adds into C); EPI_ACTGRAD reads aux0 from the same place, where the
// producer has loaded it, and overwrites it in place.  The arithmetic is the same.
template <int BN, int EPI, int ACT, bool VEC, bool STAGED = false>
__device__ __forceinline__ void tc_epilogue_mode(const GemmArgs& a, const float (&d)[BN / 2], const int64_t mw,
                                                 const int64_t n0, const int lane, const uint32_t stg = 0) {
  constexpr int G = (EPI == EPI_CROSS || EPI == EPI_CROSS_DX || EPI == EPI_SCORES) ? 2 : 4;
  constexpr bool BIAS = EPI == EPI_BIAS_ACT || EPI == EPI_CROSS || EPI == EPI_SCORES;
  constexpr bool AUX0 = EPI == EPI_ACTGRAD || EPI == EPI_CROSS || EPI == EPI_CROSS_DX;
  constexpr bool AUX1 = EPI == EPI_CROSS || EPI == EPI_CROSS_DX;
  static_assert((BN / 8) % G == 0, "column groups must tile the fragment");
  static_assert(!STAGED || EPI == EPI_STORE || EPI == EPI_BIAS_ACT || EPI == EPI_ACTGRAD || EPI == EPI_ATOMIC,
                "staged modes write C only");
  const int64_t nl = n0 + 2 * (lane & 3);
  int64_t m[2], row[2];
  bool row_ok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    m[h] = mw + (lane >> 2) + 8 * h;
    row_ok[h] = m[h] < a.M;
    row[h] = m[h] * a.ldc + nl;
  }
  // EPI_SCORES: candidate id of each row's positive, loaded only where epi_scalar_tc reads it
  int64_t rid[2] = {0, 0};
  bool rmask[2] = {false, false};
  if constexpr (EPI == EPI_SCORES) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      rmask[h] = a.cand_ids && row_ok[h] && m[h] + a.row0 < a.N;
      if (rmask[h]) rid[h] = __ldg(a.cand_ids + m[h] + a.row0);
    }
  }
#pragma unroll
  for (int j0 = 0; j0 < BN / 8; j0 += G) {
    float2 bv[G], x0[2][G], x1[2][G];
    int64_t cid[G][2];
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const int64_t n = nl + 8 * (j0 + g);
      const bool col_ok = n < a.N, two = n + 1 < a.N;
      bv[g] = make_float2(0.f, 0.f);
      if constexpr (BIAS) {
        if (a.bias && col_ok) bv[g] = ld_pair<VEC>(a.bias + n, two);
      }
      if constexpr (EPI == EPI_SCORES) {
        cid[g][0] = (rmask[0] || rmask[1]) && col_ok ? __ldg(a.cand_ids + n) : 0;
        cid[g][1] = (rmask[0] || rmask[1]) && two ? __ldg(a.cand_ids + n + 1) : 0;
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if constexpr (AUX0 && STAGED) {   // EPI_ACTGRAD: the producer has loaded aux0's tile into the staging tile
          asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(x0[h][g].x), "=f"(x0[h][g].y)
                       : "r"(stg_frag_addr(stg, lane, h, j0 + g)) : "memory");
        } else if constexpr (AUX0) {
          x0[h][g] = row_ok[h] && col_ok ? ld_pair<VEC>(a.aux0 + row[h] + 8 * (j0 + g), two) : make_float2(0.f, 0.f);
        }
        if constexpr (AUX1) x1[h][g] = row_ok[h] && col_ok ? ld_pair<VEC>(a.aux1 + row[h] + 8 * (j0 + g), two)
                                                           : make_float2(0.f, 0.f);
      }
    }
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const int j = j0 + g;
      const int64_t n = nl + 8 * j;
      if (n >= a.N) continue;
      const bool two = n + 1 < a.N;
      float2 lp = make_float2(0.f, 0.f);   // EPI_SCORES: log p of the column pair, shared by both rows
      if constexpr (EPI == EPI_SCORES) {
        if (a.bias) lp = make_float2(logf(bv[g].x), two ? logf(bv[g].y) : 0.f);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!row_ok[h]) continue;
        const float v0 = d[4 * j + 2 * h], v1 = d[4 * j + 2 * h + 1];
        const int64_t off = row[h] + 8 * j;
        float* c = a.C + off;
        float2 r = make_float2(v0, v1);
        if constexpr (EPI == EPI_ATOMIC) {
          if constexpr (!STAGED) {
            red_add_f32(c, v0);
            if (two) red_add_f32(c + 1, v1);
            continue;
          }
        } else if constexpr (EPI == EPI_BIAS_ACT) {
          r = make_float2(act_apply(v0 + bv[g].x, ACT), act_apply(v1 + bv[g].y, ACT));
        } else if constexpr (EPI == EPI_ACTGRAD) {
          r = make_float2(v0 * act_grad_from_y(x0[h][g].x, ACT), v1 * act_grad_from_y(x0[h][g].y, ACT));
        } else if constexpr (EPI == EPI_CROSS) {
          float2 u = make_float2(v0 + bv[g].x, v1 + bv[g].y);
          if (a.alpha != 0.f) {
            u.x = u.x + a.alpha * x1[h][g].x;
            u.y = u.y + a.alpha * x1[h][g].y;
          }
          if (a.out2) st_pair<VEC>(a.out2 + off, u, two);
          r = make_float2(x0[h][g].x * u.x + x1[h][g].x, x0[h][g].y * u.y + x1[h][g].y);
        } else if constexpr (EPI == EPI_CROSS_DX) {
          r = make_float2(v0 + x1[h][g].x, v1 + x1[h][g].y);
          if (a.alpha != 0.f) {
            r.x += a.alpha * x0[h][g].x;
            r.y += a.alpha * x0[h][g].y;
          }
        } else if constexpr (EPI == EPI_SCORES) {
          if (a.bias) {
            r.x = r.x - lp.x;
            r.y = r.y - lp.y;
          }
          const int64_t q = m[h] + a.row0;
          if (rmask[h] && q != n && cid[g][0] == rid[h]) r.x = r.x + (-FLT_MAX / 100.0f);
          if (rmask[h] && q != n + 1 && cid[g][1] == rid[h]) r.y = r.y + (-FLT_MAX / 100.0f);
        }
        if constexpr (STAGED) {
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(stg_frag_addr(stg, lane, h, j)), "f"(r.x), "f"(r.y)
                       : "memory");
        } else {
          st_pair<VEC>(c, r, two);
        }
      }
    }
  }
}

template <int BN, int EPI, int ACT, bool STAGED = false>
__device__ __forceinline__ void tc_epilogue_vec(const GemmArgs& a, const float (&d)[BN / 2], const int64_t mw,
                                                const int64_t n0, const int lane, const bool vec_ok,
                                                const uint32_t stg = 0) {
  if (vec_ok) tc_epilogue_mode<BN, EPI, ACT, true, STAGED>(a, d, mw, n0, lane, stg);
  else tc_epilogue_mode<BN, EPI, ACT, false, STAGED>(a, d, mw, n0, lane, stg);
}

template <int BN, int EPI, bool STAGED = false>
__device__ __forceinline__ void tc_epilogue_act(const GemmArgs& a, const float (&d)[BN / 2], const int64_t mw,
                                                const int64_t n0, const int lane, const bool vec_ok,
                                                const uint32_t stg = 0) {
  switch (a.act) {
    case DR_ACT_RELU: tc_epilogue_vec<BN, EPI, DR_ACT_RELU, STAGED>(a, d, mw, n0, lane, vec_ok, stg); return;
    case DR_ACT_SIGMOID: tc_epilogue_vec<BN, EPI, DR_ACT_SIGMOID, STAGED>(a, d, mw, n0, lane, vec_ok, stg); return;
    case DR_ACT_TANH: tc_epilogue_vec<BN, EPI, DR_ACT_TANH, STAGED>(a, d, mw, n0, lane, vec_ok, stg); return;
    default: tc_epilogue_vec<BN, EPI, DR_ACT_NONE, STAGED>(a, d, mw, n0, lane, vec_ok, stg); return;
  }
}

// The epilogue mode (and the activation, where it matters) is chosen once per tile, not once per element.
// `vec_ok`: C, every auxiliary operand and the bias are 8-B aligned and ldc and N are even, so every column pair is one
// float2 access.
template <int BN>
__device__ __forceinline__ void tc_epilogue(const GemmArgs& a, const float (&d)[BN / 2], const int64_t mw, const int64_t n0,
                                            const int lane, const bool vec_ok) {
  switch (a.epi) {
    case EPI_BIAS_ACT: tc_epilogue_act<BN, EPI_BIAS_ACT>(a, d, mw, n0, lane, vec_ok); return;
    case EPI_ATOMIC: tc_epilogue_mode<BN, EPI_ATOMIC, DR_ACT_NONE, false>(a, d, mw, n0, lane); return;
    case EPI_ACTGRAD: tc_epilogue_act<BN, EPI_ACTGRAD>(a, d, mw, n0, lane, vec_ok); return;
    case EPI_CROSS: tc_epilogue_vec<BN, EPI_CROSS, DR_ACT_NONE>(a, d, mw, n0, lane, vec_ok); return;
    case EPI_CROSS_DX: tc_epilogue_vec<BN, EPI_CROSS_DX, DR_ACT_NONE>(a, d, mw, n0, lane, vec_ok); return;
    case EPI_SCORES: tc_epilogue_vec<BN, EPI_SCORES, DR_ACT_NONE>(a, d, mw, n0, lane, vec_ok); return;
    default: tc_epilogue_vec<BN, EPI_STORE, DR_ACT_NONE>(a, d, mw, n0, lane, vec_ok); return;
  }
}

// The modes whose only output is C (tc_staged_ok) write the warpgroup's staging tile at `stg`.
template <int BN>
__device__ __forceinline__ void tc_epilogue_staged(const GemmArgs& a, const float (&d)[BN / 2], const int64_t mw,
                                                   const int64_t n0, const int lane, const bool vec_ok,
                                                   const uint32_t stg) {
  switch (a.epi) {
    case EPI_BIAS_ACT: tc_epilogue_act<BN, EPI_BIAS_ACT, true>(a, d, mw, n0, lane, vec_ok, stg); return;
    case EPI_ATOMIC: tc_epilogue_mode<BN, EPI_ATOMIC, DR_ACT_NONE, false, true>(a, d, mw, n0, lane, stg); return;
    case EPI_ACTGRAD: tc_epilogue_act<BN, EPI_ACTGRAD, true>(a, d, mw, n0, lane, vec_ok, stg); return;
    default: tc_epilogue_mode<BN, EPI_STORE, DR_ACT_NONE, false, true>(a, d, mw, n0, lane, stg); return;
  }
}

// EPI_CROSS_DX_ACC (C += acc + alpha*aux0 + aux1) is a compile-time form with kernels of its own (gemm_tc_acc_kernel).
template <int BN>
__device__ __forceinline__ void tc_epilogue_acc(const GemmArgs& a, const float (&d)[BN / 2], const int64_t mw,
                                                const int64_t n0, const int lane) {
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int64_t m = mw + (lane >> 2) + 8 * half;
    if (m >= a.M) continue;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int64_t n = n0 + 8 * j + 2 * (lane & 3);
      if (n >= a.N) continue;
      const float v0 = d[4 * j + 2 * half], v1 = d[4 * j + 2 * half + 1];
      float* c = a.C + m * a.ldc + n;
      const int64_t off = m * a.ldc + n;
      c[0] += v0 + a.alpha * __ldg(a.aux0 + off) + __ldg(a.aux1 + off);
      if (n + 1 < a.N) c[1] += v1 + a.alpha * __ldg(a.aux0 + off + 1) + __ldg(a.aux1 + off + 1);
    }
  }
}

// Shared-memory stages of one tile width.  The plane ring holds [Ah | Al | Bh | Bl] in variant 1 and [Bh | Bl] in
// variant 2, whose consumers split A in registers; the raw ring (variant 2 only) holds [A raw | B raw], or
// [A raw | Bh | Bl] in the weight-plane kernel, which has no plane ring.  A launch with the staged epilogue adds the
// 128 x BN staging tile after the rings.  MAX_RAW: the deepest raw ring launched; STAGED_RAW: the deepest that leaves
// room for the staging tile (3 for the weight-plane kernel at BN = 128, whose 4-deep ring takes 192 KB).
constexpr size_t TC_SMEM_LIMIT = 232448;   // 227 KB of shared memory per CTA
constexpr size_t TC_STATIC_SMEM = 2048;     // the barriers: ptxas pads them to 1 KB granules ahead of the ring
template <int BN, bool PRESPLIT, bool WPLANES = false>
struct TcSmem {
  static constexpr int A_TILE = TC_BM * TC_BK * 4;   // 16 KB
  static constexpr int B_TILE = BN * TC_BK * 4;
  static constexpr int STG = TC_BM * BN * 4;
  static constexpr int PLANE_STAGE = WPLANES ? 0 : (PRESPLIT ? 2 * A_TILE : 0) + 2 * B_TILE;
  static constexpr int RAW_STAGE = PRESPLIT ? 0 : A_TILE + (WPLANES ? 2 : 1) * B_TILE;
  static constexpr int MAX_RAW = PRESPLIT ? 0 : (WPLANES ? TC_WP_STAGES : TC_RAW_STAGES);
  static constexpr size_t bytes(int raw_stages, bool staged) {   // + 1024: the ring base is rounded up to 1024 B
    return (size_t)TC_PLANE_STAGES * PLANE_STAGE + (size_t)raw_stages * RAW_STAGE + (staged ? STG : 0) + 1024;
  }
  // + TC_STATIC_SMEM: the static shared memory beside the dynamic ring
  static constexpr int STAGED_RAW = bytes(MAX_RAW, true) + TC_STATIC_SMEM <= TC_SMEM_LIMIT ? MAX_RAW : MAX_RAW - 1;
};

// A consumer thread's A-fragment elements in the raw A stage.  `a_frag_base`: byte offset of element 0 of k-step 0 (row
// r = the thread's fragment row, column lane % 4); `a_frag_ld`: element e of k-step ks, at that offset from the stage.
//   K-major: SWIZZLE_128B rows of 32 floats, 16-B chunk c of row r at chunk c ^ (r & 7).  The stage is 1024-B aligned, so
//   bits 4-6 of (stage + base) are r & 7 and chunk c of the same row is (stage + base) ^ (c << 4); row r + 8 is 1024 B
//   further.  A warp's 8 rows x 4 consecutive k hit 32 distinct banks.
//   MN-major: [32 k][128 rows] as stored, element (r, k) at (k * 128 + r) * 4.
// The lane index is re-read from %laneid on every call: held in a register instead, the offset would stay live across
// the epilogue, which needs all 128 registers at BN = 128.
template <bool A_MN>
__device__ __forceinline__ uint32_t a_frag_base(const int warp_row0) {
  uint32_t lane;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane));
  const int row = warp_row0 + (int)(lane >> 2), col = (int)(lane & 3);
  if constexpr (A_MN) return (uint32_t)(col * TC_BM + row) * 4u;
  else return (uint32_t)(row * TC_BK + ((row & 7) << 2) + col) * 4u;
}
template <bool A_MN>
__device__ __forceinline__ float a_frag_ld(const uint32_t at, const int ks, const int e) {
  uint32_t p;
  if constexpr (A_MN) p = at + (uint32_t)((8 * ks + 4 * (e >> 1)) * TC_BM + 8 * (e & 1)) * 4u;
  else p = (at ^ (uint32_t)((2 * ks + (e >> 1)) << 4)) + (uint32_t)(e & 1) * 1024u;
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(p));   // volatile: stays after the raw_full wait
  return v;
}

template <int N>
struct TcWidth { static constexpr int value = N; };

// Persistent, warp-specialised.  `raw_stages` (run-time: 2 to 4) is the depth of the raw ring; the plane ring is two deep.
// Shared memory: planes 2 x TcSmem::PLANE_STAGE, then (variant 2) raw_stages x [A raw | B raw].
// WPLANES (A and B K-major, !PRESPLIT): the ring is raw_stages x [A raw | Bh | Bl] with B's planes loaded by TMA
// (tmBh / tmBl); the threads are the consumers and the TMA warp only.
template <int BN, bool A_MN, bool B_MN, bool PRESPLIT, bool ACC, bool WPLANES = false>
__device__ __forceinline__ void gemm_tc_body(const CUtensorMap& tmAh, const CUtensorMap& tmAl, const CUtensorMap& tmBh,
                                             const CUtensorMap& tmBl, const CUtensorMap& tmC, const CUtensorMap& tmAux,
                                             const GemmArgs& a,
                                             const int raw_stages, const int staged, const int64_t m_tiles,
                                             const int64_t n_tiles, const int64_t per, const int64_t total_items) {
  static_assert(!WPLANES || (!PRESPLIT && !A_MN && !B_MN && !ACC), "weight planes: K-major A split in registers");
  using S = TcSmem<BN, PRESPLIT, WPLANES>;
  constexpr int A_TILE = S::A_TILE, B_TILE = S::B_TILE, PLANE_STAGE = S::PLANE_STAGE, RAW_STAGE = S::RAW_STAGE;
  constexpr int PRODUCER_WARP = (TC_CONSUMERS + (WPLANES ? 0 : TC_SPLITTERS)) / 32;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* planes = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* raws = planes + TC_PLANE_STAGES * PLANE_STAGE;
  uint8_t* stage_tile = raws + (size_t)raw_stages * RAW_STAGE;   // staged epilogue: 64 x BN per consumer warpgroup
  __shared__ __align__(8) uint64_t raw_full[TC_MAX_RAW_STAGES], raw_empty[TC_MAX_RAW_STAGES],
      pl_full[TC_PLANE_STAGES], pl_empty[TC_PLANE_STAGES];
  // staged EPI_ACTGRAD, per consumer warpgroup: aux0's tile has landed in the staging tile / the TMA store of the
  // previous tile has read it
  __shared__ __align__(8) uint64_t aux_full[2], stg_free[2];
  const bool aux_tma = staged && a.epi == EPI_ACTGRAD;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t kblocks = (a.K + TC_BK - 1) / TC_BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < TC_MAX_RAW_STAGES; ++s) {
      mbar_init(&raw_full[s], 1);                    // the producer's expect_tx arrival
      // every splitter (B) and consumer (A) thread arrives; with weight planes, every consumer once the stage has retired
      mbar_init(&raw_empty[s], (WPLANES ? 0 : TC_SPLITTERS) + TC_CONSUMERS);
    }
    for (int s = 0; s < TC_PLANE_STAGES; ++s) {
      mbar_init(&pl_full[s], PRESPLIT ? 1 : TC_SPLITTERS);
      mbar_init(&pl_empty[s], TC_CONSUMERS);         // every consumer thread arrives
    }
    for (int w = 0; w < 2; ++w) {
      mbar_init(&aux_full[w], 1);                    // the producer's expect_tx arrival
      mbar_init(&stg_free[w], 1);                    // the warpgroup's leader, once its store has read the tile
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (warp == PRODUCER_WARP) {
    if (lane == 0) {
      // ===== TMA producer =====
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmAh) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmBh) : "memory");
      if (WPLANES) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmBl) : "memory");
      uint32_t it = 0, aux_it[2] = {0, 0};
      for (int64_t item = blockIdx.x; item < total_items; item += gridDim.x) {
        const TcItem t = tc_decode(item, n_tiles, m_tiles, kblocks, per, BN);
        // staged EPI_ACTGRAD: aux0's 64 x BN block of each warpgroup with rows in range, behind the tile's last k-block
        // (by then the consumers are past the previous tile's epilogue), once the warpgroup's previous store has read
        // the staging tile
        auto load_aux = [&]() {
          const int boxes = (int)min((int64_t)(BN / 32), (a.N - t.n0 + 31) / 32);
          for (int w = 0; w < 2; ++w) {
            if (t.m0 + 64 * w >= a.M) continue;
            mbar_wait(&stg_free[w], (aux_it[w] & 1u) ^ 1u);
            ++aux_it[w];
            mbar_expect_tx(&aux_full[w], (uint32_t)boxes * (64u * 128u));
            for (int q = 0; q < boxes; ++q)
              tma_load_2d(stage_tile + (size_t)w * (64 * BN * 4) + q * (64 * 128), &tmAux, &aux_full[w],
                          (int)(t.n0 + 32 * q), (int)(t.m0 + 64 * w));
          }
        };
        for (int i = 0; i < t.nkb; ++i, ++it) {
          const int k = (t.kb0 + i) * TC_BK;
          if (PRESPLIT) {      // K-major planes from the workspace straight into the plane ring
            const int s = (int)(it % TC_PLANE_STAGES);
            mbar_wait(&pl_empty[s], ((it / TC_PLANE_STAGES) & 1u) ^ 1u);
            mbar_expect_tx(&pl_full[s], (uint32_t)PLANE_STAGE);
            uint8_t* st = planes + (size_t)s * PLANE_STAGE;
            tma_load_2d(st, &tmAh, &pl_full[s], k, (int)t.m0);
            tma_load_2d(st + A_TILE, &tmAl, &pl_full[s], k, (int)t.m0);
            tma_load_2d(st + 2 * A_TILE, &tmBh, &pl_full[s], k, (int)t.n0);
            tma_load_2d(st + 2 * A_TILE + B_TILE, &tmBl, &pl_full[s], k, (int)t.n0);
          } else {
            const int s = (int)(it % (uint32_t)raw_stages);
            mbar_wait(&raw_empty[s], ((it / (uint32_t)raw_stages) & 1u) ^ 1u);
            mbar_expect_tx(&raw_full[s], (uint32_t)RAW_STAGE);
            uint8_t* st = raws + (size_t)s * RAW_STAGE;
            if (!A_MN) tma_load_2d(st, &tmAh, &raw_full[s], k, (int)t.m0);
            else tma_load_2d(st, &tmAh, &raw_full[s], (int)t.m0, k);
            if (!B_MN) tma_load_2d(st + A_TILE, &tmBh, &raw_full[s], k, (int)t.n0);
            else tma_load_2d(st + A_TILE, &tmBh, &raw_full[s], (int)t.n0, k);
            if (WPLANES) tma_load_2d(st + A_TILE + B_TILE, &tmBl, &raw_full[s], k, (int)t.n0);
          }
          if (aux_tma && i + 1 == t.nkb) load_aux();
        }
      }
    }
  } else if (threadIdx.x >= TC_CONSUMERS) {
    // ===== splitter warps: raw fp32 B tile -> TF32 hi / lo planes, K-major =====
    if (!PRESPLIT && !WPLANES) {
      const int tid = (int)threadIdx.x - TC_CONSUMERS;
      uint32_t it = 0;
      for (int64_t item = blockIdx.x; item < total_items; item += gridDim.x) {
        const TcItem t = tc_decode(item, n_tiles, m_tiles, kblocks, per, BN);
        for (int i = 0; i < t.nkb; ++i, ++it) {
          const int s = (int)(it % (uint32_t)raw_stages), p = (int)(it % TC_PLANE_STAGES);
          mbar_wait(&raw_full[s], (it / (uint32_t)raw_stages) & 1u);        // TMA bytes of this stage have landed
          mbar_wait(&pl_empty[p], ((it / TC_PLANE_STAGES) & 1u) ^ 1u);      // wgmma has finished reading the planes
          const uint8_t* rw = raws + (size_t)s * RAW_STAGE;
          uint8_t* pl = planes + (size_t)p * PLANE_STAGE;
          split_tile<BN, B_MN>(rw + A_TILE, pl, pl + B_TILE, tid);
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to wgmma
          mbar_arrive(&pl_full[p]);
          mbar_arrive(&raw_empty[s]);
        }
      }
    }
  } else {
    // ===== consumer warpgroups: rows [64 wg, 64 wg + 64) of the tile =====
    const int wg = warp >> 2;
    const bool vec_ok = ((a.ldc & 1) == 0) && ((a.N & 1) == 0) &&
                        (((reinterpret_cast<uintptr_t>(a.C) | reinterpret_cast<uintptr_t>(a.bias) |
                           reinterpret_cast<uintptr_t>(a.aux0) | reinterpret_cast<uintptr_t>(a.aux1) |
                           reinterpret_cast<uintptr_t>(a.out2)) & 7u) == 0);
    uint32_t it = 0, aux_it = 0;
    for (int64_t item = blockIdx.x; item < total_items; item += gridDim.x) {
      const TcItem t = tc_decode(item, n_tiles, m_tiles, kblocks, per, BN);
      if (t.m0 + wg * 64 >= a.M) {
        // M tail: none of this warpgroup's rows is in range.  It only makes the arrivals the other warps' waits count,
        // each after the wait that opens its phase, so that no arrival lands in an earlier phase.
        for (int i = 0; i < t.nkb; ++i, ++it) {
          const int p = (int)(it % TC_PLANE_STAGES);
          if (!WPLANES) mbar_wait(&pl_full[p], (it / TC_PLANE_STAGES) & 1u);
          if (!PRESPLIT) {   // variant 1 has no raw ring (raw_stages = 0)
            const int s = (int)(it % (uint32_t)raw_stages);
            mbar_wait(&raw_full[s], (it / (uint32_t)raw_stages) & 1u);
            mbar_arrive(&raw_empty[s]);
          }
          if (!WPLANES) mbar_arrive(&pl_empty[p]);
        }
        continue;
      }
      float d[BN / 2];
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) d[j] = 0.f;
      // k-blocks of the in-register A split, NW-wide MMAs into the leading NW / 2 accumulators (NW < BN: the tile's
      // valid columns all lie in the first NW, the other accumulators stay zero)
      auto kblocks_ra = [&](auto width) {
        constexpr int NW = decltype(width)::value;
        float (&dn)[NW / 2] = reinterpret_cast<float (&)[NW / 2]>(d);
        for (int i = 0; i < t.nkb; ++i, ++it) {
          // A straight from the raw stage: each thread splits its own fragment elements as split_tile does and feeds
          // them to wgmma from registers, one commit group per k-step.  The fragment is rewritten only after the
          // previous k-step has retired (wait_group 0); the other consumer warpgroup keeps the tensor cores busy
          // meanwhile, and each k-step's loads are issued before its wait.  A two-buffer form (wait_group 1 after each
          // commit) compiles to the same 128 registers, measured no faster on H100, and produced wrong dX values in
          // the full-size Dense test (K = 32, N = 256), for a reason not yet found.
          const int s = (int)(it % (uint32_t)raw_stages), p = (int)(it % TC_PLANE_STAGES);
          if (!WPLANES) mbar_wait(&pl_full[p], (it / TC_PLANE_STAGES) & 1u);
          mbar_wait(&raw_full[s], (it / (uint32_t)raw_stages) & 1u);
          const uint32_t at = smem_u32(raws + (size_t)s * RAW_STAGE) + a_frag_base<A_MN>(wg * 64 + (warp & 3) * 16);
          const uint32_t sb = WPLANES ? smem_u32(raws + (size_t)s * RAW_STAGE) + A_TILE
                                      : smem_u32(planes + (size_t)p * PLANE_STAGE);
#pragma unroll
          for (int k = 0; k < TC_BK / 8; ++k) {
            float v[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) v[e] = a_frag_ld<A_MN>(at, k, e);
            wgmma_wait<0>();
            if (k == 0 && i > 0) {   // k-block i - 1 has retired: its B planes (its whole stage, WPLANES) are free
              if (WPLANES) mbar_arrive(&raw_empty[(it - 1) % (uint32_t)raw_stages]);
              else mbar_arrive(&pl_empty[p ^ 1]);
            }
            uint32_t ah[4], al[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float h = __uint_as_float(__float_as_uint(v[e]) & 0xFFFFE000u);
              ah[e] = __float_as_uint(h);
              al[e] = __float_as_uint(v[e] - h);
            }
            if (!WPLANES && k + 1 == TC_BK / 8) mbar_arrive(&raw_empty[s]);   // every A element of the stage is in registers
            const uint64_t dBh = make_smem_desc(sb + k * 32), dBl = make_smem_desc(sb + B_TILE + k * 32);
            wgmma_fence();
            wgmma_tf32_ra<NW>(dn, al, dBh);   // small cross terms first, as in variant 1
            wgmma_tf32_ra<NW>(dn, ah, dBl);
            wgmma_tf32_ra<NW>(dn, ah, dBh);
            wgmma_commit();
          }
        }
      };
      if constexpr (PRESPLIT) {
        for (int i = 0; i < t.nkb; ++i, ++it) {
          const int p = (int)(it % TC_PLANE_STAGES);
          mbar_wait(&pl_full[p], (it / TC_PLANE_STAGES) & 1u);
          const uint32_t sa = smem_u32(planes + (size_t)p * PLANE_STAGE) + (uint32_t)wg * (64u * 128u);
          const uint32_t sb = smem_u32(planes + (size_t)p * PLANE_STAGE) + 2 * A_TILE;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < TC_BK / 8; ++k) {
            const uint64_t dAh = make_smem_desc(sa + k * 32), dAl = make_smem_desc(sa + A_TILE + k * 32);
            const uint64_t dBh = make_smem_desc(sb + k * 32), dBl = make_smem_desc(sb + B_TILE + k * 32);
            wgmma_tf32<BN>(d, dAl, dBh);   // small cross terms first
            wgmma_tf32<BN>(d, dAh, dBl);
            wgmma_tf32<BN>(d, dAh, dBh);
          }
          wgmma_commit();
          if (i > 0) {                     // the previous k-block has retired: its planes may be overwritten
            wgmma_wait<1>();
            mbar_arrive(&pl_empty[p ^ 1]);
          }
        }
      } else if constexpr (WPLANES && BN > 32) {
        // N tail: the last n-tile of N = 416 at BN = 128 has 32 valid columns.  One MMA width per tile, each with a
        // k-loop of its own, so the loop carries no width test.
        const int64_t w = a.N - t.n0;
        if (w <= 32) kblocks_ra(TcWidth<32>{});
        else if (BN > 64 && w <= 64) kblocks_ra(TcWidth<64>{});
        else kblocks_ra(TcWidth<BN>{});
      } else {
        kblocks_ra(TcWidth<BN>{});
      }
      wgmma_wait<0>();
      if (WPLANES) mbar_arrive(&raw_empty[(it - 1) % (uint32_t)raw_stages]);
      else mbar_arrive(&pl_empty[(it - 1) % TC_PLANE_STAGES]);
      const int64_t mw = t.m0 + wg * 64 + (warp & 3) * 16;
      if constexpr (ACC) {
        tc_epilogue_acc<BN>(a, d, mw, t.n0, lane);
      } else if (staged) {
        // Staged epilogue: the warpgroup writes its 64 x BN results into its staging tile and one thread hands the
        // tile to TMA (a store, or a reduce-add for split-K), which drains it while the warpgroup runs the next tile's
        // MMAs.  The tile is rewritten only after the previous tile's TMA has finished reading it.
        const bool leader = (threadIdx.x & 127) == 0;
        uint8_t* stg = stage_tile + (size_t)wg * (64 * BN * 4);
        if (leader) bulk_wait_read0();
        named_barrier_sync(1 + wg, 128);
        if (aux_tma) mbar_wait(&aux_full[wg], (aux_it++) & 1u);
        tc_epilogue_staged<BN>(a, d, mw, t.n0, lane, vec_ok, smem_u32(stg) + (uint32_t)(warp & 3) * (16u * 128u));
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to TMA
        named_barrier_sync(1 + wg, 128);
        if (leader) {
          // TMA clips the rows past M and the columns past N; a box wholly past N is not issued
          for (int q = 0; q < BN / 32 && t.n0 + 32 * q < a.N; ++q)
            tma_store_2d(&tmC, stg + q * (64 * 128), (int)(t.n0 + 32 * q), (int)(t.m0 + 64 * wg), a.epi == EPI_ATOMIC);
          bulk_commit();
          if (aux_tma) {   // the producer loads the next tile's aux0 block here
            bulk_wait_read0();
            mbar_arrive(&stg_free[wg]);
          }
        }
      } else {
        tc_epilogue<BN>(a, d, mw, t.n0, lane, vec_ok);
      }
    }
    if (staged && (threadIdx.x & 127) == 0) bulk_wait0();
  }
}

// Registers are allocated to warps in groups of four, so 13 warps count as 16: 65536 / 512 = 128 registers per thread.
// The BN = 128 instantiations hold 64 accumulators and use all 128.  The variant-2 ones (A split in registers) spill one
// 4-byte value: stored once before the consumers' tile loop and reloaded once after it, outside the k-loop.
template <int BN, bool A_MN, bool B_MN, bool PRESPLIT>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
               const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl,
               const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmAux, const GemmArgs a,
               const int raw_stages, const int staged, const int64_t m_tiles, const int64_t n_tiles, const int64_t per,
               const int64_t total_items) {
  gemm_tc_body<BN, A_MN, B_MN, PRESPLIT, false>(tmAh, tmAl, tmBh, tmBl, tmC, tmAux, a, raw_stages, staged, m_tiles, n_tiles, per,
                                                total_items);
}

// EPI_CROSS_DX_ACC: the only GEMM that accumulates into C is the Cross input gradient h @ W^T, both operands K-major.
template <int BN, bool PRESPLIT>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_acc_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
                   const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl,
                   const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmAux,
                   const GemmArgs a, const int raw_stages, const int staged, const int64_t m_tiles,
                   const int64_t n_tiles, const int64_t per, const int64_t total_items) {
  gemm_tc_body<BN, false, false, PRESPLIT, true>(tmAh, tmAl, tmBh, tmBl, tmC, tmAux, a, raw_stages, 0, m_tiles, n_tiles, per,
                                                 total_items);
}

// Weight planes: K-major raw A (tmAh) split in registers, B's K-major hi / lo planes (tmBh / tmBl) from the workspace.
// 9 warps count as 12 for register allocation: up to 168 registers per thread, so the BN = 128 epilogue does not spill.
template <int BN>
__global__ void __launch_bounds__(TC_WP_THREADS, 1)
gemm_tc_wplanes_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
                       const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl,
                       const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmAux,
                       const GemmArgs a, const int raw_stages, const int staged, const int64_t m_tiles,
                       const int64_t n_tiles, const int64_t per, const int64_t total_items) {
  gemm_tc_body<BN, false, false, false, false, true>(tmAh, tmAl, tmBh, tmBl, tmC, tmAux, a, raw_stages, staged, m_tiles,
                                                     n_tiles, per, total_items);
}

// ---- host side ---------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;

static int get_encode() {
  if (g_encode) return DR_OK;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
    set_error("gemm_tc: cuTensorMapEncodeTiled entry point not available (%s)", cudaGetErrorString(e));
    return e != cudaSuccess ? (int)e : DR_ENOTSUP;
  }
  g_encode = (EncodeTiledFn)fn;
  return DR_OK;
}

// 2-D fp32 tensor [outer, inner] (inner contiguous, pitch floats), box {box_inner, box_outer}.  K-major operand tiles
// are boxes {32, rows} in SWIZZLE_128B (the layout wgmma reads); MN-major ones are boxes {rows, 32} staged unswizzled
// for the transposing splitter pass.
static int make_map(CUtensorMap* tm, const float* base, int64_t inner, int64_t outer, int64_t pitch, int box_inner,
                    int box_outer, bool swizzle) {
  cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t strides[1] = {(cuuint64_t)pitch * 4};
  cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = g_encode(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                        // K-major operand: consecutive k-blocks of a tile walk along each row 128 B at a time -- fetch 256 B
                        // per L2 miss so every second k-block finds its rows in L2 (knob tc_l2_promo: 128 / 256)
                        (swizzle && g_tune_tc_l2_promo == 256) ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B
                                                               : CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("gemm_tc: cuTensorMapEncodeTiled failed (CUresult %d; inner=%lld outer=%lld pitch=%lld)", (int)r,
              (long long)inner, (long long)outer, (long long)pitch);
    return DR_EINVAL;
  }
  return DR_OK;
}

static inline int64_t round4(int64_t v) { return (v + 3) & ~(int64_t)3; }

// Sizes (floats) of the K-major hi/lo planes of variant 1: A -> [M, pitch], B -> [N, pitch].  An operand that is
// already K-major keeps its source pitch (one flat float4 pass); a transposed one gets round4(K).
static void plane_elems(const GemmArgs& a, bool ta, bool tb, size_t* ae, size_t* be) {
  const int64_t kp = round4(a.K);
  *ae = (size_t)a.M * (size_t)(!ta ? a.lda : kp);
  *be = (size_t)a.N * (size_t)(tb ? a.ldb : kp);
}

static const PlaneEntry* plane_cached(const float* src, bool transposed, int64_t rows, int64_t K, int64_t ld) {
  for (int i = 0; i < g_nplanes; ++i) {
    const PlaneEntry& e = g_planes[i];
    if (e.src == src && e.transposed == transposed && e.rows == rows && e.K == K && e.ld == ld) return &e;
  }
  return nullptr;
}

bool gemm_tc_eligible(const GemmArgs& a, bool ta, bool tb) {
  if (g_tune_gemm_variant != 1 && g_tune_gemm_variant != 2) return false;
  if (a.N < g_tune_tc_min_n || (a.N & 3) || a.M < 64 || a.K < 32) return false;
  if (a.M >= ((int64_t)1 << 31) || a.K >= ((int64_t)1 << 31) || a.N >= ((int64_t)1 << 31)) return false;
  if (a.epi == EPI_CROSS_DX_ACC && (ta || !tb)) return false;     // accumulate form: K-major operands only (gemm_tc_acc_kernel)
  if (g_tune_gemm_variant == 2)     // in-kernel split: raw operands by TMA, no workspace
    return !((a.lda & 3) || !aligned16(a.A) || (a.ldb & 3) || !aligned16(a.B));
  // operands already K-major are split in place with float4 accesses
  if (!ta && ((a.lda & 3) || !aligned16(a.A))) return false;
  if (tb && ((a.ldb & 3) || !aligned16(a.B))) return false;
  // that flat split reads rows * ld floats from the operand's first element: a K-major operand whose pitch is wider than
  // K (a column block of a wider matrix, as the grouped Dense passes) would be read past its last row, so it goes to FFMA
  if ((!ta && a.lda != a.K) || (tb && a.ldb != a.K)) return false;
  if (!g_ws_ptr) return false;
  size_t ae, be;
  plane_elems(a, ta, tb, &ae, &be);
  size_t need = 0;
  if (!(g_cache_on && plane_cached(a.A, ta, a.M, a.K, a.lda))) need += 2 * ae;
  if (!(g_cache_on && plane_cached(a.B, !tb, a.N, a.K, a.ldb))) need += 2 * be;
  return ((g_cache_on ? g_bump : 0) + need) * sizeof(float) <= g_ws_bytes;
}

int g_tune_tc_stages = 0;    // 0 = three raw stages; 2 = two (32 KB less shared memory at the widest tile)
int g_tune_tc_pair = 1;      // accepted and read back for callers that set it; H100 has no two-CTA MMA, so it selects nothing

// The staged epilogue serves the modes whose only output is C, when TMA can address C (16-B aligned base, ldc % 4 == 0).
// EPI_ACTGRAD's aux0 (pitch ldc, as C) is loaded by TMA into the staging tile, so it must be 16-B aligned too.
static bool tc_staged_ok(const GemmArgs& a) {
  return (a.epi == EPI_STORE || a.epi == EPI_BIAS_ACT || a.epi == EPI_ACTGRAD || a.epi == EPI_ATOMIC) &&
         aligned16(a.C) && (a.ldc & 3) == 0 && (a.epi != EPI_ACTGRAD || aligned16(a.aux0));
}

// `tms`: the operand maps [Ah, Al, Bh, Bl] and room for C's and aux0's.  `raw_stages`: the ring depth of the register epilogue.
// A splitter kernel with the two-stage ring (it runs beside another kernel) keeps the register epilogue and its smaller
// shared-memory footprint; the weight-plane kernel gives up a ring stage for the staging tile where both do not fit.
template <int BN, bool A_MN, bool B_MN, bool PRESPLIT, bool WPLANES = false>
static int launch_tc(CUtensorMap* tms, const GemmArgs& a, int raw_stages, cudaStream_t st) {
  using S = TcSmem<BN, PRESPLIT, WPLANES>;
  static_assert(S::bytes(S::MAX_RAW, false) + TC_STATIC_SMEM <= TC_SMEM_LIMIT &&
                    S::bytes(S::STAGED_RAW, true) + TC_STATIC_SMEM <= TC_SMEM_LIMIT,
                "the rings and the staging tile exceed the 227 KB of shared memory per CTA");
  auto k = gemm_tc_kernel<BN, A_MN, B_MN, PRESPLIT>;
  if constexpr (WPLANES) k = gemm_tc_wplanes_kernel<BN>;
  if constexpr (!A_MN && !B_MN && BN <= 64 && !WPLANES) {
    if (a.epi == EPI_CROSS_DX_ACC) k = gemm_tc_acc_kernel<BN, PRESPLIT>;
  }
  const bool staged = tc_staged_ok(a) && raw_stages != 2;
  if (staged) {
    raw_stages = raw_stages < S::STAGED_RAW ? raw_stages : S::STAGED_RAW;
    // boxes of 64 rows x 32 floats (one warpgroup's rows, one 128-B swizzle row), in the staging tile's layout
    if (int rc = make_map(&tms[4], a.C, a.N, a.M, a.ldc, 32, 64, true)) return rc;
    if (a.epi == EPI_ACTGRAD)
      if (int rc = make_map(&tms[5], a.aux0, a.N, a.M, a.ldc, 32, 64, true)) return rc;
  }
  const size_t smem = S::bytes(raw_stages, staged);
  DR_CUDA_CALL(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t m_tiles = (a.M + TC_BM - 1) / TC_BM, n_tiles = (a.N + BN - 1) / BN;
  const int64_t kblocks = (a.K + TC_BK - 1) / TC_BK;
  const int64_t per = (kblocks + a.splitk - 1) / a.splitk;
  const int64_t splits = (kblocks + per - 1) / per;          // every split owns >= 1 k-block
  const int64_t total = m_tiles * n_tiles * splits;
  const int64_t ctas = total < (int64_t)num_sms() ? total : (int64_t)num_sms();
  k<<<(unsigned)ctas, WPLANES ? TC_WP_THREADS : TC_THREADS, smem, st>>>(tms[0], tms[1], tms[2], tms[3], tms[4], tms[5], a,
                                                                         raw_stages, staged ? 1 : 0, m_tiles, n_tiles,
                                                                         per, total);
  DR_CUDA_LAUNCH_CHECK("gemm_tc");
  return DR_OK;
}

// Produce K-major hi/lo planes [rows, pitch] of an operand.  `stored_k_major`: src is [rows, K] with
// pitch ld (flat split, same pitch); otherwise src is [K, rows] with pitch ld (transpose-split).
static int make_planes(const float* src, bool stored_k_major, int64_t rows, int64_t K, int64_t ld, float* hi,
                       float* lo, int64_t* pitch_out, cudaStream_t st) {
  if (stored_k_major) {
    const int64_t n4 = rows * ld / 4;
    int64_t ctas = (n4 + 255) / 256;
    if (ctas > num_sms() * 8) ctas = num_sms() * 8;
    if (ctas < 1) ctas = 1;
    split_tf32_kernel<<<(unsigned)ctas, 256, 0, st>>>(src, n4, hi, lo);
    DR_CUDA_LAUNCH_CHECK("split_tf32");
    *pitch_out = ld;
  } else {
    const int64_t kp = round4(K);
    const int64_t tiles = ((K + 31) / 32) * ((rows + 31) / 32);
    int64_t ctas = tiles < (int64_t)num_sms() * 16 ? tiles : (int64_t)num_sms() * 16;
    if (ctas < 1) ctas = 1;
    split_tf32_transpose_kernel<<<(unsigned)ctas, dim3(32, 8), 0, st>>>(src, K, rows, ld, kp, hi, lo);
    DR_CUDA_LAUNCH_CHECK("split_tf32_transpose");
    *pitch_out = kp;
  }
  return DR_OK;
}

int gemm_tc_launch(const GemmArgs& a0, bool ta, bool tb, cudaStream_t st) {
  GemmArgs a = a0;
  if (int rc = get_encode()) return rc;
  if (a.splitk < 1) a.splitk = 1;
  const int64_t kblocks = (a.K + TC_BK - 1) / TC_BK;
  if (a.splitk > kblocks) a.splitk = (int)kblocks;
  // skinny outputs (the 256->32 tower layer and its weight gradient) get a 128 x 32 / 128 x 64 tile
  int bn = a.N <= 32 ? 32 : (a.N <= 64 ? 64 : 128);
  if (g_tune_gemm_bn == 32 || g_tune_gemm_bn == 64) bn = g_tune_gemm_bn;
  // the accumulating epilogue holds three addresses per element: beside the 64 accumulators of a 128-wide tile it does not
  // fit the 128-register cap without spilling, so it runs 128 x 64 tiles at most
  if (a.epi == EPI_CROSS_DX_ACC && bn == 128) bn = 64;
  CUtensorMap tms[6] = {};
  size_t ae, be;
  plane_elems(a, ta, tb, &ae, &be);
  auto planes = [&](const float* src, size_t elems, bool transposed, int64_t rows, int64_t ld, float** hi, float** lo,
                    int64_t* pitch) -> int {
    if (g_cache_on)
      if (const PlaneEntry* e = plane_cached(src, transposed, rows, a.K, ld)) {
        *hi = e->hi; *lo = e->lo; *pitch = e->pitch;
        return DR_OK;
      }
    DR_REQUIRE(g_ws_ptr && (g_bump + 2 * elems) * sizeof(float) <= g_ws_bytes, DR_EINVAL,
               "gemm_tc: workspace exhausted (%zu B registered)", g_ws_bytes);
    *hi = reinterpret_cast<float*>(g_ws_ptr) + g_bump;
    *lo = *hi + elems;
    g_bump += 2 * elems;
    if (int rc = make_planes(src, !transposed, rows, a.K, ld, *hi, *lo, pitch, st)) return rc;
    if (g_cache_on && g_nplanes < 64)
      g_planes[g_nplanes++] = PlaneEntry{src, transposed, rows, a.K, ld, *hi, *lo, *pitch};
    return DR_OK;
  };
  // Weight planes: inside a train step (plane cache on) B is split once and read by every m-tile, instead of being split
  // again by every tile's splitters.  Taken when B is small against A (N <= M / 16: the forward and dX of a Dense layer
  // over a batch, where each plane element is reused by at least M / 128 >= N / 8 tiles and the split pass over B moves
  // at most 3/16 of A's bytes) and A is K-major.  Only for 128-wide tiles (N > 64) with more than one k-block (K > 32):
  // on H100 the 256 -> 32 layer's forward (N = 32) and dX (K = 32), where the splitters do little per tile, measured
  // about 1 us slower with the extra split launch than without.  A K-major B is split flat over rows x ldb floats, so its
  // pitch must be K.  The dW (A transposed) and the accumulating Cross dX keep the splitter kernels.
  if (g_tune_gemm_variant == 2 && g_cache_on && !ta && a.epi != EPI_CROSS_DX_ACC && a.N * 16 <= a.M && a.N > 64 &&
      a.K > TC_BK && (!tb || a.ldb == a.K) &&
      (plane_cached(a.B, !tb, a.N, a.K, a.ldb) || (g_ws_ptr && (g_bump + 2 * be) * sizeof(float) <= g_ws_bytes))) {
    float *Bh, *Bl;
    int64_t pb = 0;
    if (int rc = planes(a.B, be, !tb, a.N, a.ldb, &Bh, &Bl, &pb)) return rc;
    if (int rc = make_map(&tms[0], a.A, a.K, a.M, a.lda, TC_BK, TC_BM, true)) return rc;
    if (int rc = make_map(&tms[2], Bh, a.K, a.N, pb, TC_BK, bn, true)) return rc;
    if (int rc = make_map(&tms[3], Bl, a.K, a.N, pb, TC_BK, bn, true)) return rc;
    tms[1] = tms[0];
    if (bn == 32) return launch_tc<32, false, false, false, true>(tms, a, TC_WP_STAGES, st);
    if (bn == 64) return launch_tc<64, false, false, false, true>(tms, a, TC_WP_STAGES, st);
    return launch_tc<128, false, false, false, true>(tms, a, TC_WP_STAGES, st);
  }
  if (g_tune_gemm_variant == 2) {
    // Variant 2: tensor maps straight on the source operands (staged as stored), split in shared memory.
    const bool A_MN = ta, B_MN = !tb;
    const int raw_stages = (g_tune_tc_stages == 2 || a.stages == 2 || a.share) ? 2 : TC_RAW_STAGES;
    if (!A_MN) {
      if (int rc = make_map(&tms[0], a.A, a.K, a.M, a.lda, TC_BK, TC_BM, true)) return rc;
    } else {
      if (int rc = make_map(&tms[0], a.A, a.M, a.K, a.lda, TC_BM, TC_BK, false)) return rc;
    }
    if (!B_MN) {
      if (int rc = make_map(&tms[2], a.B, a.K, a.N, a.ldb, TC_BK, bn, true)) return rc;
    } else {
      if (int rc = make_map(&tms[2], a.B, a.N, a.K, a.ldb, bn, TC_BK, false)) return rc;
    }
    tms[1] = tms[0];
    tms[3] = tms[2];
#define DR_TC2_LAUNCH(BN_)                                                                  \
    do {                                                                                    \
      if (!A_MN && !B_MN) return launch_tc<BN_, false, false, false>(tms, a, raw_stages, st);  \
      if (!A_MN && B_MN) return launch_tc<BN_, false, true, false>(tms, a, raw_stages, st);    \
      if (A_MN && !B_MN) return launch_tc<BN_, true, false, false>(tms, a, raw_stages, st);    \
      return launch_tc<BN_, true, true, false>(tms, a, raw_stages, st);                        \
    } while (0)
    if (bn == 32) DR_TC2_LAUNCH(32);
    if (bn == 64) DR_TC2_LAUNCH(64);
    DR_TC2_LAUNCH(128);
#undef DR_TC2_LAUNCH
  }
  // Variant 1: K-major hi/lo planes in the workspace.  A(m,k): !ta -> stored [M,K] (flat split), ta -> stored [K,M]
  // (transposing split); B(k,n): tb -> stored [N,K] (flat), !tb -> stored [K,N] (transposing).
  if (!g_cache_on) g_bump = 0;
  float *Ah, *Al, *Bh, *Bl;
  int64_t pa = 0, pb = 0;
  if (int rc = planes(a.A, ae, ta, a.M, a.lda, &Ah, &Al, &pa)) return rc;
  if (int rc = planes(a.B, be, !tb, a.N, a.ldb, &Bh, &Bl, &pb)) return rc;
  if (int rc = make_map(&tms[0], Ah, a.K, a.M, pa, TC_BK, TC_BM, true)) return rc;
  if (int rc = make_map(&tms[1], Al, a.K, a.M, pa, TC_BK, TC_BM, true)) return rc;
  if (int rc = make_map(&tms[2], Bh, a.K, a.N, pb, TC_BK, bn, true)) return rc;
  if (int rc = make_map(&tms[3], Bl, a.K, a.N, pb, TC_BK, bn, true)) return rc;
  if (bn == 32) return launch_tc<32, false, false, true>(tms, a, 0, st);
  if (bn == 64) return launch_tc<64, false, false, true>(tms, a, 0, st);
  return launch_tc<128, false, false, true>(tms, a, 0, st);
}

}  // namespace dr

extern "C" int dr_gemm_plane_cache(int enable) {
  dr::g_nplanes = 0;
  dr::g_bump = 0;
  dr::g_cache_on = enable != 0;
  return DR_OK;
}

extern "C" int dr_set_workspace(void* ptr, uint64_t bytes) {
  dr::g_nplanes = 0;
  dr::g_bump = 0;
  using namespace dr;
  DR_REQUIRE(ptr == nullptr || aligned16(ptr), DR_EALIGN, "dr_set_workspace: pointer not 16-B aligned");
  g_ws_ptr = ptr;
  g_ws_bytes = ptr ? (size_t)bytes : 0;
  return DR_OK;
}
