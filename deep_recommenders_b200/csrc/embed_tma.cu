// Opt-in variant of the fused gather + first-order + FM forward (rows E + L + F) that STAGES THE ROWS THROUGH THE TMA
// UNIT INTO SHARED MEMORY: one `cp.async.bulk.shared::cluster.global` (UBLKCP) per looked-up row copies its D floats into
// a per-warp tile (Hopper's TMA has no gather-by-index tensor mode, so every row is its own bulk copy), completion on an
// mbarrier, the FM sums are computed from shared memory and the stacked rows leave as one `cp.async.bulk` store per tile.
// Same reference lines as embed_fm.cu (keras/models/ranking/fm.py:23-37, deepfm.py:36-46).
//
// It is NOT the default: the register-load kernel of embed_fm.cu is.  This one exists so that the comparison between
// the two is a product measurement (bench.py --embed-fwd tma), not a claim.
//
// Scope: the fused row layout of embedding.py (one 128-B line [emb D | w | pad] per row, all tables in one arena),
// D = 16, S <= 32.  Everything else uses dr_embed_fm_fwd.
#include "common.cuh"

namespace dr {

__device__ __forceinline__ uint32_t tsm_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void t_mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void t_mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void t_mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}"
      ::"r"(bar), "r"(parity)
      : "memory");
}
// one row of `bytes` (multiple of 16) from global to shared memory through the TMA unit
__device__ __forceinline__ void t_bulk_load(uint32_t sdst, const void* gsrc, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(sdst), "l"(gsrc), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void t_bulk_store(void* gdst, uint32_t ssrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(ssrc), "r"(bytes) : "memory");
}

constexpr int TMA_EX = 8;          // examples per warp tile
constexpr int TMA_WARPS = 4;
constexpr int TMA_NBUF = 2;
constexpr int TMA_D = 16;

struct EmbedTmaParams {
  const float* arena;
  int64_t total_rows;
  const int64_t* slot_offsets;
  const int64_t* rows;
  const void* ids;
  const float* bias;
  int64_t B;
  int S;
  int64_t row_stride;
  float* out_stack;
  float* out_sum;
  float* out_logit;
};

template <typename IdT>
__global__ void __launch_bounds__(TMA_WARPS * 32) embed_fm_fwd_tma_kernel(const EmbedTmaParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) uint64_t bars[TMA_WARPS * TMA_NBUF];
  __shared__ int64_t s_off[32], s_rows[32];
  const int S = p.S, LK = TMA_EX * S;              // lookups per tile (a multiple of 4)
  const int tile_bytes = LK * 64, buf_bytes = (tile_bytes + LK * 4 + 127) / 128 * 128;   // rows + first-order weights, 128-B multiple (TMA destination alignment)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char* mybuf = smem + (size_t)warp * TMA_NBUF * buf_bytes;
  for (int i = threadIdx.x; i < S; i += blockDim.x) { s_off[i] = p.slot_offsets[i]; s_rows[i] = p.rows[i]; }
  if (lane == 0)
    for (int k = 0; k < TMA_NBUF; ++k) t_mbar_init(tsm_u32(&bars[warp * TMA_NBUF + k]), 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  const IdT* __restrict__ ids = reinterpret_cast<const IdT*>(p.ids);
  const int64_t ntiles = (p.B + TMA_EX - 1) / TMA_EX;
  const int64_t w0 = (int64_t)blockIdx.x * TMA_WARPS + warp, nw = (int64_t)gridDim.x * TMA_WARPS;
  const float bias = p.bias ? __ldg(p.bias) : 0.f;

  auto issue = [&](int64_t tile, int buf) {
    unsigned char* tb = mybuf + buf * buf_bytes;
    const uint32_t bar = tsm_u32(&bars[warp * TMA_NBUF + buf]);
    const int64_t b0 = tile * TMA_EX;
    const int n = (int)min((int64_t)LK, (p.B - b0) * S);
    int copies = 0;
    for (int j = lane; j < LK; j += 32) {          // lookup j of the tile -> one bulk copy of its row (OOV id -> zero row)
      float w = 0.f;
      bool hit = false;
      if (j < n) {
        const int s = j % S;
        const int64_t id = (int64_t)__ldg(ids + b0 * S + j);
        if ((uint64_t)id < (uint64_t)s_rows[s]) {
          const float* row = p.arena + (size_t)(s_off[s] + id) * p.row_stride;
          w = ldg_nc_na_f32(row + TMA_D);                                         // in-row first-order weight
          t_bulk_load(tsm_u32(tb + j * 64), row, 64u, bar);
          hit = true;
          ++copies;
        }
      }
      if (!hit) {
#pragma unroll
        for (int c = 0; c < 4; ++c) *reinterpret_cast<float4*>(tb + j * 64 + c * 16) = f4_zero();
      }
      *reinterpret_cast<float*>(tb + tile_bytes + j * 4) = w;
    }
    // the bytes to expect are known only now; complete_tx of copies that already landed is accounted for when the
    // expectation is posted, and the phase cannot complete before this one arrival
    copies = (int)group_sum<32>((float)copies);
    if (lane == 0) t_mbar_expect_tx(bar, (uint32_t)copies * 64u);
  };

  int it = 0;
  if (w0 < ntiles) issue(w0, 0);
  for (int64_t tile = w0; tile < ntiles; tile += nw, ++it) {
    const int buf = it % TMA_NBUF;
    const int64_t nxt = tile + nw;
    // the buffer refilled now was stored from by the previous iteration: its bulk store must have read it
    if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    __syncwarp();
    if (nxt < ntiles) issue(nxt, (it + 1) % TMA_NBUF);
    t_mbar_wait(tsm_u32(&bars[warp * TMA_NBUF + buf]), (uint32_t)((it / TMA_NBUF) & 1));
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // zero rows were ordinary stores; the bulk store reads them
    __syncwarp();                                   // the first-order weights were ordinary shared-memory stores
    unsigned char* tb = mybuf + buf * buf_bytes;
    const int64_t b0 = tile * TMA_EX;
    const int nex = (int)min((int64_t)TMA_EX, p.B - b0);
    if (p.out_stack && lane == 0) {
      t_bulk_store(p.out_stack + b0 * S * TMA_D, tsm_u32(tb), (uint32_t)nex * S * 64);
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    // FM sums from shared memory: for one example the 32 lanes read its S rows x 4 chunks contiguously (conflict free),
    // lanes with equal (lane & 3) combine by xor-shuffles
    for (int e = 0; e < nex; ++e) {
      float4 a = f4_zero(), q = f4_zero();
      const float4* src = reinterpret_cast<const float4*>(tb + e * (S * 64));
      for (int idx = lane; idx < S * 4; idx += 32) {
        const float4 v = src[idx];
        a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
        q.x = fmaf(v.x, v.x, q.x); q.y = fmaf(v.y, v.y, q.y); q.z = fmaf(v.z, v.z, q.z); q.w = fmaf(v.w, v.w, q.w);
      }
      float lin = 0.f;
      for (int s = lane; s < S; s += 32) lin += *reinterpret_cast<const float*>(tb + tile_bytes + (e * S + s) * 4);
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        a.x += __shfl_xor_sync(0xffffffffu, a.x, o); a.y += __shfl_xor_sync(0xffffffffu, a.y, o);
        a.z += __shfl_xor_sync(0xffffffffu, a.z, o); a.w += __shfl_xor_sync(0xffffffffu, a.w, o);
        q.x += __shfl_xor_sync(0xffffffffu, q.x, o); q.y += __shfl_xor_sync(0xffffffffu, q.y, o);
        q.z += __shfl_xor_sync(0xffffffffu, q.z, o); q.w += __shfl_xor_sync(0xffffffffu, q.w, o);
      }
      lin = group_sum<32>(lin);
      float t = (a.x * a.x - q.x) + (a.y * a.y - q.y) + (a.z * a.z - q.z) + (a.w * a.w - q.w);
      t += __shfl_xor_sync(0xffffffffu, t, 1);
      t += __shfl_xor_sync(0xffffffffu, t, 2);
      if (p.out_sum && lane < 4) stg4(p.out_sum + (b0 + e) * TMA_D + lane * 4, a);
      if (p.out_logit && lane == 0) p.out_logit[b0 + e] = (bias + lin) + 0.5f * t;
    }
    __syncwarp();
  }
  if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

}  // namespace dr

using namespace dr;

extern "C" int dr_embed_fm_fwd_tma(const float* arena, int64_t total_rows, const int64_t* slot_offsets,
                                   const int64_t* rows, const void* ids, int id_bytes, const float* bias, int64_t B, int S,
                                   int D, int64_t row_stride, float* out_stack, float* out_sum, float* out_logit,
                                   void* stream) {
  DR_REQUIRE(arena && slot_offsets && rows && ids, DR_EINVAL, "dr_embed_fm_fwd_tma: null pointer");
  DR_REQUIRE(B >= 0 && S >= 1, DR_EINVAL, "dr_embed_fm_fwd_tma: B=%lld S=%d", (long long)B, S);
  DR_REQUIRE(id_bytes == 8 || id_bytes == 4, DR_EINVAL, "dr_embed_fm_fwd_tma: id_bytes=%d (need 4 or 8)", id_bytes);
  DR_REQUIRE(D == TMA_D && S <= 32 && row_stride >= D + 4 && row_stride % 4 == 0 && total_rows >= 1 &&
                 total_rows < ((int64_t)1 << 31) - 1,
             DR_ENOTSUP, "dr_embed_fm_fwd_tma: this variant serves fused rows with D=16, S<=32 (got D=%d S=%d stride=%lld)", D, S,
             (long long)row_stride);
  DR_REQUIRE(aligned16(arena) && (!out_stack || aligned16(out_stack)) && (!out_sum || aligned16(out_sum)), DR_EALIGN,
             "dr_embed_fm_fwd_tma: arena / out_stack / out_sum not 16-B aligned");
  if (B == 0) return DR_OK;
  EmbedTmaParams p{};
  p.arena = arena; p.total_rows = total_rows; p.slot_offsets = slot_offsets; p.rows = rows; p.ids = ids; p.bias = bias;
  p.B = B; p.S = S; p.row_stride = row_stride; p.out_stack = out_stack; p.out_sum = out_sum; p.out_logit = out_logit;
  const size_t smem = (size_t)TMA_WARPS * TMA_NBUF * (((size_t)TMA_EX * S * 64 + (size_t)TMA_EX * S * 4 + 127) / 128 * 128);
  const int64_t ntiles = (B + TMA_EX - 1) / TMA_EX;
  return with_id_type(id_bytes, [&](auto id) {
    auto k = embed_fm_fwd_tma_kernel<decltype(id)>;
    DR_CUDA_CALL(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 1;
    DR_CUDA_CALL(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, TMA_WARPS * 32, smem));
    const int64_t ctas = capped_grid(ntiles, TMA_WARPS, occ > 0 ? occ : 1);
    k<<<(unsigned)ctas, TMA_WARPS * 32, smem, (cudaStream_t)stream>>>(p);
    DR_CUDA_LAUNCH_CHECK("dr_embed_fm_fwd_tma");
    return DR_OK;
  });
}
