// SURVEY.md section 8(e): row-sharded embedding tables, owner(r) = r mod G, local row r div G.
// The reference has no multi-device path at all; these kernels are the device half of the
// exchange whose NCCL all-to-all is issued by the host (torch.distributed).  All S tables
// live in one global row space (row = slot_offset[s] + id) so the exchange is slot-agnostic.
#include "common.cuh"

namespace dr {

template <typename IdT>
__device__ __forceinline__ int64_t global_row(const IdT* __restrict__ ids, int64_t i, int S,
                                              const int64_t* __restrict__ slot_offsets,
                                              const int64_t* __restrict__ rows) {
  const int64_t id = (int64_t)__ldg(ids + i);
  if (id < 0) return -1;
  if (!slot_offsets) return id;
  const int s = (int)(i % S);
  if (rows && id >= __ldg(rows + s)) return -1;
  return __ldg(slot_offsets + s) + id;
}

// One pass: every flat lookup i claims a slot in its owner's padded segment of the send buffer
// (segment g = [g*cap, (g+1)*cap)), writes its local row id there and remembers the slot in
// inv[i].  Slots are claimed with one atomic per distinct owner per warp (match.any aggregation).
// A segment that would exceed cap raises the overflow flag (the lookup then reads slot -1 = zero row).
template <typename IdT>
__global__ void __launch_bounds__(256) shard_bucket_kernel(const IdT* __restrict__ ids, int64_t n, int S,
                                                            const int64_t* __restrict__ slot_offsets,
                                                            const int64_t* __restrict__ rows, int G, int64_t cap,
                                                            unsigned long long* __restrict__ cursor,
                                                            int64_t* __restrict__ send_ids, int32_t* __restrict__ inv,
                                                            int32_t* __restrict__ overflow) {
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t nround = (n + stride - 1) / stride;
  for (int64_t it = 0; it < nround; ++it) {
    const int64_t i = it * stride + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t r = -1;
    int owner = 0;
    if (i < n) {
      r = global_row(ids, i, S, slot_offsets, rows);
      if (r < 0) {          // out-of-vocabulary: zero row, nothing to exchange
        inv[i] = -1;
      } else {
        owner = (int)(r % G);
      }
    }
    const bool live = i < n && r >= 0;
    const unsigned peers = __match_any_sync(0xffffffffu, live ? owner : (64 + lane));
    unsigned long long base = 0;
    const int leader = __ffs(peers) - 1;
    if (live && lane == leader) base = atomicAdd(cursor + owner, (unsigned long long)__popc(peers));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (live) {
      const unsigned long long pos = base + (unsigned long long)__popc(peers & ((1u << lane) - 1u));
      if (pos < (unsigned long long)cap) {
        const int64_t slot = (int64_t)owner * cap + (int64_t)pos;
        send_ids[slot] = r / G;
        inv[i] = (int32_t)slot;
      } else {
        inv[i] = -1;
        atomicExch(overflow, 1);
      }
    }
  }
}

// out[i] = in[perm[i]] (PERMUTE) or out[perm[i]] = in[i] (UNPERMUTE); rows of D floats, D % 4 == 0.
template <bool UNPERMUTE>
__global__ void __launch_bounds__(256) permute_rows_kernel(const float* __restrict__ in,
                                                            const int32_t* __restrict__ perm, int64_t n, int D,
                                                            float* __restrict__ out) {
  const int chunks = D / 4;
  const int64_t total = n * chunks;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < total; f += stride) {
    const int64_t i = f / chunks;
    const int c = (int)(f % chunks);
    const int64_t j = __ldg(perm + i);
    if (j < 0) continue;
    if (UNPERMUTE) stg4(out + (size_t)j * D + c * 4, ldg_nc_na(in + (size_t)i * D + c * 4));
    else stg4(out + (size_t)i * D + c * 4, ldg_nc_na(in + (size_t)j * D + c * 4));
  }
}

}  // namespace dr

using namespace dr;

extern "C" int dr_shard_bucket_ids(const void* ids, int id_bytes, int64_t n, int S,
                                   const int64_t* slot_offsets, const int64_t* rows, int G, int64_t cap,
                                   int64_t* send_counts, int64_t* send_ids, int32_t* inv, int32_t* overflow,
                                   void* stream) {
  DR_REQUIRE(ids && send_counts && send_ids && inv && overflow, DR_EINVAL, "dr_shard_bucket_ids: null pointer");
  DR_REQUIRE(n >= 0, DR_EINVAL, "dr_shard_bucket_ids: n=%lld < 0", (long long)n);
  DR_REQUIRE(G >= 1 && G <= 64, DR_EINVAL, "dr_shard_bucket_ids: G=%d outside [1,64]", G);
  DR_REQUIRE(S >= 1, DR_EINVAL, "dr_shard_bucket_ids: S=%d", S);
  DR_REQUIRE(cap >= 1 && (int64_t)G * cap < ((int64_t)1 << 31), DR_EINVAL,
             "dr_shard_bucket_ids: G*cap=%lld must fit int32", (long long)((int64_t)G * cap));
  DR_REQUIRE(id_bytes == 8 || id_bytes == 4, DR_EINVAL, "dr_shard_bucket_ids: id_bytes=%d", id_bytes);
  cudaStream_t st = (cudaStream_t)stream;
  DR_CUDA_CALL(cudaMemsetAsync(send_counts, 0, sizeof(int64_t) * G, st));
  // `overflow` is STICKY: the kernel only ever sets it; the caller clears it after reading it (a per-call memset
  // here would let a later, well-behaved batch erase the evidence of an earlier truncated one).
  DR_CUDA_CALL(cudaMemsetAsync(send_ids, 0xFF, sizeof(int64_t) * (size_t)G * cap, st));   // all -1
  if (n == 0) return DR_OK;
  const int64_t ctas = capped_grid(n, 256, 8);
  return with_id_type(id_bytes, [&](auto id) {
    using IdT = decltype(id);
    shard_bucket_kernel<IdT><<<(unsigned)ctas, 256, 0, st>>>((const IdT*)ids, n, S, slot_offsets, rows, G, cap,
                                                             reinterpret_cast<unsigned long long*>(send_counts), send_ids,
                                                             inv, overflow);
    DR_CUDA_LAUNCH_CHECK("shard_bucket");
    return DR_OK;
  });
}

static int permute_common(const float* in, const int32_t* perm, int64_t n, int D, float* out, void* stream,
                          bool un) {
  DR_REQUIRE(in && perm && out, DR_EINVAL, "dr_permute_rows: null pointer");
  DR_REQUIRE(n >= 0 && D >= 4 && D % 4 == 0, DR_EINVAL, "dr_permute_rows: bad shape n=%lld D=%d", (long long)n, D);
  DR_REQUIRE(aligned16(in) && aligned16(out), DR_EALIGN, "dr_permute_rows: in/out not 16-B aligned");
  if (n == 0) return DR_OK;
  const int64_t ctas = capped_grid(n * (D / 4), 256, 8);
  if (un) permute_rows_kernel<true><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(in, perm, n, D, out);
  else permute_rows_kernel<false><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(in, perm, n, D, out);
  DR_CUDA_LAUNCH_CHECK("permute_rows");
  return DR_OK;
}

extern "C" int dr_permute_rows(const float* in, const int32_t* perm, int64_t n, int D, float* out, void* stream) {
  return permute_common(in, perm, n, D, out, stream, false);
}
extern "C" int dr_unpermute_rows(const float* in, const int32_t* perm, int64_t n, int D, float* out, void* stream) {
  return permute_common(in, perm, n, D, out, stream, true);
}
