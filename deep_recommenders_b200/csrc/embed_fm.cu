// Rows E + L + F of SURVEY.md section 8(a): the fused multi-slot embedding gather, first-order
// term and FM second-order interaction (forward), and the backward whose embedding
// gradient is a warp-aggregated vector-atomic scatter-add.  HBM-bandwidth bound.
//
// Reference semantics restated (never executed here):
//   keras/models/ranking/fm.py:23-37   FM.call          linear + 0.5*sum((sum e)^2 - sum e^2)
//   keras/models/ranking/deepfm.py:36-46  per-column DenseFeatures -> stack/concat
//   estimator/models/feature_interaction/fm.py:10-26,41-56
//
// Thread mapping (both kernels).  A row of D fp32 is D/4 128-bit chunks; LPR = the power of
// two >= D/4 lanes own one chunk each, so the LPR lanes of a "lane group" read one whole
// row with one LDG.128 each (D=16: 4 lanes x 16 B = one 64 B row = two 32 B sectors).  A
// warp holds G = 32/LPR lane groups; a lane group walks the S slots of ONE example, keeping
// sum_s e and sum_s e^2 for its chunk in registers, so the FM reduction needs no memory
// traffic at all and only log2(LPR) shuffles at the very end.  The ids of the warp's G
// examples are one contiguous G*S block of the [B,S] id matrix: they are fetched with
// coalesced loads into a per-warp shared-memory slice (no block barrier in the main loop).
// Each lane then has up to U independent 16 B row loads in flight.
#include "common.cuh"

namespace dr {

int g_tune_embed_fwd_unroll = 0;      // 0 = default per LPR
int g_tune_embed_bwd_unroll = 0;
int g_tune_embed_block = 256;         // threads per CTA
int g_tune_embed_ctas_per_sm = 0;     // 0 = as many as fit (2048 threads / SM)
int g_tune_embed_bwd_agg = 1;         // example-parallel mode: warp-aggregate duplicate ids before the atomics
int g_tune_embed_bwd_mode = 0;        // 0 = slot-parallel (default), 1 = example-parallel (+ optional aggregation)
int g_tune_embed_fwd_linx = 1;        // 1 (default) = LINX forward mapping for in-row first-order weights (no idle lanes,
                                      // twice the rows in flight per warp); 0 = a lane of its own for the weight; bit-identical
int g_tune_embed_bwd_linx = 0;        // LINX mapping for the slot-parallel backward (in-row weight, D <= 32): unmeasured
int g_tune_embed_fwd_linx_shard = 0;  // same mapping for the row-sharded (peer-memory) forward: off until measured at N > 1
int g_tune_embed_l2_hints = 0;        // bit 0: forward row loads L2::evict_first; bit 1: stacked-output stores L2::evict_last;
                                      // bit 2: backward vector atomics L2::evict_first; bit 3: backward stack / g_stack loads evict_first
int g_tune_embed_bwd_carveout = 0;     // backward: preferred shared-memory carveout in percent (0 = leave the driver default)
int g_tune_embed_fwd_minblocks = 0;   // forward register cap: 0 = none (ptxas picks, 108 regs -> 2 CTAs of 256 / SM),
                                      // 3 / 4 = __launch_bounds__(256, n): <= 85 / 64 registers, 24 / 32 warps per SM

struct EmbedFwdParams {
  const float* const* table_ptrs;
  const float* const* lin_ptrs;
  const int64_t* rows;
  const float* single_table;   // S == 1 fast form (dr_gather_fwd); table_ptrs == nullptr
  int64_t single_rows;
  const void* ids;
  const float* bias;
  int64_t B;
  int S, D;
  int64_t row_stride;   // floats between consecutive rows of a table (>= D)
  int64_t lin_stride;   // floats between consecutive first-order weights (>= 1)
  int lin_in_row;       // first-order weight lives in the row at float index D (fetched with the row)
  // row-sharded mode (shard_world > 0): global row = slot_offsets[s] + id lives on rank row % G at
  // local row row / G of that rank's arena; peer_bases[g] is rank g's arena mapped into this
  // process (NVLink peer memory), so the gather itself is the exchange.
  int shard_world;
  const float* const* peer_bases;
  const int64_t* slot_offsets;
  int64_t shard_lin_off;   // > 0: first-order weights live at peer_bases[g] + shard_lin_off + local_row (wide rows)
  float* out_stack;
  float* out_sum;
  float* out_logit;
  int l2_hints;
};

struct EmbedBwdParams {
  const void* ids;
  const int64_t* rows;
  int64_t single_rows;
  const float* stack;
  const float* sum_e;
  const float* g_logit;
  const float* g_stack;
  int64_t B;
  int S, D;
  float* const* grad_table_ptrs;
  float* const* grad_lin_ptrs;
  float* single_grad;
  float* g_bias;
  float scale;
  int64_t row_stride;
  int64_t lin_stride;
  int lin_in_row;
  int shard_world;
  float* const* peer_bases;
  const int64_t* slot_offsets;
  int64_t shard_lin_off;
  int l2_hints;
  int mode;     // 0 = slot-parallel kernel, 1 = example-parallel; a per-call copy of the developer knob (the entry
                // points never write a knob: sharded addressing simply passes mode = 0)
};

// shared memory carve-up: [S] table ptr | [S] lin ptr | [S] rows | per-warp id slices
__host__ __device__ inline size_t embed_smem_bytes(int S, int warps, int G, int id_bytes) {
  size_t hdr = (size_t)S * (sizeof(void*) * 2 + sizeof(int64_t) * 2) + kMaxShardWorld * sizeof(void*);
  size_t ids = (size_t)warps * G * S * id_bytes;
  return hdr + ((ids + 15) & ~(size_t)15);
}

// LINX (experiment, knob embed_fwd_linx): with the in-row first-order weight, size the lane group for the D/4
// embedding chunks only (D = 16: 4 lanes, 8 examples per warp, no idle lanes) and let lane 0 of the group fetch
// the weight with a second, scalar load issued right behind its 16-B chunk load (same 128-B line, in flight).
// NOFM (DR_EMBED_NO_FM): the logit is bias + first order only (xDeepFM's linear unit); the FM sums are dead code then.
template <int LPR, typename IdT, int U, bool SHARD, int MINB = 0, bool LINX = false, bool NOFM = false>
__global__ void __launch_bounds__(MINB ? 256 : 512, MINB ? MINB : 1) embed_fm_fwd_kernel(const EmbedFwdParams p) {
  constexpr int G = 32 / LPR;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int S = p.S, D = p.D;
  const float** s_tab = reinterpret_cast<const float**>(smem_raw);
  const float** s_lin = s_tab + S;
  int64_t* s_rows = reinterpret_cast<int64_t*>(s_lin + S);
  int64_t* s_off = s_rows + S;
  const float** s_peer = reinterpret_cast<const float**>(s_off + S);
  const int warp_in_cta = threadIdx.x >> 5;
  const int warps_per_cta = blockDim.x >> 5;
  IdT* s_ids = reinterpret_cast<IdT*>(s_peer + kMaxShardWorld) + (size_t)warp_in_cta * G * S;
  const int SW = SHARD ? p.shard_world : 0;
  const bool sw_pow2 = (SW & (SW - 1)) == 0;
  const int sw_shift = 31 - __clz(SW > 0 ? SW : 1);

  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    s_tab[i] = p.table_ptrs ? p.table_ptrs[i] : p.single_table;
    s_lin[i] = p.lin_ptrs ? p.lin_ptrs[i] : nullptr;
    s_rows[i] = p.rows ? p.rows[i] : p.single_rows;
    if (SHARD) s_off[i] = p.slot_offsets ? p.slot_offsets[i] : 0;
  }
  if (SHARD)
    for (int i = threadIdx.x; i < SW; i += blockDim.x) s_peer[i] = p.peer_bases[i];
  __syncthreads();

  const int lane = threadIdx.x & 31;
  const int c = lane % LPR;          // 16-byte chunk of the row this lane owns
  const int g = lane / LPR;          // example (lane group) inside the warp tile
  const bool chunk_ok = (c * 4) < D;
  // lin_in_row: the lane owning chunk D/4 fetches [w | pad] with the SAME LDG.128 as the embedding
  // chunks, so the first-order weight costs no extra request / DRAM line.
  const bool lin_lane = !LINX && p.lin_in_row && (c * 4 == D);
  const bool has_lin = p.lin_ptrs != nullptr && !p.lin_in_row;
  const bool linx_lane = LINX && p.lin_in_row && c == 0 && p.out_logit != nullptr;
  const float bias = p.bias ? __ldg(p.bias) : 0.f;
  const IdT* __restrict__ ids = reinterpret_cast<const IdT*>(p.ids);
  const bool h_ld = (p.l2_hints & 1) != 0, h_st = (p.l2_hints & 2) != 0;
  const uint64_t pol_first = l2_policy_evict_first(), pol_last = l2_policy_evict_last();

  const int64_t ntiles = (p.B + G - 1) / G;
  const int64_t warp0 = (int64_t)blockIdx.x * warps_per_cta + warp_in_cta;
  const int64_t nwarps = (int64_t)gridDim.x * warps_per_cta;

  for (int64_t tile = warp0; tile < ntiles; tile += nwarps) {
    const int64_t b0 = tile * G;
    const int nex = (int)min((int64_t)G, p.B - b0);
    {  // coalesced id staging: G*S consecutive ids of the [B,S] matrix
      const IdT* src = ids + b0 * S;
      const int n = nex * S;
      for (int i = lane; i < n; i += 32) s_ids[i] = __ldg(src + i);
    }
    __syncwarp();

    const int64_t b = b0 + g;
    const bool ex_ok = g < nex;
    const IdT* my = s_ids + g * S;
    float4 sum = f4_zero(), sq = f4_zero();
    float lin = 0.f;
    float* ostack = p.out_stack ? p.out_stack + ((size_t)b * S) * D + c * 4 : nullptr;

    for (int s0 = 0; s0 < S; s0 += U) {
      float4 v[U];
      float wv[LINX ? U : 1];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int s = s0 + u;
        v[u] = f4_zero();
        if (LINX) wv[u] = 0.f;
        if (s < S && ex_ok && (chunk_ok || lin_lane)) {
          const int64_t id = (int64_t)my[s];
          if ((uint64_t)id < (uint64_t)s_rows[s]) {
            const float* rowp;
            if (!SHARD) {
              rowp = s_tab[s] + (size_t)id * p.row_stride;
            } else {   // row-sharded: the owner's arena is read directly over NVLink
              const int64_t r = s_off[s] + id;
              const int owner = sw_pow2 ? (int)(r & (SW - 1)) : (int)(r % SW);
              const int64_t local = sw_pow2 ? (r >> sw_shift) : (r / SW);
              rowp = s_peer[owner] + (size_t)local * p.row_stride;
            }
            if (h_ld) {
              v[u] = ldg_nc_na_hint(rowp + c * 4, pol_first);
              if (LINX && linx_lane) wv[u] = ldg_nc_na_f32_hint(rowp + D, pol_first);
            } else {
              v[u] = ldg_nc_na(rowp + c * 4);
              if (LINX && linx_lane) wv[u] = ldg_nc_na_f32(rowp + D);
            }
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int s = s0 + u;
        if (s < S) {
          if (LINX) lin += wv[u];
          if (lin_lane) {
            lin += v[u].x;
          } else {
            sum.x += v[u].x; sum.y += v[u].y; sum.z += v[u].z; sum.w += v[u].w;
            sq.x = fmaf(v[u].x, v[u].x, sq.x); sq.y = fmaf(v[u].y, v[u].y, sq.y);
            sq.z = fmaf(v[u].z, v[u].z, sq.z); sq.w = fmaf(v[u].w, v[u].w, sq.w);
            if (ostack && ex_ok && chunk_ok) {
              if (h_st) stg4_hint(ostack + (size_t)s * D, v[u], pol_last);
              else stg4(ostack + (size_t)s * D, v[u]);
            }
          }
        }
      }
    }

    if (p.out_sum && ex_ok && chunk_ok) stg4(p.out_sum + (size_t)b * D + c * 4, sum);

    if (p.out_logit) {
      if (has_lin && ex_ok) {
        for (int s = c; s < S; s += LPR) {   // the LPR lanes split the S scalar gathers
          const int64_t id = (int64_t)my[s];
          if ((uint64_t)id < (uint64_t)s_rows[s]) lin += __ldg(s_lin[s] + (size_t)id * p.lin_stride);
        }
      }
      if (SHARD && p.shard_lin_off > 0 && ex_ok) {   // wide sharded rows: first-order weights trail the owner's shard
        for (int s = c; s < S; s += LPR) {
          const int64_t id = (int64_t)my[s];
          if ((uint64_t)id < (uint64_t)s_rows[s]) {
            const int64_t r = s_off[s] + id;
            const int owner = sw_pow2 ? (int)(r & (SW - 1)) : (int)(r % SW);
            const int64_t local = sw_pow2 ? (r >> sw_shift) : (r / SW);
            lin += __ldg(s_peer[owner] + p.shard_lin_off + local);
          }
        }
      }
      float t = (sum.x * sum.x - sq.x) + (sum.y * sum.y - sq.y) + (sum.z * sum.z - sq.z) +
                (sum.w * sum.w - sq.w);
      t = group_sum<LPR>(t);
      lin = group_sum<LPR>(lin);
      if (c == 0 && ex_ok) p.out_logit[b] = NOFM ? (bias + lin) : (bias + lin) + 0.5f * t;
    }
    __syncwarp();   // the id slice is overwritten by the next tile
  }
}

template <int LPR, typename IdT, int U, bool AGG>
__global__ void __launch_bounds__(512) embed_fm_bwd_kernel(const EmbedBwdParams p) {
  constexpr int G = 32 / LPR;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ float s_bias_part[16];
  const int S = p.S, D = p.D;
  float** s_tab = reinterpret_cast<float**>(smem_raw);
  float** s_lin = s_tab + S;
  int64_t* s_rows = reinterpret_cast<int64_t*>(s_lin + S);
  const int warp_in_cta = threadIdx.x >> 5;
  const int warps_per_cta = blockDim.x >> 5;
  IdT* s_ids = reinterpret_cast<IdT*>(s_rows + S) + (size_t)warp_in_cta * G * S;

  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    s_tab[i] = p.grad_table_ptrs ? p.grad_table_ptrs[i] : p.single_grad;
    s_lin[i] = p.grad_lin_ptrs ? p.grad_lin_ptrs[i] : nullptr;
    s_rows[i] = p.rows ? p.rows[i] : p.single_rows;
  }
  __syncthreads();

  const int lane = threadIdx.x & 31;
  const int c = lane % LPR;
  const int g = lane / LPR;
  const bool chunk_ok = (c * 4) < D;
  const bool has_fm = p.g_logit != nullptr;
  const bool has_gs = p.g_stack != nullptr;
  const bool lin_lane = p.lin_in_row && has_fm && (c * 4 == D);
  const bool has_lin = p.grad_lin_ptrs != nullptr && has_fm && !p.lin_in_row;
  const float scale = p.scale;
  const IdT* __restrict__ ids = reinterpret_cast<const IdT*>(p.ids);

  const int64_t ntiles = (p.B + G - 1) / G;
  const int64_t warp0 = (int64_t)blockIdx.x * warps_per_cta + warp_in_cta;
  const int64_t nwarps = (int64_t)gridDim.x * warps_per_cta;
  float bias_acc = 0.f;

  for (int64_t tile = warp0; tile < ntiles; tile += nwarps) {
    const int64_t b0 = tile * G;
    const int nex = (int)min((int64_t)G, p.B - b0);
    {
      const IdT* src = ids + b0 * S;
      const int n = nex * S;
      for (int i = lane; i < n; i += 32) s_ids[i] = __ldg(src + i);
    }
    __syncwarp();

    const int64_t b = b0 + g;
    const bool ex_ok = g < nex;
    const IdT* my = s_ids + g * S;
    const size_t row0 = ((size_t)b * S) * D + c * 4;
    const float gl = (has_fm && ex_ok) ? __ldg(p.g_logit + b) : 0.f;
    if (c == 0) bias_acc += gl;

    float4 sum = f4_zero();
    if (has_fm && ex_ok && chunk_ok) {
      if (p.sum_e) {
        sum = ldg4(p.sum_e + (size_t)b * D + c * 4);
      } else {
        for (int s = 0; s < S; ++s) sum = f4_add(sum, ldg4(p.stack + row0 + (size_t)s * D));
      }
    }

    for (int s0 = 0; s0 < S; s0 += U) {
      float4 e[U], gs[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int s = s0 + u;
        e[u] = f4_zero();
        gs[u] = f4_zero();
        if (s < S && ex_ok && chunk_ok) {
          if (has_fm) e[u] = ldg_nc_na(p.stack + row0 + (size_t)s * D);
          if (has_gs) gs[u] = ldg_nc_na(p.g_stack + row0 + (size_t)s * D);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int s = s0 + u;
        if (s >= S) break;     // warp-uniform
        int64_t id = -1;
        if (ex_ok) id = (int64_t)my[s];
        const bool ok = ex_ok && (chunk_ok || lin_lane) && (uint64_t)id < (uint64_t)s_rows[s];
        float4 d;
        d.x = scale * fmaf(gl, sum.x - e[u].x, gs[u].x);
        d.y = scale * fmaf(gl, sum.y - e[u].y, gs[u].y);
        d.z = scale * fmaf(gl, sum.z - e[u].z, gs[u].z);
        d.w = scale * fmaf(gl, sum.w - e[u].w, gs[u].w);
        if (lin_lane) d = make_float4(scale * gl, 0.f, 0.f, 0.f);   // [dw | pad] rides in the same request
        bool leader = true;
        if (AGG && G > 1) {
          // lanes that target the same 16 B of the same table row are merged: the lowest
          // lane adds its peers' contributions and issues the single vector atomic.
          const unsigned long long key =
              ok ? (((unsigned long long)id << 5) | (unsigned)c) : (0x8000000000000000ull | (unsigned)lane);
          const unsigned peers = __match_any_sync(0xffffffffu, key);
          if (!__all_sync(0xffffffffu, peers == (1u << lane))) {
            const float4 d0 = d;   // shuffle the ORIGINAL contributions (d is being accumulated)
#pragma unroll
            for (int k = 1; k < G; ++k) {
              const float4 o = f4_shfl_down(d0, k * LPR);
              const int src = lane + k * LPR;
              if (src < 32 && ((peers >> src) & 1u)) d = f4_add(d, o);
            }
            leader = (__ffs(peers) - 1) == lane;
          }
        }
        if (ok && leader) red_add_v4(s_tab[s] + (size_t)id * p.row_stride + c * 4, d);
      }
    }

    if (has_lin && ex_ok) {
      const float gv = scale * gl;
      for (int s = c; s < S; s += LPR) {
        const int64_t id = (int64_t)my[s];
        if ((uint64_t)id < (uint64_t)s_rows[s]) red_add_f32(s_lin[s] + (size_t)id * p.lin_stride, gv);
      }
    }
    __syncwarp();
  }

  if (p.g_bias && has_fm) {   // one atomic per CTA for the scalar bias gradient
    bias_acc = group_sum<32>(bias_acc);
    if (lane == 0) s_bias_part[warp_in_cta] = bias_acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int w = 0; w < warps_per_cta; ++w) t += s_bias_part[w];
      red_add_f32(p.g_bias, scale * t);
    }
  }
}

// Backward, slot-parallel mapping (default).  A warp walks ONE example at a time: its 32/LPR lane
// groups take 32/LPR consecutive SLOTS of that example, so
//   * the saved stack and the upstream g_stack are read as one contiguous run per instruction
//     ((32/LPR) rows x D floats), the ids of the example as one contiguous run,
//   * the lookups a warp issues together belong to DIFFERENT tables and can never collide, so no
//     intra-warp duplicate detection is needed before the vector atomics (duplicates across warps
//     are resolved by the L2 atomic unit),
//   * no shared-memory staging and no cross-lane reduction: sum_e arrives precomputed.
// U slot-steps are loaded before any atomic is issued (the red.global asm is a compiler barrier).
// LINX (knob embed_bwd_linx, off by default: unmeasured): lane group sized for the D/4 embedding chunks only, the
// first-order gradient of an in-row weight issued by lane 0 as a scalar red.global.add behind its vector atomic.
// NOFM (DR_EMBED_NO_FM): dE = g_stack only; g_logit still reaches the first-order weights and the bias.
template <int LPR, typename IdT, int U, bool SHARD, bool LINX = false, bool NOFM = false>
__global__ void __launch_bounds__(256) embed_fm_bwd_sp_kernel(const EmbedBwdParams p) {
  constexpr int SPW = 32 / LPR;      // slots per warp-instruction
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ float s_bias_part[8];
  const int S = p.S, D = p.D;
  float** s_tab = reinterpret_cast<float**>(smem_raw);
  float** s_lin = s_tab + S;
  int64_t* s_rows = reinterpret_cast<int64_t*>(s_lin + S);
  int64_t* s_off = s_rows + S;
  float** s_peer = reinterpret_cast<float**>(s_off + S);
  const int SW = SHARD ? p.shard_world : 0;
  const bool sw_pow2 = (SW & (SW - 1)) == 0;
  const int sw_shift = 31 - __clz(SW > 0 ? SW : 1);
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    s_tab[i] = p.grad_table_ptrs ? p.grad_table_ptrs[i] : p.single_grad;
    s_lin[i] = p.grad_lin_ptrs ? p.grad_lin_ptrs[i] : nullptr;
    s_rows[i] = p.rows ? p.rows[i] : p.single_rows;
    if (SHARD) s_off[i] = p.slot_offsets ? p.slot_offsets[i] : 0;
  }
  if (SHARD)
    for (int i = threadIdx.x; i < SW; i += blockDim.x) s_peer[i] = p.peer_bases[i];
  __syncthreads();

  const int lane = threadIdx.x & 31, warp_in_cta = threadIdx.x >> 5, warps_per_cta = blockDim.x >> 5;
  const int c = lane % LPR, sg = lane / LPR;
  const bool chunk_ok = (c * 4) < D;
  const bool has_fm = p.g_logit != nullptr, has_gs = p.g_stack != nullptr;
  const bool lin_lane = !LINX && p.lin_in_row && has_fm && (c * 4 == D);
  const bool linx_lane = LINX && p.lin_in_row && has_fm && c == 0;
  const bool has_lin = p.grad_lin_ptrs != nullptr && has_fm && !p.lin_in_row;
  const float scale = p.scale;
  const IdT* __restrict__ ids = reinterpret_cast<const IdT*>(p.ids);
  const int64_t warp0 = (int64_t)blockIdx.x * warps_per_cta + warp_in_cta;
  const int64_t nwarps = (int64_t)gridDim.x * warps_per_cta;
  float bias_acc = 0.f;
  const bool h_red = (p.l2_hints & 4) != 0, h_ld = (p.l2_hints & 8) != 0;
  const uint64_t pol_first = l2_policy_evict_first();

  for (int64_t b = warp0; b < p.B; b += nwarps) {
    const float gl = has_fm ? __ldg(p.g_logit + b) : 0.f;
    if (lane == 0) bias_acc += gl;
    const float gfm = NOFM ? 0.f : gl;   // weight of the FM term in dE
    float4 sum = f4_zero();
    if (!NOFM && has_fm && chunk_ok) {
      if (p.sum_e) {
        sum = ldg4(p.sum_e + (size_t)b * D + c * 4);
      } else {
        for (int s = 0; s < S; ++s) sum = f4_add(sum, ldg4(p.stack + ((size_t)b * S + s) * D + c * 4));
      }
    }
    const IdT* my_ids = ids + (size_t)b * S;
    const size_t ex0 = (size_t)b * S * D + c * 4;
    for (int s0 = 0; s0 < S; s0 += SPW * U) {
      float4 e[U], gs[U];
      int64_t id[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int s = s0 + u * SPW + sg;
        e[u] = f4_zero();
        gs[u] = f4_zero();
        id[u] = -1;
        if (s < S) {
          id[u] = (int64_t)__ldg(my_ids + s);
          if (chunk_ok) {
            if (h_ld) {
              if (!NOFM && has_fm) e[u] = ldg_nc_na_hint(p.stack + ex0 + (size_t)s * D, pol_first);
              if (has_gs) gs[u] = ldg_nc_na_hint(p.g_stack + ex0 + (size_t)s * D, pol_first);
            } else {
              if (!NOFM && has_fm) e[u] = ldg_nc_na(p.stack + ex0 + (size_t)s * D);
              if (has_gs) gs[u] = ldg_nc_na(p.g_stack + ex0 + (size_t)s * D);
            }
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int s = s0 + u * SPW + sg;
        if (s < S && (uint64_t)id[u] < (uint64_t)s_rows[s]) {
          float* row;
          if (!SHARD) {
            row = s_tab[s] + (size_t)id[u] * p.row_stride;
          } else {     // row-sharded: vector atomics straight into the owner's arena over NVLink
            const int64_t r = s_off[s] + id[u];
            const int owner = sw_pow2 ? (int)(r & (SW - 1)) : (int)(r % SW);
            const int64_t local = sw_pow2 ? (r >> sw_shift) : (r / SW);
            row = s_peer[owner] + (size_t)local * p.row_stride;
          }
          if (chunk_ok) {
            float4 d;
            d.x = scale * fmaf(gfm, sum.x - e[u].x, gs[u].x);
            d.y = scale * fmaf(gfm, sum.y - e[u].y, gs[u].y);
            d.z = scale * fmaf(gfm, sum.z - e[u].z, gs[u].z);
            d.w = scale * fmaf(gfm, sum.w - e[u].w, gs[u].w);
            if (h_red) {
              red_add_v4_hint(row + c * 4, d, pol_first);
              if (LINX && linx_lane) red_add_f32_hint(row + D, scale * gl, pol_first);
            } else {
              red_add_v4(row + c * 4, d);
              if (LINX && linx_lane) red_add_f32(row + D, scale * gl);
            }
          } else if (lin_lane) {
            if (h_red) red_add_v4_hint(row + c * 4, make_float4(scale * gl, 0.f, 0.f, 0.f), pol_first);
            else red_add_v4(row + c * 4, make_float4(scale * gl, 0.f, 0.f, 0.f));
          }
          if (has_lin && c == 0) red_add_f32(s_lin[s] + (size_t)id[u] * p.lin_stride, scale * gl);
          if (SHARD && has_fm && p.shard_lin_off > 0 && c == 0) {
            const int64_t r = s_off[s] + id[u];
            const int owner = sw_pow2 ? (int)(r & (SW - 1)) : (int)(r % SW);
            const int64_t local = sw_pow2 ? (r >> sw_shift) : (r / SW);
            red_add_f32(s_peer[owner] + p.shard_lin_off + local, scale * gl);
          }
        }
      }
    }
  }

  if (p.g_bias && has_fm) {
    bias_acc = group_sum<32>(bias_acc);
    if (lane == 0) s_bias_part[warp_in_cta] = bias_acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int w = 0; w < warps_per_cta; ++w) t += s_bias_part[w];
      red_add_f32(p.g_bias, scale * t);
    }
  }
}

// Plain single-table row gather / scatter-add (two-tower towers, owner side of the sharded
// exchange): one 16-byte chunk per thread, flat over (row, chunk), grid-stride.  OOV id -> zeros.
template <typename IdT>
__global__ void __launch_bounds__(256) gather_rows_kernel(const float* __restrict__ table, int64_t rows,
                                                           const IdT* __restrict__ ids, int64_t n, int chunks,
                                                           float* __restrict__ out) {
  const int64_t total = n * chunks;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < total; f += stride) {
    const int64_t i = f / chunks;
    const int c = (int)(f - i * chunks);
    const int64_t id = (int64_t)__ldg(ids + i);
    float4 v = f4_zero();
    if ((uint64_t)id < (uint64_t)rows) v = ldg_nc_na(table + ((size_t)id * chunks + c) * 4);
    stg4(out + (size_t)f * 4, v);
  }
}

template <typename IdT>
__global__ void __launch_bounds__(256) scatter_add_rows_kernel(float* __restrict__ table, int64_t rows,
                                                                const IdT* __restrict__ ids, int64_t n, int chunks,
                                                                const float* __restrict__ g, float scale) {
  const int64_t total = n * chunks;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < total; f += stride) {
    const int64_t i = f / chunks;
    const int c = (int)(f - i * chunks);
    const int64_t id = (int64_t)__ldg(ids + i);
    if ((uint64_t)id < (uint64_t)rows) {
      float4 v = ldg_nc_na(g + (size_t)f * 4);
      v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
      red_add_v4(table + ((size_t)id * chunks + c) * 4, v);
    }
  }
}

// ---- host-side dispatch -----------------------------------------------------------------
struct LaunchGeom {
  int threads, ctas;
  size_t smem;
};

// B >= 1: the entries return before a launch at B = 0
static LaunchGeom geom(int64_t B, int S, int LPR, int id_bytes) {
  LaunchGeom lg;
  lg.threads = g_tune_embed_block;
  if (lg.threads != 128 && lg.threads != 256 && lg.threads != 512) lg.threads = 256;
  const int warps = lg.threads / 32, G = 32 / LPR;
  lg.smem = embed_smem_bytes(S, warps, G, id_bytes);
  int per_sm = 2048 / lg.threads;
  if (g_tune_embed_ctas_per_sm > 0 && g_tune_embed_ctas_per_sm < per_sm) per_sm = g_tune_embed_ctas_per_sm;
  lg.ctas = (int)capped_grid((B + G - 1) / G, warps, per_sm);
  return lg;
}

template <typename Params>
static int launch(void (*k)(Params), const LaunchGeom& lg, const Params& p, cudaStream_t st, const char* what) {
  if (int rc = allow_dynamic_smem(k, lg.smem)) return rc;
  k<<<lg.ctas, lg.threads, lg.smem, st>>>(p);
  DR_CUDA_LAUNCH_CHECK(what);
  return DR_OK;
}

template <int LPR, typename IdT, int U, bool LINXSEL = false>
static int launch_fwd_u(const EmbedFwdParams& p, cudaStream_t st) {
  // experiment instantiations (same arithmetic, same results): narrow rows, U = 8 / 13 only
  //   MINB 3 / 4: register cap via __launch_bounds__(256, n);  LINX: see the kernel comment
  constexpr bool kExp = (LPR <= 8) && (U == 8 || U == 13);
  constexpr int UU = kExp ? U : 8;
  static_assert(!LINXSEL || kExp, "LINX is instantiated for LPR <= 8 and U in {8, 13} only");
  LaunchGeom lg = geom(p.B, p.S, LPR, sizeof(IdT));
  if (p.shard_world > 0) {
    if (LINXSEL && U == 8) return launch(embed_fm_fwd_kernel<LPR, IdT, 8, true, 0, LINXSEL>, lg, p, st, "embed_fm_fwd");
    return launch(embed_fm_fwd_kernel<LPR, IdT, U, true>, lg, p, st, "embed_fm_fwd");
  }
  const int minb = (kExp && lg.threads <= 256 && lg.smem <= 48 * 1024) ? g_tune_embed_fwd_minblocks : 0;
  if (kExp && (minb >= 3 || LINXSEL)) {
    int per_sm = minb >= 4 ? 4 : (minb == 3 ? 3 : 2);
    per_sm *= (lg.threads <= 256 ? 256 / lg.threads : 1);
    if (g_tune_embed_ctas_per_sm > 0 && g_tune_embed_ctas_per_sm < per_sm) per_sm = g_tune_embed_ctas_per_sm;
    const int G = 32 / LPR;
    lg.ctas = (int)capped_grid((p.B + G - 1) / G, lg.threads / 32, per_sm);   // one resident wave
    void (*k)(EmbedFwdParams) = minb >= 4    ? embed_fm_fwd_kernel<LPR, IdT, UU, false, 4, LINXSEL>
                                : minb == 3 ? embed_fm_fwd_kernel<LPR, IdT, UU, false, 3, LINXSEL>
                                            : embed_fm_fwd_kernel<LPR, IdT, UU, false, 0, LINXSEL>;
    return launch(k, lg, p, st, "embed_fm_fwd(linx/capped)");
  }
  return launch(embed_fm_fwd_kernel<LPR, IdT, U, false>, lg, p, st, "embed_fm_fwd");
}

template <int LPR, typename IdT>
static int launch_fwd_linx(const EmbedFwdParams& p, cudaStream_t st) {
  if (g_tune_embed_fwd_unroll == 13 && p.shard_world == 0) return launch_fwd_u<LPR, IdT, 13, true>(p, st);
  return launch_fwd_u<LPR, IdT, 8, true>(p, st);
}

// lane group sized for the embedding chunks only (LINX): D <= 32 with the weight in the row
static int dispatch_fwd_linx(const EmbedFwdParams& p, int id_bytes, cudaStream_t st) {
  return with_lpr_id<8>(lanes_per_row(p.D / 4), id_bytes,
                        [&](auto L, auto id) { return launch_fwd_linx<L, decltype(id)>(p, st); });
}

// DR_EMBED_NO_FM forward: the default (non-LINX, uncapped) mapping at the default unroll
template <int LPR, typename IdT>
static int launch_fwd_nofm(const EmbedFwdParams& p, cudaStream_t st) {
  constexpr int U = (LPR <= 8) ? 8 : 4;
  return launch(embed_fm_fwd_kernel<LPR, IdT, U, false, 0, false, true>, geom(p.B, p.S, LPR, sizeof(IdT)), p, st,
                "embed_fm_fwd(no_fm)");
}

template <int LPR, typename IdT>
static int launch_fwd(const EmbedFwdParams& p, cudaStream_t st) {
  int U = g_tune_embed_fwd_unroll;
  if (U <= 0) U = (LPR <= 8) ? 8 : 4;
  switch (U) {
    case 1: return launch_fwd_u<LPR, IdT, 1>(p, st);
    case 2: return launch_fwd_u<LPR, IdT, 2>(p, st);
    case 4: return launch_fwd_u<LPR, IdT, 4>(p, st);
    case 13: return launch_fwd_u<LPR, IdT, 13>(p, st);
    case 26: return launch_fwd_u<LPR, IdT, 26>(p, st);
    default: return launch_fwd_u<LPR, IdT, 8>(p, st);
  }
}

template <int LPR, typename IdT, int U>
static int launch_bwd_u(const EmbedBwdParams& p, cudaStream_t st) {
  void (*k)(EmbedBwdParams) =
      g_tune_embed_bwd_agg ? embed_fm_bwd_kernel<LPR, IdT, U, true> : embed_fm_bwd_kernel<LPR, IdT, U, false>;
  return launch(k, geom(p.B, p.S, LPR, sizeof(IdT)), p, st, "embed_fm_bwd");
}

// Slot-parallel backward: a warp per example, at most embed_ctas_per_sm (default 8) CTAs of 256 threads per SM.
static int launch_bwd_sp(void (*k)(EmbedBwdParams), const EmbedBwdParams& p, cudaStream_t st, const char* what) {
  const int threads = 256;
  const size_t smem = (size_t)p.S * (sizeof(void*) * 2 + sizeof(int64_t) * 2) + kMaxShardWorld * sizeof(void*);
  const int64_t ctas = capped_grid(p.B, threads / 32, g_tune_embed_ctas_per_sm > 0 ? g_tune_embed_ctas_per_sm : 8);
  // The update runs beside the persistent wgmma weight-gradient GEMM, which configures its SMs with the maximum
  // shared-memory carveout (up to 224 KB of dynamic shared memory).  A kernel that prefers another L1 / shared split cannot
  // become resident on an SM in that configuration, so the update asks for the same carveout (it uses 2 KB either way).
  if (g_tune_embed_bwd_carveout)
    DR_CUDA_CALL(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, g_tune_embed_bwd_carveout));
  k<<<(unsigned)ctas, threads, smem, st>>>(p);
  DR_CUDA_LAUNCH_CHECK(what);
  return DR_OK;
}

template <int LPR, typename IdT, int U, bool LINX = false>
static int launch_bwd_sp_u(const EmbedBwdParams& p, cudaStream_t st) {
  static_assert(!LINX || LPR <= 8, "LINX is instantiated for LPR <= 8 only");
  void (*k)(EmbedBwdParams) = p.shard_world > 0 ? embed_fm_bwd_sp_kernel<LPR, IdT, U, true>
                              : (LINX ? embed_fm_bwd_sp_kernel<LPR, IdT, U, false, LINX>
                                      : embed_fm_bwd_sp_kernel<LPR, IdT, U, false>);
  return launch_bwd_sp(k, p, st, "embed_fm_bwd_sp");
}

// DR_EMBED_NO_FM backward: the slot-parallel kernel (the default mode) whatever the developer mode knob says
template <int LPR, typename IdT>
static int launch_bwd_nofm(const EmbedBwdParams& p, cudaStream_t st) {
  return launch_bwd_sp(embed_fm_bwd_sp_kernel<LPR, IdT, 2, false, false, true>, p, st, "embed_fm_bwd_sp(no_fm)");
}

template <int LPR, typename IdT>
static int launch_bwd(const EmbedBwdParams& p, cudaStream_t st) {
  if (p.mode == 0) {
    switch (g_tune_embed_bwd_unroll) {
      case 1: return launch_bwd_sp_u<LPR, IdT, 1>(p, st);
      case 4: return launch_bwd_sp_u<LPR, IdT, 4>(p, st);
      default: return launch_bwd_sp_u<LPR, IdT, 2>(p, st);
    }
  }
  int U = g_tune_embed_bwd_unroll;
  if (U <= 0) U = 4;
  switch (U) {
    case 1: return launch_bwd_u<LPR, IdT, 1>(p, st);
    case 2: return launch_bwd_u<LPR, IdT, 2>(p, st);
    case 8: return launch_bwd_u<LPR, IdT, 8>(p, st);
    default: return launch_bwd_u<LPR, IdT, 4>(p, st);
  }
}

}  // namespace dr

using namespace dr;

extern "C" int dr_embed_fm_fwd(const float* const* table_ptrs, const float* const* lin_ptrs,
                               const int64_t* rows, const void* ids, int id_bytes, const float* bias,
                               int64_t B, int S, int D, int64_t row_stride, int64_t lin_stride, int flags,
                               float* out_stack, float* out_sum, float* out_logit, void* stream) {
  if (int rc = check_lookup_dims("dr_embed_fm_fwd", B, S, D, id_bytes)) return rc;
  if (B == 0) return DR_OK;
  DR_REQUIRE(table_ptrs && rows && ids, DR_EINVAL, "dr_embed_fm_fwd: null table_ptrs/rows/ids");
  DR_REQUIRE(out_stack || out_logit || out_sum, DR_EINVAL, "dr_embed_fm_fwd: no output requested");
  if (row_stride == 0) row_stride = D;
  if (lin_stride == 0) lin_stride = 1;
  DR_REQUIRE(row_stride >= D && row_stride % 4 == 0, DR_EINVAL,
             "dr_embed_fm_fwd: row_stride=%lld must be >= D and a multiple of 4", (long long)row_stride);
  DR_REQUIRE(lin_stride >= 1, DR_EINVAL, "dr_embed_fm_fwd: lin_stride=%lld < 1", (long long)lin_stride);
  const int lin_in_row = (flags & DR_EMBED_LIN_IN_ROW) ? 1 : 0;
  DR_REQUIRE(!lin_in_row || (row_stride >= D + 4 && D <= 124), DR_EINVAL,
             "dr_embed_fm_fwd: DR_EMBED_LIN_IN_ROW needs row_stride >= D+4 and D <= 124");
  DR_REQUIRE(!out_stack || aligned16(out_stack), DR_EALIGN, "dr_embed_fm_fwd: out_stack not 16-B aligned");
  DR_REQUIRE(!out_sum || aligned16(out_sum), DR_EALIGN, "dr_embed_fm_fwd: out_sum not 16-B aligned");
  EmbedFwdParams p{};
  p.table_ptrs = table_ptrs; p.lin_ptrs = lin_ptrs; p.rows = rows; p.ids = ids; p.bias = bias;
  p.B = B; p.S = S; p.D = D; p.out_stack = out_stack; p.out_sum = out_sum; p.out_logit = out_logit;
  p.row_stride = row_stride; p.lin_stride = lin_stride; p.lin_in_row = lin_in_row;
  p.l2_hints = g_tune_embed_l2_hints;
  cudaStream_t st = (cudaStream_t)stream;
  const int lpr = lanes_per_row(D / 4 + lin_in_row);
  if (flags & DR_EMBED_NO_FM)
    return with_lpr_id(lpr, id_bytes, [&](auto L, auto id) { return launch_fwd_nofm<L, decltype(id)>(p, st); });
  if (g_tune_embed_fwd_linx && lin_in_row && out_logit && lanes_per_row(D / 4) <= 8)
    return dispatch_fwd_linx(p, id_bytes, st);
  return with_lpr_id(lpr, id_bytes, [&](auto L, auto id) { return launch_fwd<L, decltype(id)>(p, st); });
}

extern "C" int dr_embed_fm_bwd(const void* ids, int id_bytes, const int64_t* rows, const float* stack,
                               const float* sum_e, const float* g_logit, const float* g_stack,
                               int64_t B, int S, int D, int64_t row_stride, int64_t lin_stride, int flags,
                               float* const* grad_table_ptrs, float* const* grad_lin_ptrs, float* g_bias,
                               float scale, void* stream) {
  if (int rc = check_lookup_dims("dr_embed_fm_bwd", B, S, D, id_bytes)) return rc;
  if (B == 0) return DR_OK;
  DR_REQUIRE(ids && rows && grad_table_ptrs, DR_EINVAL, "dr_embed_fm_bwd: null ids/rows/grad_table_ptrs");
  DR_REQUIRE(g_logit || g_stack, DR_EINVAL, "dr_embed_fm_bwd: both g_logit and g_stack are NULL");
  DR_REQUIRE(!g_logit || stack, DR_EINVAL, "dr_embed_fm_bwd: g_logit given but stack is NULL");
  DR_REQUIRE(!stack || aligned16(stack), DR_EALIGN, "dr_embed_fm_bwd: stack not 16-B aligned");
  DR_REQUIRE(!g_stack || aligned16(g_stack), DR_EALIGN, "dr_embed_fm_bwd: g_stack not 16-B aligned");
  DR_REQUIRE(!sum_e || aligned16(sum_e), DR_EALIGN, "dr_embed_fm_bwd: sum_e not 16-B aligned");
  if (row_stride == 0) row_stride = D;
  if (lin_stride == 0) lin_stride = 1;
  DR_REQUIRE(row_stride >= D && row_stride % 4 == 0 && lin_stride >= 1, DR_EINVAL,
             "dr_embed_fm_bwd: bad strides row=%lld lin=%lld", (long long)row_stride, (long long)lin_stride);
  const int lin_in_row = (flags & DR_EMBED_LIN_IN_ROW) ? 1 : 0;
  DR_REQUIRE(!lin_in_row || (row_stride >= D + 4 && D <= 124), DR_EINVAL,
             "dr_embed_fm_bwd: DR_EMBED_LIN_IN_ROW needs row_stride >= D+4 and D <= 124");
  EmbedBwdParams p{};
  p.ids = ids; p.rows = rows; p.stack = stack; p.sum_e = sum_e; p.g_logit = g_logit; p.g_stack = g_stack;
  p.B = B; p.S = S; p.D = D; p.grad_table_ptrs = grad_table_ptrs; p.grad_lin_ptrs = grad_lin_ptrs;
  p.g_bias = g_bias; p.scale = scale; p.row_stride = row_stride; p.lin_stride = lin_stride;
  p.lin_in_row = lin_in_row;
  p.l2_hints = g_tune_embed_l2_hints;
  p.mode = g_tune_embed_bwd_mode;
  cudaStream_t st = (cudaStream_t)stream;
  const int lpr = lanes_per_row(D / 4 + lin_in_row);
  if (flags & DR_EMBED_NO_FM)
    return with_lpr_id(lpr, id_bytes, [&](auto L, auto id) { return launch_bwd_nofm<L, decltype(id)>(p, st); });
  if (g_tune_embed_bwd_linx && p.mode == 0 && lin_in_row && g_logit && lanes_per_row(D / 4) <= 8)
    return with_lpr_id<8>(lanes_per_row(D / 4), id_bytes,
                          [&](auto L, auto id) { return launch_bwd_sp_u<L, decltype(id), 2, true>(p, st); });
  return with_lpr_id(lpr, id_bytes, [&](auto L, auto id) { return launch_bwd<L, decltype(id)>(p, st); });
}

extern "C" int dr_gather_fwd(const float* table, int64_t rows, const void* ids, int id_bytes, int64_t n,
                             int D, float* out, void* stream) {
  if (int rc = check_lookup_dims("dr_gather_fwd", n, 1, D, id_bytes)) return rc;
  if (n == 0) return DR_OK;
  DR_REQUIRE(table && ids && out, DR_EINVAL, "dr_gather_fwd: null pointer");
  DR_REQUIRE(rows >= 0, DR_EINVAL, "dr_gather_fwd: rows < 0");
  DR_REQUIRE(aligned16(table) && aligned16(out), DR_EALIGN, "dr_gather_fwd: table/out not 16-B aligned");
  const int chunks = D / 4;
  const int64_t ctas = capped_grid(n * chunks, 256, 8);
  return with_id_type(id_bytes, [&](auto id) {
    using IdT = decltype(id);
    gather_rows_kernel<IdT><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(table, rows, (const IdT*)ids, n, chunks, out);
    DR_CUDA_LAUNCH_CHECK("gather_rows");
    return DR_OK;
  });
}

extern "C" int dr_scatter_add(float* grad_table, int64_t rows, const void* ids, int id_bytes, int64_t n,
                              int D, const float* g, float scale, void* stream) {
  if (int rc = check_lookup_dims("dr_scatter_add", n, 1, D, id_bytes)) return rc;
  if (n == 0) return DR_OK;
  DR_REQUIRE(grad_table && ids && g, DR_EINVAL, "dr_scatter_add: null pointer");
  DR_REQUIRE(rows >= 0, DR_EINVAL, "dr_scatter_add: rows < 0");
  DR_REQUIRE(aligned16(grad_table) && aligned16(g), DR_EALIGN, "dr_scatter_add: table/g not 16-B aligned");
  const int chunks = D / 4;
  const int64_t ctas = capped_grid(n * chunks, 256, 8);
  return with_id_type(id_bytes, [&](auto id) {
    using IdT = decltype(id);
    scatter_add_rows_kernel<IdT><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(grad_table, rows, (const IdT*)ids, n,
                                                                                   chunks, g, scale);
    DR_CUDA_LAUNCH_CHECK("scatter_add_rows");
    return DR_OK;
  });
}

// ---- row-sharded entries: the gather / scatter IS the exchange (NVLink peer memory) -------------------
extern "C" int dr_embed_fm_fwd_sharded(const float* const* peer_bases, int world, const int64_t* slot_offsets,
                                       const int64_t* rows, const void* ids, int id_bytes, const float* bias,
                                       int64_t B, int S, int D, int64_t row_stride, int flags, int64_t lin_offset,
                                       float* out_stack, float* out_sum, float* out_logit, void* stream) {
  if (int rc = check_lookup_dims("dr_embed_fm_fwd_sharded", B, S, D, id_bytes)) return rc;
  DR_REQUIRE(!(flags & DR_EMBED_NO_FM), DR_ENOTSUP, "dr_embed_fm_fwd_sharded: DR_EMBED_NO_FM is not served");
  DR_REQUIRE(lin_offset >= 0 && !((flags & DR_EMBED_LIN_IN_ROW) && lin_offset > 0), DR_EINVAL,
             "dr_embed_fm_fwd_sharded: lin_offset=%lld (must be >= 0 and exclusive with DR_EMBED_LIN_IN_ROW)",
             (long long)lin_offset);
  if (B == 0) return DR_OK;
  DR_REQUIRE(peer_bases && slot_offsets && rows && ids, DR_EINVAL, "dr_embed_fm_fwd_sharded: null pointer");
  DR_REQUIRE(world >= 1 && world <= kMaxShardWorld, DR_EINVAL, "dr_embed_fm_fwd_sharded: world=%d outside [1,%d]",
             world, kMaxShardWorld);
  DR_REQUIRE(out_stack || out_logit || out_sum, DR_EINVAL, "dr_embed_fm_fwd_sharded: no output requested");
  const int lin_in_row = (flags & DR_EMBED_LIN_IN_ROW) ? 1 : 0;
  DR_REQUIRE(row_stride >= D + (lin_in_row ? 4 : 0) && row_stride % 4 == 0 && (!lin_in_row || D <= 124), DR_EINVAL,
             "dr_embed_fm_fwd_sharded: bad row_stride=%lld for D=%d", (long long)row_stride, D);
  DR_REQUIRE(!out_stack || aligned16(out_stack), DR_EALIGN, "dr_embed_fm_fwd_sharded: out_stack not 16-B aligned");
  EmbedFwdParams p{};
  p.rows = rows; p.ids = ids; p.bias = bias; p.B = B; p.S = S; p.D = D;
  p.out_stack = out_stack; p.out_sum = out_sum; p.out_logit = out_logit;
  p.row_stride = row_stride; p.lin_stride = row_stride; p.lin_in_row = lin_in_row;
  p.shard_world = world; p.peer_bases = peer_bases; p.slot_offsets = slot_offsets; p.shard_lin_off = lin_offset;
  cudaStream_t st = (cudaStream_t)stream;
  if (g_tune_embed_fwd_linx_shard && lin_in_row && out_logit && lanes_per_row(D / 4) <= 8)
    return dispatch_fwd_linx(p, id_bytes, st);
  return with_lpr_id(lanes_per_row(D / 4 + lin_in_row), id_bytes,
                     [&](auto L, auto id) { return launch_fwd<L, decltype(id)>(p, st); });
}

extern "C" int dr_embed_fm_bwd_sharded(float* const* peer_bases, int world, const int64_t* slot_offsets,
                                       const int64_t* rows, const void* ids, int id_bytes, const float* stack,
                                       const float* sum_e, const float* g_logit, const float* g_stack, int64_t B,
                                       int S, int D, int64_t row_stride, int flags, int64_t lin_offset, float* g_bias,
                                       float scale, void* stream) {
  if (int rc = check_lookup_dims("dr_embed_fm_bwd_sharded", B, S, D, id_bytes)) return rc;
  DR_REQUIRE(!(flags & DR_EMBED_NO_FM), DR_ENOTSUP, "dr_embed_fm_bwd_sharded: DR_EMBED_NO_FM is not served");
  DR_REQUIRE(lin_offset >= 0 && !((flags & DR_EMBED_LIN_IN_ROW) && lin_offset > 0), DR_EINVAL,
             "dr_embed_fm_bwd_sharded: lin_offset=%lld (must be >= 0 and exclusive with DR_EMBED_LIN_IN_ROW)",
             (long long)lin_offset);
  if (B == 0) return DR_OK;
  DR_REQUIRE(peer_bases && slot_offsets && rows && ids, DR_EINVAL, "dr_embed_fm_bwd_sharded: null pointer");
  DR_REQUIRE(world >= 1 && world <= kMaxShardWorld, DR_EINVAL, "dr_embed_fm_bwd_sharded: world=%d outside [1,%d]",
             world, kMaxShardWorld);
  DR_REQUIRE(g_logit || g_stack, DR_EINVAL, "dr_embed_fm_bwd_sharded: both g_logit and g_stack are NULL");
  DR_REQUIRE(!g_logit || stack, DR_EINVAL, "dr_embed_fm_bwd_sharded: g_logit given but stack is NULL");
  const int lin_in_row = (flags & DR_EMBED_LIN_IN_ROW) ? 1 : 0;
  DR_REQUIRE(row_stride >= D + (lin_in_row ? 4 : 0) && row_stride % 4 == 0 && (!lin_in_row || D <= 124), DR_EINVAL,
             "dr_embed_fm_bwd_sharded: bad row_stride=%lld for D=%d", (long long)row_stride, D);
  EmbedBwdParams p{};
  p.ids = ids; p.rows = rows; p.stack = stack; p.sum_e = sum_e; p.g_logit = g_logit; p.g_stack = g_stack;
  p.B = B; p.S = S; p.D = D; p.g_bias = g_bias; p.scale = scale;
  p.row_stride = row_stride; p.lin_stride = row_stride; p.lin_in_row = lin_in_row;
  p.shard_world = world; p.peer_bases = peer_bases; p.slot_offsets = slot_offsets; p.shard_lin_off = lin_offset;
  p.mode = 0;                     // only the slot-parallel kernel implements sharded addressing
  cudaStream_t st = (cudaStream_t)stream;
  return with_lpr_id(lanes_per_row(D / 4 + lin_in_row), id_bytes,
                     [&](auto L, auto id) { return launch_bwd<L, decltype(id)>(p, st); });
}
