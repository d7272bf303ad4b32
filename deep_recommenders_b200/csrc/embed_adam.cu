// SURVEY.md 8(f) #1 proper: Adam for the embedding tables INSIDE the backward scatter path (one kernel), row-sparse.
//
// Reference call sites: examples/train_deepfm_on_movielens_keras.py:44 (tf.keras.optimizers.Adam()),
// examples/train_fm_on_movielens_estimator.py:51 (tf.train.AdamOptimizer(0.01)).
//
// Adam is not linear in the gradient, so the row gradient must be complete (summed over every lookup of that row in
// the batch) before (p, m, v) move.  One kernel does both phases with a per-row countdown:
//   0. dr_embed_adam_count (tiny, runs early in the step on a side stream): count[row] += 1 per lookup.
//   1. dr_embed_fm_bwd_adam: every lookup adds its gradient row into the row's state block with vector atomics
//      (red.global.add.v4.f32), fences, and decrements count[row]; the lane group that takes the count to zero is the
//      LAST contributor of that row: it reads the finished gradient, applies TensorFlow's ApplyAdam functor to the
//      row's 16-B chunks of (p, m, v) -- the arithmetic of dr_adam_step, bit for bit -- and clears the gradient, so the
//      state block is ready for the next step.  No dense gradient arena sweep, no second kernel, no per-row stamp.
// Per-row state lives in ONE block of `stride` floats ([g D | m D | v D | g_w m_w v_w count | pad], 128-B multiple,
// same DRAM page): a touched row costs the parameter line plus this block.
//
// Semantics: rows the batch did not touch keep p, m, v (tfa.optimizers.LazyAdam).  tf.keras Adam additionally decays m, v
// of EVERY row each step and moves every row by its decayed momentum (dr_adam_step over the arena is that exact form, at
// 7 arena sweeps per step); this is the documented deviation of the row-sparse form.  On the rows a step touches the
// update is TensorFlow's functor exactly.
#include "adam.cuh"

namespace dr {

template <typename IdT>
__global__ void __launch_bounds__(256) embed_adam_count_kernel(const IdT* __restrict__ ids, int64_t n, int S,
                                                                const int64_t* __restrict__ rows,
                                                                const int64_t* __restrict__ slot_offsets,
                                                                float* __restrict__ state, int SS, int cnt_off) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int s = (int)(i % S);
    const int64_t id = (int64_t)__ldg(ids + i);
    if ((uint64_t)id < (uint64_t)__ldg(rows + s))
      atomicAdd(reinterpret_cast<int*>(state + (size_t)(__ldg(slot_offsets + s) + id) * SS + cnt_off), 1);
  }
}

// EXACT, before the forward: count the batch's lookups per row (as embed_adam_count_kernel) AND bring every row the batch
// touches up to date with step t-1, so that the forward reads what tf.keras Adam's dense update would have left there.
// One lane group per lookup; the lookup that raises a row's count from 0 is the row's first arriver and replays the
// row's pending steps (stamp, t-1]; the others only count.
template <int LPR, typename IdT>
__global__ void __launch_bounds__(256) embed_adam_prepare_kernel(const IdT* __restrict__ ids, int64_t n_lookups, int S, int D,
                                                                  const int64_t* __restrict__ rows,
                                                                  const int64_t* __restrict__ slot_offsets,
                                                                  float* const* __restrict__ table_ptrs,
                                                                  float* const* __restrict__ lin_ptrs, int64_t row_stride,
                                                                  int64_t lin_stride, int lin_in_row,
                                                                  float* __restrict__ state, int SS,
                                                                  const int64_t* __restrict__ step_dev, AdamHist hist,
                                                                  float omb1, float omb2, float eps) {
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31, c = lane % LPR, grp = lane / LPR;
  const int64_t t_now = *step_dev;
  const int o_m = D, o_v = 2 * D, o_s = 3 * D;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t base = warp * G; base < n_lookups; base += nwarps * G) {
    const int64_t L = base + grp;
    int64_t id = -1;
    int s = 0;
    if (L < n_lookups) {
      s = (int)(L % S);
      id = (int64_t)__ldg(ids + L);
      if ((uint64_t)id >= (uint64_t)__ldg(rows + s)) id = -1;
    }
    float* st = id >= 0 ? state + (size_t)(__ldg(slot_offsets + s) + id) * SS : nullptr;
    int first = 0, stamp_i = 0;
    if (id >= 0 && c == 0) {
      first = atomicAdd(reinterpret_cast<int*>(st + o_s + 3), 1) == 0;
      if (first) stamp_i = __float_as_int(ld_cg1(st + o_s + 4));
    }
    first = __shfl_sync(0xffffffffu, first, grp * LPR);
    stamp_i = __shfl_sync(0xffffffffu, stamp_i, grp * LPR);
    const int64_t stamp = stamp_i;
    if (first && stamp > 0 && stamp < t_now - 1) {
      float* prow = table_ptrs[s] + (size_t)id * row_stride;
      if (c * 4 < D)
        adam_replay_chunk<LdCg>(st, o_m, o_v, prow, c * 4, stamp, t_now - 1, t_now, hist, omb1,
                                omb2, eps);
      if (c == 0) {
        if (lin_in_row || lin_ptrs) {
          float* wp = lin_in_row ? prow + D : lin_ptrs[s] + (size_t)id * lin_stride;
          adam_replay_weight<LdCg>(wp, st, o_s, stamp, t_now - 1, t_now, hist, omb1, omb2, eps);
        }
        st[o_s + 4] = __int_as_float((int)(t_now - 1));
      }
    }
  }
}

struct AdamBwdParams {
  const void* ids;
  const int64_t* rows;
  const int64_t* slot_offsets;
  const float* stack;
  const float* sum_e;
  const float* g_logit;
  const float* g_stack;
  int64_t B;
  int S, D;
  float* const* table_ptrs;
  float* const* lin_ptrs;
  int64_t row_stride, lin_stride;
  int lin_in_row;
  float* state;
  int SS;
  float* g_bias;
  const float* lr_t_dev;
  float omb1, omb2, eps;
  const int64_t* step_dev;     // EXACT: current step t (dr_adam_advance_hist)
  AdamHist hist;
};

// Slot-parallel mapping of embed_fm_bwd_sp_kernel: a warp walks examples, its lane groups take consecutive slots.
template <int LPR, typename IdT, bool EXACT>
__global__ void __launch_bounds__(256) embed_fm_bwd_adam_kernel(const AdamBwdParams p) {
  constexpr int SPW = 32 / LPR;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ float s_bias_part[8];
  const int S = p.S, D = p.D;
  float** s_tab = reinterpret_cast<float**>(smem_raw);
  float** s_lin = s_tab + S;
  int64_t* s_rows = reinterpret_cast<int64_t*>(s_lin + S);
  int64_t* s_off = s_rows + S;
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    s_tab[i] = p.table_ptrs[i];
    s_lin[i] = p.lin_ptrs ? p.lin_ptrs[i] : nullptr;
    s_rows[i] = p.rows[i];
    s_off[i] = p.slot_offsets[i];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp_in_cta = threadIdx.x >> 5, warps_per_cta = blockDim.x >> 5;
  const int c = lane % LPR, sg = lane / LPR;
  const bool chunk_ok = (c * 4) < D;
  const bool has_fm = p.g_logit != nullptr, has_gs = p.g_stack != nullptr;
  const bool has_w = has_fm && (p.lin_in_row || p.lin_ptrs != nullptr);     // a first-order weight exists and gets a gradient
  const IdT* __restrict__ ids = reinterpret_cast<const IdT*>(p.ids);
  const int64_t warp0 = (int64_t)blockIdx.x * warps_per_cta + warp_in_cta;
  const int64_t nwarps = (int64_t)gridDim.x * warps_per_cta;
  const float lr_t = __ldg(p.lr_t_dev);
  const float omb1 = p.omb1, omb2 = p.omb2, eps = p.eps;
  const int SS = p.SS, o_m = D, o_v = 2 * D, o_s = 3 * D;
  const int64_t t_now = EXACT ? *p.step_dev : 0;
  float bias_acc = 0.f;

  for (int64_t b = warp0; b < p.B; b += nwarps) {
    const float gl = has_fm ? __ldg(p.g_logit + b) : 0.f;
    if (lane == 0) bias_acc += gl;
    float4 sum = f4_zero();
    if (has_fm && chunk_ok) {
      if (p.sum_e) {
        sum = ldg4(p.sum_e + (size_t)b * D + c * 4);
      } else {
        for (int s = 0; s < S; ++s) sum = f4_add(sum, ldg4(p.stack + ((size_t)b * S + s) * D + c * 4));
      }
    }
    const IdT* my_ids = ids + (size_t)b * S;
    const size_t ex0 = (size_t)b * S * D + c * 4;
    for (int s0 = 0; s0 < S; s0 += SPW) {       // trip count is warp-uniform: every lane reaches the barriers below
      const int s = s0 + sg;
      int64_t id = -1;
      float4 e = f4_zero(), gs = f4_zero();
      if (s < S) {
        id = (int64_t)__ldg(my_ids + s);
        if (chunk_ok) {
          if (has_fm) e = ldg_nc_na(p.stack + ex0 + (size_t)s * D);
          if (has_gs) gs = ldg_nc_na(p.g_stack + ex0 + (size_t)s * D);
        }
      }
      const bool valid = s < S && (uint64_t)id < (uint64_t)s_rows[s];
      float* st = nullptr;
      if (valid) {
        st = p.state + (size_t)(s_off[s] + id) * SS;
        if (chunk_ok) {
          float4 d;
          d.x = fmaf(gl, sum.x - e.x, gs.x);
          d.y = fmaf(gl, sum.y - e.y, gs.y);
          d.z = fmaf(gl, sum.z - e.z, gs.z);
          d.w = fmaf(gl, sum.w - e.w, gs.w);
          red_add_v4(st + c * 4, d);
        }
        if (c == 0 && has_w) red_add_f32(st + o_s, gl);
      }
      __threadfence();     // this lane's contributions are performed before the group leader announces them
      __syncwarp();
      int old = 0;
      if (valid && c == 0) old = atomicSub(reinterpret_cast<int*>(st + o_s + 3), 1);
      old = __shfl_sync(0xffffffffu, old, sg * LPR);
      int stamp_i = 0;             // EXACT: the row's step stamp, read by the group leader, broadcast while the warp is converged
      if (EXACT) {
        if (valid && c == 0 && old == 1) stamp_i = __float_as_int(ld_cg1(st + o_s + 4));
        stamp_i = __shfl_sync(0xffffffffu, stamp_i, sg * LPR);
      }
      if (valid && old == 1) {     // last contributor of this row in this batch: the gradient is complete
        __threadfence();
        float* prow = s_tab[s] + (size_t)id * p.row_stride;
        const int64_t stamp = stamp_i;
        if (chunk_ok) {
          const float4 g = ld_cg4(st + c * 4);
          float4 m = ld_cg4(st + o_m + c * 4), v = ld_cg4(st + o_v + c * 4);
          float4 w = *reinterpret_cast<const float4*>(prow + c * 4);
          if (EXACT)     // replay the steps this row sat out, then take this step's update
            adam_catch_up4(w, m, v, stamp, t_now - 1, t_now, p.hist, omb1, omb2, eps);
          adam_functor(w.x, g.x, m.x, v.x, lr_t, omb1, omb2, eps);
          adam_functor(w.y, g.y, m.y, v.y, lr_t, omb1, omb2, eps);
          adam_functor(w.z, g.z, m.z, v.z, lr_t, omb1, omb2, eps);
          adam_functor(w.w, g.w, m.w, v.w, lr_t, omb1, omb2, eps);
          *reinterpret_cast<float4*>(prow + c * 4) = w;
          stg4(st + o_m + c * 4, m);
          stg4(st + o_v + c * 4, v);
          stg4(st + c * 4, f4_zero());
        }
        if (c == 0 && has_w) {
          float* wp = p.lin_in_row ? prow + D : s_lin[s] + (size_t)id * p.lin_stride;
          float w = *wp, m = ld_cg1(st + o_s + 1), v = ld_cg1(st + o_s + 2);
          const float g = ld_cg1(st + o_s);
          if (EXACT) adam_catch_up1(w, m, v, stamp, t_now - 1, t_now, p.hist, omb1, omb2, eps);
          adam_functor(w, g, m, v, lr_t, omb1, omb2, eps);
          *wp = w;
          st[o_s + 1] = m;
          st[o_s + 2] = v;
          st[o_s] = 0.f;
        }
        if (EXACT && c == 0) st[o_s + 4] = __int_as_float((int)t_now);
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
      red_add_f32(p.g_bias, t);
    }
  }
}

// EXACT: bring EVERY row up to date with step `t_now` (before reading the tables for evaluation / a checkpoint):
// one lane group per table row, rows whose stamp is already t_now are skipped.
template <int LPR>
__global__ void __launch_bounds__(256) embed_adam_flush_kernel(float* const* __restrict__ table_ptrs,
                                                                float* const* __restrict__ lin_ptrs,
                                                                const int64_t* __restrict__ rows,
                                                                const int64_t* __restrict__ slot_offsets, int S, int D,
                                                                int64_t row_stride, int64_t lin_stride, int lin_in_row,
                                                                float* __restrict__ state, int SS, int64_t total_rows,
                                                                const int64_t* __restrict__ step_dev, AdamHist hist,
                                                                float omb1, float omb2, float eps) {
  const int lane = threadIdx.x & 31, c = lane % LPR, grp = lane / LPR;
  constexpr int G = 32 / LPR;
  const int64_t t_now = *step_dev;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int o_m = D, o_v = 2 * D, o_s = 3 * D;
  for (int64_t base = warp * G; base < total_rows; base += nwarps * G) {
    const int64_t r = base + grp;
    const bool in = r < total_rows;
    float* st = state + (size_t)(in ? r : 0) * SS;
    const int64_t stamp = in ? (int64_t)__float_as_int(st[o_s + 4]) : 0;   // every lane reads its group's stamp ...
    __syncwarp();                                                         // ... before any lane of the warp writes one
    if (!in || stamp <= 0 || stamp >= t_now) continue;
    int s = 0;                                             // table of global row r (S is small: linear scan)
    while (s + 1 < S && __ldg(slot_offsets + s + 1) <= r) ++s;
    const int64_t id = r - __ldg(slot_offsets + s);
    float* prow = table_ptrs[s] + (size_t)id * row_stride;
    if (c * 4 < D)
      adam_replay_chunk<LdPlain>(st, o_m, o_v, prow, c * 4, stamp, t_now, t_now, hist, omb1,
                                 omb2, eps);
    if (c == 0 && (lin_in_row || lin_ptrs)) {
      float* wp = lin_in_row ? prow + D : lin_ptrs[s] + (size_t)id * lin_stride;
      adam_replay_weight<LdPlain>(wp, st, o_s, stamp, t_now, t_now, hist, omb1, omb2, eps);
    }
    if (c == 0) st[o_s + 4] = __int_as_float((int)t_now);
  }
}

// ---- the same tf.keras-equal Adam for the layer API (optimizers.RowSparseAdam) ----------------------------------------
// There a forward may run without a backward (evaluation), so the forward-side pass must leave no count behind:
//   catch_up : before a forward, bring every row the lookups read up to the current step t_now (the flush, restricted to
//              the batch's rows).  The lane group whose CAS moves the row's stamp to t_now replays (stamp, t_now].
//   rows_tf  : after the clock has advanced to t, step t from per-lookup gradient rows given with strides (FNN's input
//              row, a [B, S, D] stack gradient, a bag's row gradient), counted beforehand by dr_embed_adam_count; the
//              count / accumulate / last-applies scheme of embed_fm_bwd_adam_kernel on the same state blocks.
template <int LPR, typename IdT>
__global__ void __launch_bounds__(256) embed_adam_catch_up_kernel(const IdT* __restrict__ ids, int64_t n_lookups, int S,
                                                                   int D, const int64_t* __restrict__ rows,
                                                                   const int64_t* __restrict__ slot_offsets,
                                                                   float* const* __restrict__ table_ptrs,
                                                                   float* const* __restrict__ lin_ptrs, int64_t row_stride,
                                                                   int64_t lin_stride, int lin_in_row,
                                                                   float* __restrict__ state, int SS,
                                                                   const int64_t* __restrict__ step_dev, AdamHist hist,
                                                                   float omb1, float omb2, float eps) {
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31, c = lane % LPR, grp = lane / LPR;
  const int64_t t_now = *step_dev;
  const int o_m = D, o_v = 2 * D, o_s = 3 * D;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t base = warp * G; base < n_lookups; base += nwarps * G) {
    const int64_t L = base + grp;
    int64_t id = -1;
    int s = 0;
    if (L < n_lookups) {
      s = (int)(L % S);
      id = (int64_t)__ldg(ids + L);
      if ((uint64_t)id >= (uint64_t)__ldg(rows + s)) id = -1;
    }
    float* st = id >= 0 ? state + (size_t)(__ldg(slot_offsets + s) + id) * SS : nullptr;
    int won = 0, stamp_i = 0;
    if (id >= 0 && c == 0) {
      stamp_i = __float_as_int(ld_cg1(st + o_s + 4));
      if (stamp_i > 0 && stamp_i < t_now)      // never updated (m = v = 0) or already current: nothing to replay
        won = atomicCAS(reinterpret_cast<int*>(st + o_s + 4), stamp_i, (int)t_now) == stamp_i;
    }
    won = __shfl_sync(0xffffffffu, won, grp * LPR);
    stamp_i = __shfl_sync(0xffffffffu, stamp_i, grp * LPR);
    if (!won) continue;
    const int64_t stamp = stamp_i;
    float* prow = table_ptrs[s] + (size_t)id * row_stride;
    if (c * 4 < D)
      adam_replay_chunk<LdCg>(st, o_m, o_v, prow, c * 4, stamp, t_now, t_now, hist, omb1, omb2,
                              eps);
    if (c == 0 && (lin_in_row || lin_ptrs)) {
      float* wp = lin_in_row ? prow + D : lin_ptrs[s] + (size_t)id * lin_stride;
      adam_replay_weight<LdCg>(wp, st, o_s, stamp, t_now, t_now, hist, omb1, omb2, eps);
    }
  }
}

struct AdamRowsParams {
  const void* ids;
  const int64_t* row_splits;     // bags: lookup L is a member of bag b, row_splits[b] <= L < row_splits[b + 1] (S == 1)
  int64_t n, B;
  int S, D;
  const int64_t* rows;
  const int64_t* slot_offsets;
  const float* g_emb;            // gradient row of lookup (b, s) at g_emb + b * g_ld + s * g_slot
  int64_t g_ld, g_slot;
  const float* g_lin;            // nullable: first-order gradient of lookup (b, s) at g_lin + b * gl_ld + s * gl_slot
  int64_t gl_ld, gl_slot;
  float* const* table_ptrs;
  float* const* lin_ptrs;
  int64_t row_stride, lin_stride;
  int lin_in_row;
  float* state;
  int SS;
  const int64_t* step_dev;
  const float* lr_t_dev;
  AdamHist hist;
  float omb1, omb2, eps;
};

template <int LPR, typename IdT, bool BAGS>
__global__ void __launch_bounds__(256) embed_adam_rows_tf_kernel(const AdamRowsParams p) {
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31, c = lane % LPR, grp = lane / LPR;
  const int D = p.D, SS = p.SS, o_m = D, o_v = 2 * D, o_s = 3 * D;
  const bool chunk_ok = c * 4 < D;
  const bool has_w = p.g_lin != nullptr;
  const IdT* __restrict__ ids = reinterpret_cast<const IdT*>(p.ids);
  const int64_t t_now = *p.step_dev;
  const float lr_t = __ldg(p.lr_t_dev);
  const float omb1 = p.omb1, omb2 = p.omb2, eps = p.eps;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t base = warp * G; base < p.n; base += nwarps * G) {     // warp-uniform trip count: the shuffles below
    const int64_t L = base + grp;
    int64_t id = -1, b = 0;
    int s = 0;
    float den = 1.f;
    if (L < p.n) {
      id = (int64_t)__ldg(ids + L);
      if (BAGS) {                                       // the bag of member L: the last b with row_splits[b] <= L
        int64_t lo = 0, hi = p.B;
        while (hi - lo > 1) {
          const int64_t mid = (lo + hi) >> 1;
          if (__ldg(p.row_splits + mid) <= L) lo = mid; else hi = mid;
        }
        b = lo;
      } else {
        s = (int)(L % p.S);
        b = L / p.S;
      }
      const int64_t nrows = __ldg(p.rows + s);
      if ((uint64_t)id >= (uint64_t)nrows) {
        id = -1;
      } else if (BAGS) {                                // mean combiner: the bag's valid members share its gradient
        int cnt = 0;
        for (int64_t j = __ldg(p.row_splits + b), e = __ldg(p.row_splits + b + 1); j < e; ++j) {
          const int64_t q = (int64_t)__ldg(ids + j);
          cnt += (q >= 0 && q < nrows) ? 1 : 0;
        }
        den = (float)cnt;
      }
    }
    float* st = nullptr;
    if (id >= 0) {
      st = p.state + (size_t)(__ldg(p.slot_offsets + s) + id) * SS;
      if (chunk_ok) {
        float4 g = ldg4(p.g_emb + (size_t)b * p.g_ld + (size_t)s * p.g_slot + c * 4);
        if (BAGS) g = make_float4(g.x / den, g.y / den, g.z / den, g.w / den);
        red_add_v4(st + c * 4, g);
      }
      if (c == 0 && has_w) red_add_f32(st + o_s, __ldg(p.g_lin + (size_t)b * p.gl_ld + (size_t)s * p.gl_slot));
    }
    __threadfence();     // this lane's contributions are performed before the group leader announces them
    __syncwarp();
    int old = 0;
    if (id >= 0 && c == 0) old = atomicSub(reinterpret_cast<int*>(st + o_s + 3), 1);
    old = __shfl_sync(0xffffffffu, old, grp * LPR);
    int stamp_i = 0;
    if (id >= 0 && c == 0 && old == 1) stamp_i = __float_as_int(ld_cg1(st + o_s + 4));
    stamp_i = __shfl_sync(0xffffffffu, stamp_i, grp * LPR);
    if (id < 0 || old != 1) continue;                  // not the last contributor of this row in this step
    __threadfence();
    const int64_t stamp = stamp_i;
    float* prow = p.table_ptrs[s] + (size_t)id * p.row_stride;
    if (chunk_ok)
      adam_replay_step_chunk(st + c * 4, st + o_m + c * 4, st + o_v + c * 4, prow + c * 4, stamp, t_now - 1, t_now,
                                   p.hist, lr_t, omb1, omb2, eps);
    if (c == 0) {
      if (has_w) {
        float* wp = p.lin_in_row ? prow + D : p.lin_ptrs[s] + (size_t)id * p.lin_stride;
        adam_replay_step_weight(wp, st, o_s, stamp, t_now - 1, t_now, p.hist, lr_t,
                                      omb1, omb2, eps);
      }
      st[o_s + 4] = __int_as_float((int)t_now);
    }
  }
}

__global__ void adam_advance_hist_kernel(int64_t* step, float lr, float b1, float b2, float* lr_t, float* lr_hist,
                                         int hist_len) {
  const int64_t t = *step + 1;
  *step = t;
  const double p1 = pow((double)b1, (double)t), p2 = pow((double)b2, (double)t);
  const float v = (float)((double)lr * sqrt(1.0 - p2) / (1.0 - p1));
  *lr_t = v;
  if (lr_hist && hist_len > 0) lr_hist[t % hist_len] = v;
}

// ---- the same tf.keras-equal Adam on a row-sharded table (owner(r) = r mod G, local row r div G) ----------------------
// Every cross-rank access is a plain store (mark) or a vector red.add (the backward into the owners' gradient arenas),
// and nothing reads it before the ranks meet at a barrier; all Adam arithmetic runs on the owner, in its own memory:
//   mark    : touch[owner][local] = t for every valid lookup (idempotent stores: races between ranks are harmless)
//   prepare : the owner collects its rows with touch == t into `list` / `count` and replays their pending steps (stamp,
//             t-1] (as embed_adam_prepare_kernel), so the forward reads what dense Adam would have left there
//   apply   : after the backward, step t on every listed row from its gradient row (then zeroed); stamp = t.
// The gradient arena and the shard share one layout (row stride, first-order weight in the row or trailing at
// lin_offset); the state blocks are those of dr_embed_adam_state_stride, so dr_embed_adam_flush runs on them unchanged.
template <typename IdT>
__global__ void __launch_bounds__(256) shard_adam_mark_kernel(const IdT* __restrict__ ids, int64_t n, int S,
                                                               const int64_t* __restrict__ slot_offsets,
                                                               const int64_t* __restrict__ rows, int W,
                                                               int32_t* const* __restrict__ touch_bases,
                                                               const int64_t* __restrict__ step_dev) {
  const int32_t t = (int32_t)*step_dev;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int s = (int)(i % S);
    const int64_t id = (int64_t)__ldg(ids + i);
    if ((uint64_t)id >= (uint64_t)__ldg(rows + s)) continue;     // -1 padding, out-of-vocabulary ids
    const int64_t r = __ldg(slot_offsets + s) + id;
    touch_bases[r % W][r / W] = t;
  }
}

__device__ __forceinline__ float* lin_at(float* base, float* row, int64_t r, int D, int lin_in_row, int64_t lin_off) {
  return lin_in_row ? row + D : base + lin_off + r;
}

template <int LPR>
__global__ void __launch_bounds__(256) shard_adam_prepare_kernel(const int32_t* __restrict__ touch, int64_t n_rows,
                                                                  int32_t* __restrict__ list, int32_t* __restrict__ count,
                                                                  float* __restrict__ w, int64_t row_stride,
                                                                  int64_t lin_off, int lin_in_row,
                                                                  float* __restrict__ state, int SS, int D,
                                                                  const int64_t* __restrict__ step_dev, AdamHist hist,
                                                                  float omb1, float omb2, float eps) {
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31, c = lane % LPR, grp = lane / LPR;
  const int64_t t_now = *step_dev;
  const int o_m = D, o_v = 2 * D, o_s = 3 * D;
  const bool has_lin = lin_in_row || lin_off > 0;
  // one list slot reservation per CTA pass (not per warp: a single counter serialises its atomics)
  __shared__ int s_cnt[8], s_pos[8];
  const int wid = threadIdx.x >> 5;
  for (int64_t cbase = (int64_t)blockIdx.x * 256; cbase < n_rows; cbase += (int64_t)gridDim.x * 256) {   // CTA-uniform
    const int64_t base = cbase + wid * 32;
    const int64_t r = base + lane;
    const bool hit = r < n_rows && __ldcg(touch + r) == (int32_t)t_now;         // marks of other ranks: not via L1
    const unsigned mask = __ballot_sync(0xffffffffu, hit);
    const int nhit = __popc(mask);
    if (lane == 0) s_cnt[wid] = nhit;
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int w = 0; w < 8; ++w) { s_pos[w] = tot; tot += s_cnt[w]; }
      const int pos0 = tot ? atomicAdd(count, tot) : 0;
      for (int w = 0; w < 8; ++w) s_pos[w] += pos0;
    }
    __syncthreads();
    if (hit) list[s_pos[wid] + __popc(mask & ((1u << lane) - 1u))] = (int32_t)r;
    __syncthreads();                                                            // s_pos is rewritten next pass
    for (int k = 0; k < nhit; k += G) {                                         // G hit rows at a time, one per group
      const int j = k + grp;
      int64_t row = -1;
      if (j < nhit) {
        unsigned m = mask;
        for (int q = 0; q < j; ++q) m &= m - 1u;
        row = base + (__ffs(m) - 1);
      }
      float* st = state + (size_t)(row >= 0 ? row : 0) * SS;
      const int64_t stamp = row >= 0 ? (int64_t)__float_as_int(st[o_s + 4]) : 0;   // every lane reads the stamp ...
      __syncwarp();                                                               // ... before its leader rewrites it
      if (row < 0 || stamp <= 0 || stamp >= t_now - 1) continue;
      float* prow = w + (size_t)row * row_stride;
      if (c * 4 < D)
        adam_replay_chunk<LdPlain>(st, o_m, o_v, prow, c * 4, stamp, t_now - 1, t_now, hist,
                                   omb1, omb2, eps);
      if (c == 0) {
        if (has_lin)
          adam_replay_weight<LdPlain>(lin_at(w, prow, row, D, lin_in_row, lin_off), st, o_s, stamp,
                                      t_now - 1, t_now, hist, omb1, omb2, eps);
        st[o_s + 4] = __int_as_float((int)(t_now - 1));
      }
    }
  }
}

template <int LPR>
__global__ void __launch_bounds__(256) shard_adam_apply_kernel(const int32_t* __restrict__ list,
                                                                const int32_t* __restrict__ count,
                                                                float* __restrict__ w, float* __restrict__ g,
                                                                int64_t row_stride, int64_t lin_off, int lin_in_row,
                                                                float* __restrict__ state, int SS, int D,
                                                                const int64_t* __restrict__ step_dev,
                                                                const float* __restrict__ lr_t_dev, float omb1,
                                                                float omb2, float eps) {
  constexpr int G = 32 / LPR;
  const int lane = threadIdx.x & 31, c = lane % LPR, grp = lane / LPR;
  const int64_t n = *count;
  const int t_now = (int)*step_dev;
  const float lr_t = __ldg(lr_t_dev);
  const int o_m = D, o_v = 2 * D, o_s = 3 * D;
  const bool has_lin = lin_in_row || lin_off > 0;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp * G + grp; i < n; i += nwarps * G) {
    const int64_t r = __ldg(list + i);
    float* st = state + (size_t)r * SS;
    float* prow = w + (size_t)r * row_stride;
    float* grow = g + (size_t)r * row_stride;
    if (c * 4 < D) {
      const float4 gg = __ldcg(reinterpret_cast<const float4*>(grow + c * 4));   // red.add of every rank landed here
      float4 m = *reinterpret_cast<float4*>(st + o_m + c * 4), v = *reinterpret_cast<float4*>(st + o_v + c * 4);
      float4 p = *reinterpret_cast<float4*>(prow + c * 4);
      adam_functor4(p, gg, m, v, lr_t, omb1, omb2, eps);
      *reinterpret_cast<float4*>(prow + c * 4) = p;
      *reinterpret_cast<float4*>(st + o_m + c * 4) = m;
      *reinterpret_cast<float4*>(st + o_v + c * 4) = v;
      *reinterpret_cast<float4*>(grow + c * 4) = f4_zero();
    }
    if (c == 0) {
      if (has_lin) {
        float* wp = lin_at(w, prow, r, D, lin_in_row, lin_off);
        float* gp = lin_at(g, grow, r, D, lin_in_row, lin_off);
        float p = *wp, m = st[o_s + 1], v = st[o_s + 2];
        adam_functor(p, __ldcg(gp), m, v, lr_t, omb1, omb2, eps);
        *wp = p; st[o_s + 1] = m; st[o_s + 2] = v;
        *gp = 0.f;
      }
      st[o_s + 3] = __int_as_float(0);
      st[o_s + 4] = __int_as_float(t_now);
    }
  }
}

}  // namespace dr

using namespace dr;

extern "C" int dr_embed_adam_state_stride(int D) {
  if (D < 4 || D > 128 || (D & 3)) return -1;
  return adam_state_stride(D);
}

extern "C" int dr_embed_adam_count(const void* ids, int id_bytes, int64_t B, int S, int D, const int64_t* rows,
                                   const int64_t* slot_offsets, float* state, void* stream) {
  DR_REQUIRE(B >= 0 && S >= 1 && S <= 4096, DR_EINVAL, "dr_embed_adam_count: B=%lld S=%d", (long long)B, S);
  DR_REQUIRE(D >= 4 && D <= 128 && D % 4 == 0, DR_EINVAL, "dr_embed_adam_count: D=%d unsupported", D);
  DR_REQUIRE(id_bytes == 8 || id_bytes == 4, DR_EINVAL, "dr_embed_adam_count: id_bytes=%d (need 4 or 8)", id_bytes);
  if (B == 0) return DR_OK;
  DR_REQUIRE(ids && rows && slot_offsets && state, DR_EINVAL, "dr_embed_adam_count: null pointer");
  const int64_t n = B * S;
  const int64_t ctas = capped_grid(n, 256, 16);
  return with_id_type(id_bytes, [&](auto id) {
    using IdT = decltype(id);
    embed_adam_count_kernel<IdT><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(
        (const IdT*)ids, n, S, rows, slot_offsets, state, adam_state_stride(D), 3 * D + 3);
    DR_CUDA_LAUNCH_CHECK("dr_embed_adam_count");
    return DR_OK;
  });
}

static int embed_fm_bwd_adam_impl(const char* fn, const void* ids, int id_bytes, const int64_t* rows,
                                  const int64_t* slot_offsets, const float* stack, const float* sum_e,
                                  const float* g_logit, const float* g_stack, int64_t B, int S, int D,
                                  int64_t row_stride, int64_t lin_stride, int flags, float* const* table_ptrs,
                                  float* const* lin_ptrs, float* state, float* g_bias, const float* lr_t_dev, float beta1,
                                  float beta2, float eps, const int64_t* step_dev, const float* lr_hist, int hist_len,
                                  float lr, void* stream) {
  DR_REQUIRE(B >= 0 && S >= 1 && S <= 4096, DR_EINVAL, "%s: B=%lld S=%d", fn, (long long)B, S);
  DR_REQUIRE(D >= 4 && D <= 128 && D % 4 == 0, DR_EINVAL, "%s: D=%d unsupported", fn, D);
  DR_REQUIRE(id_bytes == 8 || id_bytes == 4, DR_EINVAL, "%s: id_bytes=%d (need 4 or 8)", fn, id_bytes);
  if (B == 0) return DR_OK;
  DR_REQUIRE(ids && rows && slot_offsets && table_ptrs && state && lr_t_dev, DR_EINVAL, "%s: null pointer", fn);
  DR_REQUIRE(g_logit || g_stack, DR_EINVAL, "%s: both g_logit and g_stack are NULL", fn);
  DR_REQUIRE(!g_logit || stack, DR_EINVAL, "%s: g_logit given but stack is NULL", fn);
  DR_REQUIRE((!stack || aligned16(stack)) && (!g_stack || aligned16(g_stack)) && (!sum_e || aligned16(sum_e)) &&
                 aligned16(state),
             DR_EALIGN, "%s: stack / g_stack / sum_e / state not 16-B aligned", fn);
  if (row_stride == 0) row_stride = D;
  if (lin_stride == 0) lin_stride = 1;
  const int lin_in_row = (flags & DR_EMBED_LIN_IN_ROW) ? 1 : 0;
  DR_REQUIRE(row_stride >= D + (lin_in_row ? 4 : 0) && row_stride % 4 == 0 && lin_stride >= 1, DR_EINVAL,
             "%s: bad strides row=%lld lin=%lld", fn, (long long)row_stride, (long long)lin_stride);
  if (int rc = check_adam_hparams(fn, beta1, beta2, eps)) return rc;
  const bool exact = step_dev != nullptr;
  AdamBwdParams p{};
  p.ids = ids; p.rows = rows; p.slot_offsets = slot_offsets; p.stack = stack; p.sum_e = sum_e; p.g_logit = g_logit;
  p.g_stack = g_stack; p.B = B; p.S = S; p.D = D; p.table_ptrs = table_ptrs; p.lin_ptrs = lin_in_row ? nullptr : lin_ptrs;
  p.row_stride = row_stride; p.lin_stride = lin_stride; p.lin_in_row = lin_in_row; p.state = state;
  p.SS = adam_state_stride(D); p.g_bias = g_bias; p.lr_t_dev = lr_t_dev;
  p.omb1 = 1.f - beta1; p.omb2 = 1.f - beta2; p.eps = eps;
  p.step_dev = step_dev; p.hist = AdamHist{lr_hist, hist_len, lr, beta1, beta2};
  const int threads = 256, warps = threads / 32;
  const size_t smem = (size_t)S * (sizeof(void*) * 2 + sizeof(int64_t) * 2);
  const int64_t ctas = capped_grid(B, warps, 8);
  cudaStream_t st = (cudaStream_t)stream;
  return with_lpr_id(lanes_per_row(D / 4), id_bytes, [&](auto L, auto id) {
    using IdT = decltype(id);
    if (exact) embed_fm_bwd_adam_kernel<L, IdT, true><<<(unsigned)ctas, threads, smem, st>>>(p);
    else embed_fm_bwd_adam_kernel<L, IdT, false><<<(unsigned)ctas, threads, smem, st>>>(p);
    DR_CUDA_LAUNCH_CHECK(fn);
    return DR_OK;
  });
}

extern "C" int dr_embed_fm_bwd_adam(const void* ids, int id_bytes, const int64_t* rows, const int64_t* slot_offsets,
                                    const float* stack, const float* sum_e, const float* g_logit, const float* g_stack,
                                    int64_t B, int S, int D, int64_t row_stride, int64_t lin_stride, int flags,
                                    float* const* table_ptrs, float* const* lin_ptrs, float* state, float* g_bias,
                                    const float* lr_t_dev, float beta1, float beta2, float eps, void* stream) {
  return embed_fm_bwd_adam_impl("dr_embed_fm_bwd_adam", ids, id_bytes, rows, slot_offsets, stack, sum_e, g_logit, g_stack, B,
                                S, D, row_stride, lin_stride, flags, table_ptrs, lin_ptrs, state, g_bias, lr_t_dev, beta1,
                                beta2, eps, nullptr, nullptr, 0, 0.f, stream);
}

extern "C" int dr_embed_fm_bwd_adam_tf(const void* ids, int id_bytes, const int64_t* rows, const int64_t* slot_offsets,
                                       const float* stack, const float* sum_e, const float* g_logit, const float* g_stack,
                                       int64_t B, int S, int D, int64_t row_stride, int64_t lin_stride, int flags,
                                       float* const* table_ptrs, float* const* lin_ptrs, float* state, float* g_bias,
                                       const int64_t* step_dev, const float* lr_t_dev, const float* lr_hist, int hist_len,
                                       float lr, float beta1, float beta2, float eps, void* stream) {
  DR_REQUIRE(step_dev, DR_EINVAL, "dr_embed_fm_bwd_adam_tf: step_dev is NULL");
  DR_REQUIRE(hist_len >= 0 && (hist_len == 0 || lr_hist), DR_EINVAL, "dr_embed_fm_bwd_adam_tf: bad lr history");
  return embed_fm_bwd_adam_impl("dr_embed_fm_bwd_adam_tf", ids, id_bytes, rows, slot_offsets, stack, sum_e, g_logit, g_stack,
                                B, S, D, row_stride, lin_stride, flags, table_ptrs, lin_ptrs, state, g_bias, lr_t_dev, beta1,
                                beta2, eps, step_dev, lr_hist, hist_len, lr, stream);
}

extern "C" int dr_adam_advance_hist(int64_t* step_dev, float lr, float beta1, float beta2, float* lr_t_dev,
                                    float* lr_hist, int hist_len, void* stream) {
  DR_REQUIRE(step_dev && lr_t_dev, DR_EINVAL, "dr_adam_advance_hist: null pointer");
  if (int rc = check_adam_hparams("dr_adam_advance_hist", beta1, beta2, 0.f)) return rc;
  DR_REQUIRE(hist_len >= 0, DR_EINVAL, "dr_adam_advance_hist: hist_len=%d out of range", hist_len);
  adam_advance_hist_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(step_dev, lr, beta1, beta2, lr_t_dev, lr_hist, hist_len);
  DR_CUDA_LAUNCH_CHECK("dr_adam_advance_hist");
  return DR_OK;
}


extern "C" int dr_embed_adam_prepare(const void* ids, int id_bytes, int64_t B, int S, int D, const int64_t* rows,
                                     const int64_t* slot_offsets, int64_t row_stride, int64_t lin_stride, int flags,
                                     float* const* table_ptrs, float* const* lin_ptrs, float* state,
                                     const int64_t* step_dev, const float* lr_hist, int hist_len, float lr, float beta1,
                                     float beta2, float eps, void* stream) {
  DR_REQUIRE(B >= 0 && S >= 1 && S <= 4096, DR_EINVAL, "dr_embed_adam_prepare: B=%lld S=%d", (long long)B, S);
  DR_REQUIRE(D >= 4 && D <= 128 && D % 4 == 0, DR_EINVAL, "dr_embed_adam_prepare: D=%d unsupported", D);
  DR_REQUIRE(id_bytes == 8 || id_bytes == 4, DR_EINVAL, "dr_embed_adam_prepare: id_bytes=%d (need 4 or 8)", id_bytes);
  if (B == 0) return DR_OK;
  DR_REQUIRE(ids && rows && slot_offsets && table_ptrs && state && step_dev, DR_EINVAL, "dr_embed_adam_prepare: null pointer");
  if (row_stride == 0) row_stride = D;
  if (lin_stride == 0) lin_stride = 1;
  const int lin_in_row = (flags & DR_EMBED_LIN_IN_ROW) ? 1 : 0;
  const AdamHist h{lr_hist, hist_len, lr, beta1, beta2};
  const int lpr = lanes_per_row(D / 4);
  const int64_t n = B * S;
  const int64_t ctas = capped_grid(n * lpr, 256, 16);
  return with_lpr_id(lpr, id_bytes, [&](auto L, auto id) {
    using IdT = decltype(id);
    embed_adam_prepare_kernel<L, IdT><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(
        (const IdT*)ids, n, S, D, rows, slot_offsets, table_ptrs, lin_in_row ? nullptr : lin_ptrs, row_stride, lin_stride,
        lin_in_row, state, adam_state_stride(D), step_dev, h, 1.f - beta1, 1.f - beta2, eps);
    DR_CUDA_LAUNCH_CHECK("dr_embed_adam_prepare");
    return DR_OK;
  });
}

extern "C" int dr_embed_adam_flush(const int64_t* rows, const int64_t* slot_offsets, int S, int D, int64_t total_rows,
                                   int64_t row_stride, int64_t lin_stride, int flags, float* const* table_ptrs,
                                   float* const* lin_ptrs, float* state, const int64_t* step_dev, const float* lr_hist,
                                   int hist_len, float lr, float beta1, float beta2, float eps, void* stream) {
  DR_REQUIRE(rows && slot_offsets && table_ptrs && state && step_dev, DR_EINVAL, "dr_embed_adam_flush: null pointer");
  DR_REQUIRE(S >= 1 && S <= 4096 && D >= 4 && D <= 128 && D % 4 == 0 && total_rows >= 0, DR_EINVAL,
             "dr_embed_adam_flush: S=%d D=%d total_rows=%lld", S, D, (long long)total_rows);
  if (total_rows == 0) return DR_OK;
  if (row_stride == 0) row_stride = D;
  if (lin_stride == 0) lin_stride = 1;
  const int lin_in_row = (flags & DR_EMBED_LIN_IN_ROW) ? 1 : 0;
  const AdamHist h{lr_hist, hist_len, lr, beta1, beta2};
  const int lpr = lanes_per_row(D / 4);
  const int64_t ctas = capped_grid(total_rows * lpr, 256, 16);
  return with_lpr(lpr, [&](auto L) {
    embed_adam_flush_kernel<L><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(
        table_ptrs, lin_in_row ? nullptr : lin_ptrs, rows, slot_offsets, S, D, row_stride, lin_stride, lin_in_row, state,
        adam_state_stride(D), total_rows, step_dev, h, 1.f - beta1, 1.f - beta2, eps);
    DR_CUDA_LAUNCH_CHECK("dr_embed_adam_flush");
    return DR_OK;
  });
}

// ---- tf.keras Adam of the layer API (see embed_adam_catch_up_kernel) --------------------------------------------------
static int adam_rows_layout_check(const char* fn, int D, int64_t& row_stride, int64_t& lin_stride, int flags,
                                  float* const* lin_ptrs, int& lin_in_row) {
  DR_REQUIRE(D >= 4 && D <= 128 && D % 4 == 0, DR_EINVAL, "%s: D=%d unsupported", fn, D);
  DR_REQUIRE(flags == (flags & DR_EMBED_LIN_IN_ROW), DR_EINVAL, "%s: flags=%d (only DR_EMBED_LIN_IN_ROW)", fn, flags);
  if (row_stride == 0) row_stride = D;
  if (lin_stride == 0) lin_stride = 1;
  lin_in_row = (flags & DR_EMBED_LIN_IN_ROW) ? 1 : 0;
  DR_REQUIRE(row_stride >= D + (lin_in_row ? 4 : 0) && row_stride % 4 == 0 && lin_stride >= 1, DR_EINVAL,
             "%s: bad strides row=%lld lin=%lld for D=%d", fn, (long long)row_stride, (long long)lin_stride, D);
  DR_REQUIRE(!(lin_in_row && lin_ptrs), DR_EINVAL, "%s: lin_ptrs given with DR_EMBED_LIN_IN_ROW", fn);
  return DR_OK;
}

extern "C" int dr_embed_adam_catch_up(const void* ids, int id_bytes, int64_t n, int S, int D, const int64_t* rows,
                                      const int64_t* slot_offsets, int64_t row_stride, int64_t lin_stride, int flags,
                                      float* const* table_ptrs, float* const* lin_ptrs, float* state,
                                      const int64_t* step_dev, const float* lr_hist, int hist_len, float lr,
                                      float beta1, float beta2, float eps, void* stream) {
  const char* fn = "dr_embed_adam_catch_up";
  DR_REQUIRE(n >= 0 && S >= 1 && S <= 4096 && n % S == 0, DR_EINVAL, "%s: n=%lld S=%d", fn, (long long)n, S);
  DR_REQUIRE(id_bytes == 8 || id_bytes == 4, DR_EINVAL, "%s: id_bytes=%d (need 4 or 8)", fn, id_bytes);
  int lin_in_row = 0;
  if (int rc = adam_rows_layout_check(fn, D, row_stride, lin_stride, flags, lin_ptrs, lin_in_row)) return rc;
  DR_REQUIRE(hist_len >= 0 && (hist_len == 0 || lr_hist), DR_EINVAL, "%s: bad lr history", fn);
  if (int rc = check_adam_hparams(fn, beta1, beta2, eps)) return rc;
  if (n == 0) return DR_OK;
  DR_REQUIRE(ids && rows && slot_offsets && table_ptrs && state && step_dev, DR_EINVAL, "%s: null pointer", fn);
  DR_REQUIRE(aligned16(state), DR_EALIGN, "%s: state not 16-B aligned", fn);
  const AdamHist h{lr_hist, hist_len, lr, beta1, beta2};
  const int lpr = lanes_per_row(D / 4);
  const int64_t ctas = capped_grid(n * lpr, 256, 16);
  return with_lpr_id(lpr, id_bytes, [&](auto L, auto id) {
    using IdT = decltype(id);
    embed_adam_catch_up_kernel<L, IdT><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(
        (const IdT*)ids, n, S, D, rows, slot_offsets, table_ptrs, lin_ptrs, row_stride, lin_stride, lin_in_row, state,
        adam_state_stride(D), step_dev, h, 1.f - beta1, 1.f - beta2, eps);
    DR_CUDA_LAUNCH_CHECK(fn);
    return DR_OK;
  });
}

extern "C" int dr_embed_adam_rows_tf(const void* ids, int id_bytes, int64_t n, int64_t B, int S,
                                     const int64_t* row_splits, const int64_t* rows, const int64_t* slot_offsets,
                                     const float* g_emb, int64_t g_ld, int64_t g_slot, const float* g_lin,
                                     int64_t gl_ld, int64_t gl_slot, int D, int64_t row_stride, int64_t lin_stride,
                                     int flags, float* const* table_ptrs, float* const* lin_ptrs, float* state,
                                     const int64_t* step_dev, const float* lr_t_dev, const float* lr_hist, int hist_len,
                                     float lr, float beta1, float beta2, float eps, void* stream) {
  const char* fn = "dr_embed_adam_rows_tf";
  DR_REQUIRE(n >= 0 && B >= 0 && S >= 1 && S <= 4096, DR_EINVAL, "%s: n=%lld B=%lld S=%d", fn, (long long)n,
             (long long)B, S);
  DR_REQUIRE(row_splits ? S == 1 : n == B * S, DR_EINVAL, "%s: %s", fn,
             row_splits ? "bags (row_splits) need S = 1" : "n != B * S");
  DR_REQUIRE(id_bytes == 8 || id_bytes == 4, DR_EINVAL, "%s: id_bytes=%d (need 4 or 8)", fn, id_bytes);
  int lin_in_row = 0;
  if (int rc = adam_rows_layout_check(fn, D, row_stride, lin_stride, flags, lin_ptrs, lin_in_row)) return rc;
  DR_REQUIRE(!g_lin == !(lin_in_row || lin_ptrs), DR_EINVAL,
             "%s: g_lin and the first-order weights (lin_ptrs or DR_EMBED_LIN_IN_ROW) come together", fn);
  // a stride of 0 broadcasts one row (a zero gradient for a term the forward did not use)
  DR_REQUIRE(g_ld >= 0 && g_slot >= 0 && g_ld % 4 == 0 && g_slot % 4 == 0 && (B <= 1 || g_ld == 0 || g_ld >= D) &&
                 (S == 1 || g_slot == 0 || g_slot >= D) && (!g_lin || (gl_ld >= 0 && gl_slot >= 0)),
             DR_EINVAL, "%s: bad gradient strides g_ld=%lld g_slot=%lld gl_ld=%lld gl_slot=%lld for D=%d", fn,
             (long long)g_ld, (long long)g_slot, (long long)gl_ld, (long long)gl_slot, D);
  DR_REQUIRE(hist_len >= 0 && (hist_len == 0 || lr_hist), DR_EINVAL, "%s: bad lr history", fn);
  if (int rc = check_adam_hparams(fn, beta1, beta2, eps)) return rc;
  if (n == 0) return DR_OK;
  DR_REQUIRE(ids && rows && slot_offsets && g_emb && table_ptrs && state && step_dev && lr_t_dev && (!row_splits || B >= 1),
             DR_EINVAL, "%s: null pointer", fn);
  DR_REQUIRE(aligned16(g_emb) && aligned16(state), DR_EALIGN, "%s: g_emb / state not 16-B aligned", fn);
  AdamRowsParams p{};
  p.ids = ids; p.row_splits = row_splits; p.n = n; p.B = B; p.S = S; p.D = D; p.rows = rows;
  p.slot_offsets = slot_offsets; p.g_emb = g_emb; p.g_ld = g_ld; p.g_slot = g_slot; p.g_lin = g_lin; p.gl_ld = gl_ld;
  p.gl_slot = gl_slot; p.table_ptrs = table_ptrs; p.lin_ptrs = lin_ptrs; p.row_stride = row_stride;
  p.lin_stride = lin_stride; p.lin_in_row = lin_in_row; p.state = state; p.SS = adam_state_stride(D);
  p.step_dev = step_dev; p.lr_t_dev = lr_t_dev; p.hist = AdamHist{lr_hist, hist_len, lr, beta1, beta2};
  p.omb1 = 1.f - beta1; p.omb2 = 1.f - beta2; p.eps = eps;
  const int lpr = lanes_per_row(D / 4);
  const int64_t ctas = capped_grid(n * lpr, 256, 16);
  cudaStream_t st = (cudaStream_t)stream;
  return with_lpr_id(lpr, id_bytes, [&](auto L, auto id) {
    using IdT = decltype(id);
    if (row_splits) embed_adam_rows_tf_kernel<L, IdT, true><<<(unsigned)ctas, 256, 0, st>>>(p);
    else embed_adam_rows_tf_kernel<L, IdT, false><<<(unsigned)ctas, 256, 0, st>>>(p);
    DR_CUDA_LAUNCH_CHECK(fn);
    return DR_OK;
  });
}

// ---- row-sharded tf.keras Adam (see shard_adam_mark_kernel) -----------------------------------------------------------
extern "C" int dr_shard_adam_mark(const void* ids, int id_bytes, int64_t n, int S, const int64_t* slot_offsets,
                                  const int64_t* rows, int world, int32_t* const* touch_bases, const int64_t* step_dev,
                                  void* stream) {
  DR_REQUIRE(n >= 0 && S >= 1 && S <= 4096, DR_EINVAL, "dr_shard_adam_mark: n=%lld S=%d", (long long)n, S);
  DR_REQUIRE(id_bytes == 8 || id_bytes == 4, DR_EINVAL, "dr_shard_adam_mark: id_bytes=%d (need 4 or 8)", id_bytes);
  DR_REQUIRE(world >= 1 && world <= kMaxShardWorld, DR_EINVAL, "dr_shard_adam_mark: world=%d outside [1,%d]", world,
             kMaxShardWorld);
  DR_REQUIRE(ids && slot_offsets && rows && touch_bases && step_dev, DR_EINVAL, "dr_shard_adam_mark: null pointer");
  if (n == 0) return DR_OK;
  const int64_t ctas = capped_grid(n, 256, 16);
  return with_id_type(id_bytes, [&](auto id) {
    using IdT = decltype(id);
    shard_adam_mark_kernel<IdT><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>((const IdT*)ids, n, S, slot_offsets,
                                                                                 rows, world, touch_bases, step_dev);
    DR_CUDA_LAUNCH_CHECK("dr_shard_adam_mark");
    return DR_OK;
  });
}

static int shard_adam_layout_check(const char* fn, int64_t local_rows, int D, int64_t row_stride, int64_t lin_offset,
                                   int flags) {
  DR_REQUIRE(local_rows >= 0 && local_rows < ((int64_t)1 << 31), DR_EINVAL, "%s: local_rows=%lld", fn,
             (long long)local_rows);
  DR_REQUIRE(D >= 4 && D <= 128 && D % 4 == 0, DR_EINVAL, "%s: D=%d unsupported", fn, D);
  const int lin_in_row = (flags & DR_EMBED_LIN_IN_ROW) ? 1 : 0;
  DR_REQUIRE(row_stride >= D + lin_in_row && row_stride % 4 == 0, DR_EINVAL, "%s: bad row_stride=%lld for D=%d", fn,
             (long long)row_stride, D);
  DR_REQUIRE(lin_offset >= 0 && !(lin_in_row && lin_offset > 0) && (lin_offset == 0 || lin_offset >= local_rows * row_stride),
             DR_EINVAL, "%s: lin_offset=%lld (must trail the rows and be exclusive with DR_EMBED_LIN_IN_ROW)", fn,
             (long long)lin_offset);
  return DR_OK;
}

extern "C" int dr_shard_adam_prepare(int32_t* touch, int64_t local_rows, int32_t* list, int32_t* count, int D,
                                     int64_t row_stride, int64_t lin_offset, int flags, float* shard, float* state,
                                     const int64_t* step_dev, const float* lr_hist, int hist_len, float lr, float beta1,
                                     float beta2, float eps, void* stream) {
  const char* fn = "dr_shard_adam_prepare";
  if (int rc = shard_adam_layout_check(fn, local_rows, D, row_stride, lin_offset, flags)) return rc;
  DR_REQUIRE(touch && list && count && shard && state && step_dev, DR_EINVAL, "%s: null pointer", fn);
  DR_REQUIRE(hist_len >= 0 && (hist_len == 0 || lr_hist), DR_EINVAL, "%s: bad lr history", fn);
  if (int rc = check_adam_hparams(fn, beta1, beta2, eps)) return rc;
  DR_REQUIRE(aligned16(shard) && aligned16(state), DR_EALIGN, "%s: shard / state not 16-B aligned", fn);
  cudaStream_t st = (cudaStream_t)stream;
  DR_CUDA_CALL(cudaMemsetAsync(count, 0, sizeof(int32_t), st));
  if (local_rows == 0) return DR_OK;
  const int lin_in_row = (flags & DR_EMBED_LIN_IN_ROW) ? 1 : 0;
  const AdamHist h{lr_hist, hist_len, lr, beta1, beta2};
  const int64_t ctas = capped_grid(local_rows, 256, 16);
  return with_lpr(lanes_per_row(D / 4), [&](auto L) {
    shard_adam_prepare_kernel<L><<<(unsigned)ctas, 256, 0, st>>>(touch, local_rows, list, count, shard, row_stride,
                                                                 lin_offset, lin_in_row, state, adam_state_stride(D), D,
                                                                 step_dev, h, 1.f - beta1, 1.f - beta2, eps);
    DR_CUDA_LAUNCH_CHECK(fn);
    return DR_OK;
  });
}

extern "C" int dr_shard_adam_apply(const int32_t* list, const int32_t* count, int64_t local_rows, int D,
                                   int64_t row_stride, int64_t lin_offset, int flags, float* shard, float* grad,
                                   float* state, const int64_t* step_dev, const float* lr_t_dev, float beta1, float beta2,
                                   float eps, void* stream) {
  const char* fn = "dr_shard_adam_apply";
  if (int rc = shard_adam_layout_check(fn, local_rows, D, row_stride, lin_offset, flags)) return rc;
  DR_REQUIRE(list && count && shard && grad && state && step_dev && lr_t_dev, DR_EINVAL, "%s: null pointer", fn);
  if (int rc = check_adam_hparams(fn, beta1, beta2, eps)) return rc;
  DR_REQUIRE(aligned16(shard) && aligned16(grad) && aligned16(state), DR_EALIGN,
             "%s: shard / grad / state not 16-B aligned", fn);
  if (local_rows == 0) return DR_OK;
  const int lin_in_row = (flags & DR_EMBED_LIN_IN_ROW) ? 1 : 0;
  const int lpr = lanes_per_row(D / 4);
  const int64_t ctas = capped_grid(local_rows * lpr, 256, 16);
  return with_lpr(lpr, [&](auto L) {
    shard_adam_apply_kernel<L><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(
        list, count, shard, grad, row_stride, lin_offset, lin_in_row, state, adam_state_stride(D), D, step_dev, lr_t_dev,
        1.f - beta1, 1.f - beta2, eps);
    DR_CUDA_LAUNCH_CHECK(fn);
    return DR_OK;
  });
}
