/*
 * deeprec_b200.h -- C-ABI of the CUDA-native (H100, sm_90a) hot path of deep_recommenders.
 *
 * One shared library (libdeeprec_b200.so), extern "C", plain pointers and sizes,
 * no torch / C++ types.  The reference (LongmaoTeamTf/deep_recommenders) has no FFI at
 * all: its "operator API" is the tf.keras Layer protocol and every op below is what a
 * TensorFlow custom op for that layer's call()/gradient would bind.  Each entry cites the
 * reference lines it replaces (paths relative to the reference repo root).
 *
 * Conventions (all entries):
 *   - return 0 on success; <0 = argument rejected on the host BEFORE any launch
 *     (DR_EINVAL ...); >0 = cudaError_t passed through.  dr_last_error() returns a
 *     thread-local, human-readable message for the last non-zero return.
 *   - every pointer is a DEVICE pointer owned by the caller (outputs and workspaces
 *     included) unless the comment says "host".  The library allocates nothing.
 *   - every compute entry takes the cudaStream_t to enqueue on (passed as void*), never
 *     synchronises, never touches the default stream, keeps no global mutable state.
 *   - tensors are row-major contiguous fp32; ids are int64 (id_bytes=8) or int32 (4).
 *   - an id outside [0, rows) (TensorFlow's OOV id -1 included) contributes a zero row
 *     and is never dereferenced.
 */
#ifndef DEEPREC_B200_H_
#define DEEPREC_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DR_OK 0
#define DR_EINVAL (-1)     /* null pointer / bad size / unsupported D            */
#define DR_EALIGN (-2)     /* a row base or tensor base is not 16-byte aligned   */
#define DR_ENOTSUP (-3)    /* valid request this build does not implement        */

/* dr_embed_fm_* flags */
#define DR_EMBED_LIN_IN_ROW 1   /* first-order weight of an id is stored IN its row, at float index D
                                   (row_stride >= D+4): it is fetched by the same 128-bit request as the
                                   embedding chunks; lin_ptrs / lin_stride are ignored                  */
#define DR_EMBED_NO_FM 2        /* dr_embed_fm_fwd / _bwd only: no FM second-order term.  Forward: out_logit =
                                   bias + sum_s lin_s[id_s] (xDeepFM's linear unit).  Backward: dE = g_stack;
                                   g_logit still reaches grad_lin and g_bias.  The sharded entries return
                                   DR_ENOTSUP for it; dr_embed_fm_fwd_tma takes no flags.                  */

/* activation codes (tf.keras.layers.Dense(activation=...)) */
/* combiner of a multi-valued slot (tf.feature_column.embedding_column(combiner=...)) */
#define DR_COMBINER_SUM 0
#define DR_COMBINER_MEAN 1
#define DR_COMBINER_SQRTN 2

#define DR_ACT_NONE 0
#define DR_ACT_RELU 1
#define DR_ACT_SIGMOID 2
#define DR_ACT_TANH 3
#define DR_ACT_SOFTMAX 4   /* dr_spmm_csr_fwd only: softmax over the output row */

/* ABI version (major*10000 + minor*100 + patch) and last error string. */
int dr_version(void);
const char* dr_last_error(void);
/* Number of kernels this library has launched since load (process-wide, for bench.py). */
uint64_t dr_launch_count(void);

/* ---------------------------------------------------------------------------------------
 * Row E + L + F fused: multi-slot embedding gather + first-order term + FM second order.
 *   replaces: keras/models/ranking/fm.py:23-37,54-63 ; deepfm.py:36-46 (DenseFeatures per
 *             column -> tf.stack -> FM.call) ; estimator/models/feature_interaction/
 *             fm.py:10-26,41-56.
 *   table_ptrs[S] : device array of S device pointers, table s is [rows[s], D] fp32 with
 *                   row_stride floats between rows (0 = D; >= D, multiple of 4), every row
 *                   base 16-B aligned.  D % 4 == 0, 4 <= D <= 128.
 *   lin_ptrs[S]   : device array of S device pointers to the first-order weights, weight of
 *                   id i at lin_ptrs[s][i * lin_stride] (0 = 1); NULL = no first-order term.
 *                   The strides let the host co-locate a row's first-order weight with its
 *                   embedding vector (row = [D floats | w | pad]) so one DRAM page serves both.
 *   rows[S]       : device int64.
 *   ids           : [B, S] int64 / int32 (id_bytes).
 *   bias          : device [1] or NULL.
 *   out_stack     : [B, S, D] (== the [B, S*D] concat) or NULL (FM-only, no stack write).
 *   out_sum       : [B, D] sum over slots (saved for backward) or NULL.
 *   out_logit     : [B] = bias + sum_s lin_s[id_s] + 0.5*sum_d((sum_s e)^2 - sum_s e^2),
 *                   or NULL (pure multi-slot gather).
 * ------------------------------------------------------------------------------------- */
int dr_embed_fm_fwd(const float* const* table_ptrs, const float* const* lin_ptrs,
                    const int64_t* rows, const void* ids, int id_bytes, const float* bias,
                    int64_t B, int S, int D, int64_t row_stride, int64_t lin_stride, int flags,
                    float* out_stack, float* out_sum, float* out_logit, void* stream);

/* Backward of the above fused with the sparse update ("IndexedSlices" scatter-add):
 *   dE[b,s,:] = g_logit[b] * (sum_e[b,:] - stack[b,s,:]) + g_stack[b,s,:]
 *   grad_table s [id] += scale * dE      (vector red.global.add, warp-aggregated)
 *   grad_lin   s [id] += scale * g_logit[b]
 *   g_bias[0]         += scale * sum_b g_logit[b]
 * scale = 1 with zeroed grad buffers gives the dense gradient TF autodiff would produce;
 * scale = -lr with grad_* aliasing the parameters is a fused sparse SGD step.
 * g_logit / g_stack / grad_lin_ptrs / g_bias / sum_e may be NULL (sum_e == NULL makes the
 * kernel re-reduce the stack).  stack is required when g_logit != NULL.
 */
int dr_embed_fm_bwd(const void* ids, int id_bytes, const int64_t* rows,
                    const float* stack, const float* sum_e,
                    const float* g_logit, const float* g_stack,
                    int64_t B, int S, int D, int64_t row_stride, int64_t lin_stride, int flags,
                    float* const* grad_table_ptrs, float* const* grad_lin_ptrs, float* g_bias,
                    float scale, void* stream);

/* Opt-in variant of dr_embed_fm_fwd that stages the rows THROUGH TMA INTO SHARED MEMORY
 * (one cp.async.bulk copy per looked-up row, mbarrier completion; the stacked rows leave as one
 * cp.async.bulk store per tile).  Same outputs as dr_embed_fm_fwd (stack bit-exact; logit / sum_e up to summation order).
 * Serves the fused row layout only: all tables in ONE arena `arena` [total_rows, row_stride] with the first-order weight
 * at float D of the row (DR_EMBED_LIN_IN_ROW), D = 16, S <= 32; slot_offsets[s] = first arena row of table s.
 * Returns DR_ENOTSUP otherwise.  Shipped as the alternative to measure against, not as the default. */
int dr_embed_fm_fwd_tma(const float* arena, int64_t total_rows, const int64_t* slot_offsets,
                        const int64_t* rows, const void* ids, int id_bytes, const float* bias, int64_t B, int S,
                        int D, int64_t row_stride, float* out_stack, float* out_sum, float* out_logit,
                        void* stream);

/* Plain single-table gather / scatter-add (two-tower user & item towers).
 *   replaces: tf.keras.layers.DenseFeatures(embedding_column) on one column
 *             (keras/models/ranking/fm.py:47-51).  D % 4 == 0, 4 <= D <= 128.      */
int dr_gather_fwd(const float* table, int64_t rows, const void* ids, int id_bytes,
                  int64_t n, int D, float* out, void* stream);
int dr_scatter_add(float* grad_table, int64_t rows, const void* ids, int id_bytes,
                   int64_t n, int D, const float* g, float scale, void* stream);

/* ---------------------------------------------------------------------------------------
 * Row F standalone: FM second-order on a dense [B, S, D] tensor (any S, D >= 1).
 *   replaces: keras/models/ranking/fm.py:28-35 ; estimator/.../fm.py:22-26.
 *   out[b] = 0.5 * sum_d((sum_s x)^2 - sum_s x^2);  gx = g[b] * (sum_s x - x).
 * ------------------------------------------------------------------------------------- */
int dr_fm_fwd(const float* x, int64_t B, int S, int D, float* out, void* stream);
int dr_fm_bwd(const float* x, const float* g, int64_t B, int S, int D, float* gx, void* stream);

/* ---------------------------------------------------------------------------------------
 * Row D: Dense layer  y = act(x @ W + b),  x [M,K], W [K,N] (Keras kernel layout), b [N].
 *   replaces: tf.keras.layers.Dense in keras/models/ranking/deepfm.py:30-34, fm.py:16-20;
 *             tf.layers.dense in estimator/models/feature_interaction/dnn.py:17-29.
 *   fp32 accumulate, fp32-accurate products (no single-pass TF32/BF16).
 * backward: gz = gy * act'(y) ; gx = gz @ W^T (NULL = skip) ; gw = x^T @ gz ; gb = colsum(gz).
 *   gz_ws: [M,N] workspace (may alias gy if the caller no longer needs gy).  gw and gb
 *   are OVERWRITTEN (not accumulated).  gw == NULL skips the weight gradient; a second call with
 *   gy = gz_ws, act = DR_ACT_NONE, gx = NULL, gb = NULL then computes only gw (lets the caller run
 *   it concurrently with whatever consumes gx).
 * ------------------------------------------------------------------------------------- */
int dr_dense_fwd(const float* x, const float* w, const float* b, int64_t M, int K, int N,
                 int act, float* y, void* stream);
int dr_dense_bwd(const float* x, const float* w, const float* y, const float* gy,
                 int64_t M, int K, int N, int act,
                 float* gz_ws, float* gx, float* gw, float* gb, void* stream);
/* Same, chained through a stack of Dense layers (deepfm.py:30-34, estimator dnn.py:17-29): x of this layer is
 * act_prev(z_prev) of the layer below with output prev_y = x; gx is then written as (gz @ W^T) * act_prev'(prev_y),
 * i.e. already the PRE-activation gradient of the layer below (fused into the GEMM epilogue), so that layer's own
 * call passes act = DR_ACT_NONE with this gx as its gy.  prev_act == DR_ACT_NONE: identical to dr_dense_bwd. */
int dr_dense_bwd_chain(const float* x, const float* w, const float* y, const float* gy,
                       int64_t M, int K, int N, int act,
                       float* gz_ws, float* gx, float* gw, float* gb,
                       const float* prev_y, int prev_act, void* stream);
/* G independent Dense layers of one shape (the expert and task towers of MMoE, ESMM's two towers):
 *   replaces: the per-tower tf.layers.dense calls of estimator/models/feature_interaction/dnn.py:17-29 as called
 *             by estimator/models/multi_task_learning/mixture_of_experts.py:64-68, :86-90 and esmm.py:38-55.
 *   x [M, G*K] (group g reads column block g*K), w [G, K, N], b [G, N] (nullable), y [M, G*N] (group g writes
 *   column block g*N).  Per group exactly dr_dense_fwd / dr_dense_bwd: same activations, gz_ws [M, G*N],
 *   gx [M, G*K] (NULL = skip), gw [G, K, N] and gb [G, N] OVERWRITTEN.  One strided GEMM per group; the backward's
 *   activation-gradient + column-sum pass runs once over the whole [M, G*N] block.  G = 1: y and gx are
 *   bit-identical to dr_dense_fwd / dr_dense_bwd; gw and gb are summed with split-K / column atomics, so their last
 *   bits depend on the summation order (as in dr_dense_bwd).  Served: any G, K, N >= 1 with G*K, G*N < 2^31.  */
int dr_dense_grouped_fwd(const float* x, const float* w, const float* b, int64_t M, int G, int K, int N,
                         int act, float* y, void* stream);
int dr_dense_grouped_bwd(const float* x, const float* w, const float* y, const float* gy,
                         int64_t M, int G, int K, int N, int act,
                         float* gz_ws, float* gx, float* gw, float* gb, void* stream);

/* ---------------------------------------------------------------------------------------
 * Row X: Cross layer (DCN-v2 matrix form).
 *   replaces: keras/models/ranking/dcn.py:70-88 (call) with build() :35-68.
 *   full rank (r == 0):  u = x @ W + b + alpha*x        W [d,d]
 *   low rank  (r  > 0):  u = (x @ U) @ V + b + alpha*x  U [d,r] (no bias), V [r,d]
 *   y = x0 * u + x ;  u is saved ([B,d]) for backward.  b may be NULL (use_bias=False).
 *   xu_ws: [B,r] workspace (low rank only; saved for backward).
 * backward (g = dL/dy, h = g*x0):
 *   gx0 = g*u ; gx = h @ W^T + alpha*h + g ; gW = x^T @ h ; gb = colsum(h)
 *   (low rank: gV = (xU)^T @ h ; t = h @ V^T ; gU = x^T @ t ; gx = t @ U^T + alpha*h + g)
 *   When the caller passed the same tensor as x0 and x it adds gx0 + gx itself.
 *   h_ws [B,d], t_ws [B,r] workspaces.  gW/gU/gV/gb are OVERWRITTEN.
 * ------------------------------------------------------------------------------------- */
int dr_cross_fwd(const float* x0, const float* x, const float* w, const float* uk,
                 const float* vk, const float* b, float alpha, int64_t B, int d, int r,
                 float* xu_ws, float* u_out, float* y, void* stream);
int dr_cross_bwd(const float* x0, const float* x, const float* w, const float* uk,
                 const float* vk, float alpha, const float* u_saved, const float* xu_saved,
                 const float* g, int64_t B, int d, int r,
                 float* h_ws, float* t_ws, float* gx0, float* gx,
                 float* gw, float* guk, float* gvk, float* gb, void* stream);
/* dr_cross_bwd for a caller that builds the gradient of x0 IN PLACE across a stack of Cross layers
 *   replaces: the backward of keras/models/ranking/dcn.py:70-88 under the stacking idiom of tests/keras/test_dcn.py:27-32
 *             (x1 = Cross()(x0, x0); x2 = Cross()(x0, x1); ...), where x0 receives a gradient from EVERY layer.
 * Same operands and mathematics as dr_cross_bwd, except
 *   gx0 is ACCUMULATED: gx0 += g*u (the caller initialises it, e.g. with the deep tower's input gradient);
 *   x_is_x0 != 0 (the bottom layer: x and x0 are the same tensor, x == x0): the input gradient goes into the same
 *     buffer, gx0 += h @ W^T + alpha*h + g (low rank: t @ U^T + alpha*h + g), and gx may be NULL;
 *   x_is_x0 == 0: gx is written as by dr_cross_bwd.  gW/gU/gV/gb are OVERWRITTEN. */
int dr_cross_bwd_acc(const float* x0, const float* x, const float* w, const float* uk,
                     const float* vk, float alpha, const float* u_saved, const float* xu_saved,
                     const float* g, int64_t B, int d, int r,
                     float* h_ws, float* t_ws, float* gx0, float* gx,
                     float* gw, float* guk, float* gvk, float* gb, int x_is_x0, void* stream);

/* ---------------------------------------------------------------------------------------
 * Row C: xDeepFM's Compressed Interaction Network layer (CIN), the outer product + width-1
 * conv1d fused into one GEMM whose operand is generated on chip (the [B, D, m*h] outer
 * product never reaches global memory).
 *   replaces: keras/models/ranking/xdeepfm.py:71-96 (CIN.call).
 *   x0 [B, m, D], x [B, h, D], w = the layer's kernel [1, m*h, H] (row i*h + j pairs field i of x0
 *   with field j of x), bias [H] (nullable), y [B, H, D]:
 *     y[b,k,d] = act(sum_{i,j} w[i*h+j, k] * x0[b,i,d] * x[b,j,d] + bias[k])
 *   pooled [B, H] (nullable) receives sum_d y[b,k,d] (xDeepFM's sum pooling), written by the same
 *   kernel in a fixed order.  act: DR_ACT_*.  Served: 1 <= m, h, H <= 1024, 1 <= D <= 128,
 *   B * D < 2^31; larger shapes return DR_ENOTSUP.  B = 0 is a no-op (the batch tensors may then
 *   be NULL; dr_cin_bwd still zeroes gw and gb).  Exact fp32 FFMA.
 *
 * dr_cin_bwd: no reference lines (TensorFlow autodiff of the above).
 *   G = (gy + gpool broadcast over d) * act'(y) is formed once into g_ws [B, H, D]; gy or gpool
 *   (not both) may be NULL.  Then, overwriting (not accumulating) every output:
 *     gx0[b,i,d] = sum_{j,k} w[i*h+j,k] x[b,j,d] G[b,k,d]      gx [b,j,d] = sum_{i,k} w[i*h+j,k] x0[b,i,d] G[b,k,d]
 *     gw[i*h+j,k] = sum_{b,d} x0[b,i,d] x[b,j,d] G[b,k,d]      gb[k] = sum_{b,d} G[b,k,d]  (gb nullable)
 *   x_is_x0 = 1 (the first layer, called on (x0, x0)): x == x0, h == m, gx must be NULL and both
 *   contributions land in gx0.  gw is split over the B*D columns and gb over the rows and both are
 *   summed with floating-point atomics, so their last bits can differ from run to run; y, pooled,
 *   gx0 and gx are deterministic.                                                          */
int dr_cin_fwd(const float* x0, const float* x, const float* w, const float* bias, int64_t B,
               int m, int h, int D, int H, int act, float* y, float* pooled, void* stream);
int dr_cin_bwd(const float* x0, const float* x, const float* w, const float* y, const float* gy,
               const float* gpool, int64_t B, int m, int h, int D, int H, int act, int x_is_x0,
               float* g_ws, float* gx0, float* gx, float* gw, float* gb, void* stream);

/* ---------------------------------------------------------------------------------------
 * Row A: DIN's activation unit as target attention over a behaviour sequence, fused with the
 * pooling (the [B*T, 3D] unit input and the [B*T, U] hidden activations never reach global memory).
 *   replaces: keras/models/ranking/din.py:59-71 (ActivationUnit.call) applied at every position
 *             of a sequence, plus DIN's weighted sum pooling (Zhou et al., KDD 2018).
 *   keys [B, T, D] (dense rows, e.g. from dr_gather_fwd), query [B, D], w1 = the hidden Dense
 *   kernel [(2|3)*D, U] whose row blocks multiply [k | q | f(k, q)], b1 [U] (nullable), w2 = the
 *   Dense(1) kernel [U], b2 [1] (nullable):
 *     f = none (interact DR_DIN_INTERACT_NONE, w1 has 2D rows), k - q (SUB) or k * q (MUL)
 *     score[b,t] = act([k | q | f] . w1 + b1) . w2 + b2          act: DR_ACT_*
 *     pooled[b,:] = sum_t score[b,t] * keys[b,t,:]               (unnormalised: no softmax)
 *   score and pooled are both nullable (not both); they are written, never accumulated, by one
 *   kernel in a fixed order (bit-identical from run to run).  Served: 1 <= D <= 128, 1 <= U <= 256,
 *   T >= 1, B*T < 2^31; larger D or U return DR_ENOTSUP.  B = 0 is a no-op.  Exact fp32 FFMA.
 *   Padding: a history padded with id -1 gathers a zero key row, which adds nothing to pooled and
 *   gets no gradient through the score; dr_scatter_add drops its g_keys row.
 *
 * dr_din_attn_bwd: no reference lines (TensorFlow autodiff of the above).  g_pooled [B, D] and
 *   g_score [B, T] are nullable (not both).  h is recomputed per tile, not saved.  Writes
 *   g_keys [B, T, D] and g_query [B, D] (each element has one owner: deterministic) and
 *   gw1, gb1, gw2, gb2, which are split across CTAs and summed with floating-point atomics, so
 *   their last bits can differ from run to run.  gb1 / gb2 are given exactly when b1 / b2 are.
 *   B = 0 still zeroes the weight gradients.                                                  */
#define DR_DIN_INTERACT_NONE 0
#define DR_DIN_INTERACT_SUB 1
#define DR_DIN_INTERACT_MUL 2
int dr_din_attn_fwd(const float* keys, const float* query, const float* w1, const float* b1,
                    const float* w2, const float* b2, int64_t B, int T, int D, int U, int interact,
                    int act, float* score, float* pooled, void* stream);
int dr_din_attn_bwd(const float* keys, const float* query, const float* w1, const float* b1,
                    const float* w2, const float* b2, const float* g_pooled, const float* g_score,
                    int64_t B, int T, int D, int U, int interact, int act, float* g_keys,
                    float* g_query, float* gw1, float* gb1, float* gw2, float* gb2, void* stream);

/* Dice activation on a rank-2 input x [N, U].
 *   replaces: keras/models/ranking/din.py:110-121 (Dice.call).  Per row: mu = mean,
 *   sigma = population std (reduce_std), p = sigmoid((x - mu) / sqrt(sigma + eps)) (the square
 *   root of the std, as the reference computes it), a = PReLU(x) with alpha [U],
 *   y = a > 0 ? p*a : (1 - p)*a (the branch tests the PReLU output, not x).  One warp per row.
 * dr_dice_bwd: gx [N, U] through PReLU, p, mu and sigma, galpha [U] (column sums, overwritten,
 *   summed with floating-point atomics).  Deviation: for a constant row (sigma = 0, every row
 *   when U = 1) the gradient through sigma is 0, where TensorFlow's autodiff gives NaN.
 *   dr_dice_bwd serves U <= 8192 (DR_ENOTSUP above).                                          */
int dr_dice_fwd(const float* x, const float* alpha, int64_t N, int U, float eps, float* y,
                void* stream);
int dr_dice_bwd(const float* x, const float* alpha, const float* gy, int64_t N, int U, float eps,
                float* gx, float* galpha, void* stream);

/* ---------------------------------------------------------------------------------------
 * Row T: multi-head scaled dot-product attention, fused (the [H*B, Lq, Lk] score matrix never
 * reaches global memory: keys stream through shared memory with an online softmax).
 *   replaces: keras/models/nlp/multi_head_attention.py:72-84 (ScaledDotProductAttention.call),
 *             :45-58 (mask, future_mask) and :134-147 (MultiHeadAttention's head split / merge).
 *   q [B, Lq, H*dh], k and v [B, Lk, H*dh], out [B, Lq, H*dh]: head h is the column block
 *   h*dh .. (h+1)*dh, so split / concat are strides.  Logical row r = h*B + b (head-major, as the
 *   reference's concat(split(x, H, axis=2), axis=0)).  The standalone layer is H = 1.
 *     s   = (q . k) / fl32(sqrt(dh))                         (a division, as TF does)
 *     s   = s + mask[r % Bm, j] * C      C = fl32(-2^32+1) = -4294967296.0f, added, not -inf;
 *                                        mask [Bm, Lk] float, nullable, Bm divides H*B (K.tile)
 *     s   = C where j > i                (causal != 0: replaced, as tf.where; needs Lq == Lk)
 *     p   = softmax_j(s);  with rate > 0: p * keep(r,i,j) * fl32(1 / (1 - rate))
 *     out = p . v
 *   So a row whose keys are all padding gets uniform weights (the mean of v), and with causal
 *   masking and key 0 padded, row 0 gets uniform weights over all Lk keys, future ones included.
 *   Dropout: rate in [0, 1), 64-bit seed.  keep(r,i,j) is a stateless splitmix64 finalizer:
 *     c = (r*Lq + i)*Lk + j;  z = seed + (c + 1) * 0x9E3779B97F4A7C15   (mod 2^64)
 *     z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;  z = (z ^ (z >> 27)) * 0x94D049BB133111EB;
 *     z ^= z >> 31;  keep = (z >> 40) >= (uint32)(rate * 2^24)     (rate widened to double)
 *   rate = 0 takes a path with no hashing.
 *   lse [H*B, Lq] float64 (saved for the backward): m + log(l).  float64 because a fully padded
 *   row has lse = C + log(Lk), which fp32 (ulp 512 at 2^32) rounds back to C.
 *   Served: 1 <= dh <= 128 (DR_ENOTSUP above), any Lq, Lk >= 1, H*B*max(Lq, Lk) < 2^31.
 *   B = 0 is a no-op.  Exact fp32 FFMA; every output element has one owner (bit-identical reruns).
 *
 * dr_mha_attn_bwd: no reference lines (TensorFlow autodiff of the above).  Recomputes p from lse;
 *   D_i = rowsum(g_out * out); ds = p * (dp - D_i), passed through the mask add and zero where the
 *   causal rule replaced the score; d(q . k) = ds * fl32(1 / fl32(sqrt(dh))) (within an ulp of the
 *   division TF's autodiff does).  Writes gq, gk, gv (overwritten; gk / gv from a CTA per key
 *   block looping over queries, gq from a CTA per query block: deterministic).  The dropout mask
 *   is regenerated from (seed, rate).                                                         */
int dr_mha_attn_fwd(const float* q, const float* k, const float* v, const float* mask, int64_t B,
                    int H, int Lq, int Lk, int dh, int64_t Bm, int causal, float rate, uint64_t seed,
                    float* out, double* lse, void* stream);
int dr_mha_attn_bwd(const float* q, const float* k, const float* v, const float* mask,
                    const float* out, const double* lse, const float* g_out, int64_t B, int H,
                    int Lq, int Lk, int dh, int64_t Bm, int causal, float rate, uint64_t seed,
                    float* gq, float* gk, float* gv, void* stream);

/* LayerNormalization of x + residual (the Transformer's Add & Norm), rows of width C.
 *   replaces: keras/models/nlp/transformer.py:109-113 (LayerNormalization.call) applied to the sum
 *   of :212-213, :218-219, :245-246, :253-254, :260-261.  residual is nullable.  Per row of
 *   s = x + residual: mu = mean, var = mean((s - mu)^2) (population, tf.nn.moments),
 *   y = gamma * ((s - mu) / (var + eps) ** 0.5) + beta.  One warp per row.
 * dr_add_layernorm_bwd: gx [N, C] (the gradient of both x and residual), ggamma and gbeta [C]
 *   (column sums, overwritten, summed with floating-point atomics: their last bits can differ
 *   from run to run).  Serves C <= 4096 (DR_ENOTSUP above).                                    */
int dr_add_layernorm_fwd(const float* x, const float* residual, const float* gamma,
                         const float* beta, int64_t N, int C, float eps, float* y, void* stream);
int dr_add_layernorm_bwd(const float* x, const float* residual, const float* gamma,
                         const float* gy, int64_t N, int C, float eps, float* gx, float* ggamma,
                         float* gbeta, void* stream);

/* Row softmax over x [N, V]: y = exp(x - max) / sum.
 *   replaces: keras/models/nlp/transformer.py:264-265 (K.softmax over the vocabulary).
 * dr_softmax_rows_bwd: gx = y * (gy - sum(gy * y)) from the saved y.  One warp per row.       */
int dr_softmax_rows_fwd(const float* x, int64_t N, int V, float* y, void* stream);
int dr_softmax_rows_bwd(const float* y, const float* gy, int64_t N, int V, float* gx,
                        void* stream);

/* GCN aggregation: CSR sparse (adjacency) times dense (features) with a fused epilogue.
 *   replaces: keras/models/retrieval/gcn.py:45-55 (tf.sparse.sparse_dense_matmul(adj, features), the Dense's bias
 *   and activation when the layer multiplies by the kernel first, and `outputs += features`).
 *   A [n_rows, n_cols] in CSR: indptr int32 [n_rows + 1], indices int32 [nnz], values fp32 [nnz]; x [n_cols, F].
 *   y[r, f] = act(sum_{p = indptr[r]}^{indptr[r+1]-1} values[p] * x[indices[p], f] + bias[f])
 *     the sum is fp32 fmaf in ascending p, from +0.0; duplicate column indices are summed, unsorted rows are summed in
 *     their stored order; an empty row gives act(bias); an index outside [0, n_cols) contributes nothing and is never
 *     dereferenced.  act: DR_ACT_NONE/RELU/SIGMOID/TANH, or DR_ACT_SOFTMAX (max subtracted, expf, divided by the sum
 *     over the row's F values; served for F <= 1024, DR_ENOTSUP above).
 *   out = y + residual (residual [n_rows, F]): written only when residual != NULL, and y is still written (the
 *     backward needs act' of y).  bias [F] and residual are nullable; out must be given with a residual.
 *   One owner (a group of 1..32 lanes) per output row, no atomics: reruns are bit-identical.
 *   Served: n_rows, n_cols, nnz < 2^31 (DR_ENOTSUP outside), any F >= 1.  n_rows = 0 is a no-op.
 *   The backward is this entry on the transposed CSR (entries of each transposed row in ascending original row) with
 *   act = DR_ACT_NONE and no bias; the CSR arrays are inputs only, so the values get no gradient.               */
int dr_spmm_csr_fwd(const int* indptr, const int* indices, const float* values, int64_t n_rows, int64_t n_cols,
                    int64_t nnz, const float* x, int F, const float* bias, const float* residual, int act, float* y,
                    float* out, void* stream);
/* Activation gradient and bias gradient of a fused epilogue such as the one above:
 *   gz = gy * act'(y) (act'(y) from the saved output y; gz may alias gy), gb[n] = sum_m gz[m, n] (OVERWRITTEN).
 *   act: DR_ACT_NONE/RELU/SIGMOID/TANH; with DR_ACT_NONE gz is gy and is not written (y and gz may be NULL).
 *   gb is nullable; it is summed with floating-point atomics, so its last bits can differ from run to run, as the
 *   gb of dr_dense_bwd can.  The same pass dr_dense_bwd runs before its GEMMs, without them.                     */
int dr_act_bwd_colsum(const float* y, const float* gy, int64_t M, int N, int act, float* gz, float* gb,
                      void* stream);

/* Multi-gate mixture of experts: every task's gate softmax and expert mixture in one pass.
 *   replaces: estimator/models/multi_task_learning/mixture_of_experts.py:46-53 (gating softmax), :69 (tf.stack of the
 *   experts), :73-78 (per gate: expand_dims, [B,1,E] @ [B,E,H] matmul, squeeze).  The reference builds num_experts
 *   gates and uses the first num_tasks; this serves exactly T gates.
 *   experts [B, E*H] (expert e = column block e*H), logits [B, T*E] (task t's gate logits = column block t*E).
 *   gates [B, T*E] (saved): gates[b,t,:] = softmax(logits[b,t,:]) -- max subtracted, expf, divided by the sum.
 *   out [B, T*H]: out[b, t*H + h] = sum_e gates[b,t,e] * experts[b, e*H + h]   (e ascending, fp32 fmaf onto an
 *   accumulator that starts at -0.0, so the first step is exactly the first product).  E = 1: the gate is exactly 1
 *   and out equals the expert bit for bit, signed zeros included (a NaN expert gives a NaN, not its payload).
 * dr_moe_mix_bwd: no reference lines (TensorFlow autodiff of the above).
 *   g_experts[b,e,h] = sum_t gates[b,t,e] * g_out[b,t,h];  dg[b,t,e] = sum_h g_out[b,t,h] * experts[b,e,h];
 *   g_logits[b,t,e] = gates[b,t,e] * (dg[b,t,e] - sum_e' gates[b,t,e'] * dg[b,t,e'])   (both overwritten).
 *   One warp owns a row; sums are per-lane in a fixed order plus a fixed butterfly: no atomics, every output element
 *   has one owner, reruns are bit-identical.
 *   Served: 1 <= E <= 32, 1 <= T <= 16, any H >= 1 with E*H, T*H < 2^31 (DR_ENOTSUP outside).  B = 0 is a no-op. */
int dr_moe_mix_fwd(const float* experts, const float* logits, int64_t B, int E, int T, int H, float* gates,
                   float* out, void* stream);
int dr_moe_mix_bwd(const float* experts, const float* gates, const float* g_out, int64_t B, int E, int T, int H,
                   float* g_experts, float* g_logits, void* stream);

/* ---------------------------------------------------------------------------------------
 * Row R (+R1, R2): in-batch softmax loss of the two-tower Retrieval task, fused
 *   Q @ C^T + online log-sum-exp; the [nq, nc] score matrix is never materialised.
 *   replaces: keras/models/retrieval/sbcnm.py:120-151 (Retrieval.call), :78-86
 *             (SamplingProbabilityCorrection), :52-75 (RemoveAccidentalNegative).
 *   s_ij = (q_i . c_j - log p_j + dup_ij * MIN_FLOAT) * inv_tau,
 *          dup_ij = [cand_ids_j == cand_ids_i] - [i == j],  MIN_FLOAT = FLT_MIN_ish/100
 *   loss = sum_i w_i * (logsumexp_j s_ij - s_ii)      (CategoricalCrossentropy, SUM)
 *   Q [nq,D], C [nc,D], nq <= nc (labels = eye(nq,nc)); w [nq] or NULL; p [nc] or NULL;
 *   cand_ids [nc] int64 or NULL; lse_out [nq] saved for backward; loss_out [1] OVERWRITTEN.
 * backward: G_ij = gl * w_i * (softmax(s)_ij - [i==j]) * inv_tau ; gQ = G @ C ; gC = G^T @ Q
 *   (gQ, gC OVERWRITTEN; gloss [1] device scalar = upstream gradient of the loss).
 * ------------------------------------------------------------------------------------- */
int dr_inbatch_softmax_fwd(const float* q, const float* c, const float* w, const float* p,
                           const int64_t* cand_ids, float inv_tau, int64_t nq, int64_t nc, int D,
                           float* lse_out, float* loss_out, void* stream);
int dr_inbatch_softmax_bwd(const float* q, const float* c, const float* w, const float* p,
                           const int64_t* cand_ids, float inv_tau, int64_t nq, int64_t nc, int D,
                           const float* lse, const float* gloss,
                           float* gq, float* gc, void* stream);

/* Tensor-core form of the same loss (the contraction of sbcnm.py:129 and both gradient contractions on the wgmma
 * 3xTF32 GEMM core).  scores_ws: caller-provided scratch [ws_rows, nc] floats; query rows are processed in blocks of
 * ws_rows (ws_rows >= nq: one block).  Same arguments, results and reduction as dr_inbatch_softmax_fwd / _bwd.
 * bwd: scores_valid != 0 and ws_rows >= nq means scores_ws still holds what the forward of the SAME inputs left there
 * (the raw corrected scores), so the score GEMM is not repeated; the workspace is consumed (overwritten) either way. */
int dr_inbatch_softmax_fwd_ws(const float* q, const float* c, const float* sample_weight, const float* sampling_prob,
                              const int64_t* cand_ids, float inv_tau, int64_t nq, int64_t nc, int D,
                              float* scores_ws, int64_t ws_rows, float* lse_out, float* loss_out, void* stream);
int dr_inbatch_softmax_bwd_ws(const float* q, const float* c, const float* sample_weight, const float* sampling_prob,
                              const int64_t* cand_ids, float inv_tau, int64_t nq, int64_t nc, int D,
                              const float* lse, const float* gloss, float* scores_ws, int64_t ws_rows,
                              int scores_valid, float* gq, float* gc, void* stream);

/* Materialised score matrix with the same corrections (needed by HardNegativeMining and
 * by metrics): scores [nq,nc] = (Q @ C^T - log p + dup*MIN_FLOAT) (no temperature).       */
int dr_scores_fwd(const float* q, const float* c, const float* p, const int64_t* cand_ids,
                  int64_t nq, int64_t nc, int D, float* scores, void* stream);

/* Row R3: HardNegativeMining (sbcnm.py:33-49): per row, indices of the k largest of
 *   logits + labels*MAX_FLOAT (labels = eye) ; emits gathered logits [nq,k], labels [nq,k]
 *   and the chosen column indices [nq,k] (int32).  Order inside a row is by descending
 *   score (TF: sorted=False => unspecified).                                              */
int dr_hard_negative_topk(const float* logits, int64_t nq, int64_t nc, int k,
                          float* out_logits, float* out_labels, int32_t* out_idx, void* stream);

/* ---------------------------------------------------------------------------------------
 * Row-sharded tables (SURVEY 8e): owner(r) = r mod G, local row = r div G.
 *   dr_shard_bucket_ids: one pass over the flat id list [n] (n = B*S, slot = index % S).
 *     global row = slot_offsets[s] + id (all S tables share one row space; slot_offsets and
 *     rows may be NULL = ids are already global rows); an id outside [0, rows[s]) becomes
 *     row -1 (owner 0, local id -1 => zero vector at the owner).
 *     The send buffer is PADDED to a fixed capacity so the exchange is an equal-split
 *     all-to-all with no host synchronisation: segment g = send_ids[g*cap, (g+1)*cap) holds the
 *     local row ids (row div G) destined to rank g, -1 in unused slots.  inv[i] = slot of
 *     lookup i (-1 on overflow).  send_counts[G] = used slots per segment; overflow[0] is SET to 1 if
 *     some segment needed more than cap slots and never cleared by the library (sticky: the caller zeroes it
 *     before the first call and after each read, then re-runs the truncated batch with a larger cap).
 *     Order inside a segment is unspecified.  Requires G*cap < 2^31.
 *   The exchange (ids out, vectors back, gradients out) is an NCCL all-to-all issued by the
 *   host through torch.distributed.  Because inv IS a gather index, the returned vectors are
 *   consumed directly by dr_embed_fm_fwd (table = the receive buffer, ids = inv), which fuses
 *   the un-permute with the FM reduction; dr_embed_fm_bwd with the same ids packs the
 *   per-lookup gradients for the way back.  dr_permute_rows / dr_unpermute_rows are the plain
 *   row shuffles (out[i] = in[perm[i]] / out[perm[i]] = in[i]; negative perm entries skipped).
 * ------------------------------------------------------------------------------------- */
int dr_shard_bucket_ids(const void* ids, int id_bytes, int64_t n, int S,
                        const int64_t* slot_offsets, const int64_t* rows, int G, int64_t cap,
                        int64_t* send_counts, int64_t* send_ids, int32_t* inv, int32_t* overflow,
                        void* stream);
/* Row-sharded gather / update fused with the exchange over NVLink peer memory (the multi-GPU path for
 * N > 1).  peer_bases[world] (device array): base of every rank's arena, mapped into this process
 * (CUDA IPC / symmetric memory); all ranks use the same row_stride.  Lookup (s, id) reads global
 * row slot_offsets[s] + id from rank (row mod world) at local row (row div world) -- the LDG.128
 * wave that gathers the row is itself the transfer, so there is no id exchange, no owner-side
 * gather and no all-to-all.  The backward issues its vector atomics (red.global.add.v4.f32)
 * straight into the owner's arena.  The caller separates a step's remote reads from its remote
 * updates with a collective on the tower gradients and ends the step with a barrier.
 * Same outputs / gradient formulas as dr_embed_fm_fwd / dr_embed_fm_bwd.
 * First-order weights: with DR_EMBED_LIN_IN_ROW they ride in the row at float D (D <= 124, rows of 128-B lines);
 * for wider rows (BASELINE config C5, D = 128) pass flags = 0 and lin_offset > 0: rank g keeps the weight of its
 * local row l at peer_bases[g] + lin_offset + l (floats), i.e. a [local rows] array trailing the [local rows, D]
 * shard in the same mapped allocation.  lin_offset = 0 and flags = 0: no first-order term.                  */
int dr_embed_fm_fwd_sharded(const float* const* peer_bases, int world, const int64_t* slot_offsets,
                            const int64_t* rows, const void* ids, int id_bytes, const float* bias,
                            int64_t B, int S, int D, int64_t row_stride, int flags, int64_t lin_offset,
                            float* out_stack, float* out_sum, float* out_logit, void* stream);
int dr_embed_fm_bwd_sharded(float* const* peer_bases, int world, const int64_t* slot_offsets,
                            const int64_t* rows, const void* ids, int id_bytes, const float* stack,
                            const float* sum_e, const float* g_logit, const float* g_stack,
                            int64_t B, int S, int D, int64_t row_stride, int flags, int64_t lin_offset,
                            float* g_bias, float scale, void* stream);

int dr_permute_rows(const float* in, const int32_t* perm, int64_t n, int D, float* out, void* stream);
int dr_unpermute_rows(const float* in, const int32_t* perm, int64_t n, int D, float* out, void* stream);

/* Fused SGD for dense parameters: p -= lr * g  (n elements). */
int dr_sgd_step(float* p, const float* g, int64_t n, float lr, void* stream);
/* Binary cross-entropy on logits, mean over B (tf.keras.losses.binary_crossentropy on
 * sigmoid outputs == this on logits), and its gradient wrt the logits.  The logit is
 * z[b] + z_add[b] (z_add may be NULL): DeepFM's  fm_logit + dnn_logit  (deepfm.py:46-47).
 *   loss[0] = mean_b( max(z,0) - z*y + log1p(exp(-|z|)) ) ; gz[b] = (sigmoid(z)-y)/B.
 *   prob_out [B] (sigmoid) and gz may be NULL.                                            */
int dr_bce_logits_fwd_bwd(const float* z, const float* z_add, const float* y, int64_t B,
                          float* prob_out, float* loss_out, float* gz, void* stream);

/* The skinny end of the deep tower in ONE kernel: the final Dense(1) layer (deepfm.py:30-34 `+ [Dense(1)]`, estimator
 * dnn.py hidden_units + [1]), `fm + dnn` (deepfm.py:46-47), binary cross-entropy on the sigmoid, and their backward.
 *   a [B,K] = act_prev(z_prev): output of the layer below (K <= 256), w [K] (= kernel [K,1]), bias [1] (nullable).
 *   logit = a.w + bias (+ z_add);  loss[0] = mean BCE as in dr_bce_logits_fwd_bwd;  g_logit[b] = (sigmoid - y)/B.
 *   g_prev [B,K] = g_logit * w * act_prev'(a): already the PRE-activation gradient of the layer below (cf.
 *   dr_dense_bwd_chain);  gw [K], gb [1], gb_prev [K] = colsum(g_prev) are OVERWRITTEN.
 *   logit_out (the Dense(1) output without z_add), prob_out, g_logit, g_prev, gw, gb, gb_prev may each be NULL. */
int dr_dense_head_bce_fwd_bwd(const float* a, const float* w, const float* bias, const float* z_add,
                              const float* y, int64_t B, int K, int prev_act, float* logit_out,
                              float* prob_out, float* loss_out, float* g_logit, float* g_prev, float* gw,
                              float* gb, float* gb_prev, void* stream);

/* The tail of a DCN in ONE kernel and without the concat: Dense(1)(concat[x_cross, deep]) -> sigmoid cross-entropy (mean
 * over B, as dr_bce_logits_fwd_bwd) -> their backward.
 *   replaces: keras/models/ranking/dcn.py:70-88 stacked as in tests/keras/test_dcn.py:27-32 (Cross ... -> Dense(1)), with
 *             the deep tower's output as the second block of the Dense(1) input.
 *   x_cross [B,d]: output of the top Cross layer; deep [B,n] = act(z): output of the last DNN layer; w [d+n] (= kernel
 *   [d+n,1]: rows 0..d-1 multiply x_cross, the rest deep); bias [1] (nullable).  d + n <= 4096, else DR_ENOTSUP.
 *   logit = x_cross.w[0:d] + deep.w[d:] + bias;  g_logit[b] = (sigmoid - y)/B
 *   g_xc [B,d] = g_logit * w[0:d]                   gradient into the top Cross layer
 *   g_deep [B,n] = g_logit * w[d:] * act'(deep)     PRE-activation gradient of the last DNN layer (cf. dr_dense_bwd_chain)
 *   gw [d+n], gb [1], gb_deep [n] = colsum(g_deep) are OVERWRITTEN;  loss_out [1] OVERWRITTEN.
 *   logit_out, prob_out, g_logit, g_xc, g_deep, gw, gb, gb_deep may each be NULL. */
int dr_dcn_head_bce_fwd_bwd(const float* x_cross, const float* deep, const float* w, const float* bias,
                            const float* y, int64_t B, int d, int n, int deep_act, float* logit_out,
                            float* prob_out, float* loss_out, float* g_logit, float* g_xc, float* g_deep,
                            float* gw, float* gb, float* gb_deep, void* stream);

/* =======================================================================================
 * SURVEY.md 8(f) "next" rows: the callers either side of the hot path.
 * ======================================================================================= */

/* ---- 8(f) #1  Adam (examples/train_deepfm_on_movielens_keras.py:44, train_fm_on_movielens_estimator.py:51).
 * TensorFlow's Adam is dense even for IndexedSlices gradients (every row's m, v decay and every row moves
 * each step), so the parity-exact form is one pass over the whole parameter / table arena:
 *   m += (g - m)(1 - beta1);  v += (g*g - v)(1 - beta2);  p -= lr_t * m / (sqrt(v) + eps)
 * with lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t) computed by the caller (t = 1, 2, ...).
 * g holds the accumulated gradient (dr_embed_fm_bwd / dr_scatter_add with scale = 1, or a dense gradient);
 * zero_grad = 1 clears it in the same pass.  eps = 1e-7 (tf.keras) or 1e-8 (tf.train.AdamOptimizer).   */
/* lr_t_dev (nullable): device float that overrides lr_t -- the bias-corrected rate dr_adam_advance maintains, so
 * a captured CUDA graph needs no per-step scalar.                                                          */
int dr_adam_step(float* p, float* g, float* m, float* v, int64_t n, float lr_t, float beta1, float beta2,
                 float eps, int zero_grad, const float* lr_t_dev, void* stream);

/* dr_adam_step (zero_grad = 0) over n_tensors flat tensors p[i], g[i], m[i], v[i] of n[i] floats each, in one launch
 * per 64 non-empty tensors: the dense half of tf.keras.optimizers.Adam over a whole model, which the reference compiles
 * every Keras model with (examples/train_deepfm_on_movielens_keras.py:44 `Adam()`, train_gcn_on_cora_keras.py:29
 * `Adam(0.01)`, train_transformer_on_imdb_keras.py:45 `Adam(beta_1=0.9, beta_2=0.98, epsilon=1e-9)`).  Every element
 * is bitwise what dr_adam_step gives it: a tensor whose four pointers are 16-B aligned takes the float4 path, any other
 * and every tail the scalar one.  The arrays are host memory, read before the call returns; their contents travel in
 * the kernel's argument block (no copy, no synchronisation: graph-capturable).  lr_t_dev (nullable) overrides lr_t.
 * n[i] = 0 skips tensor i (its pointers may be NULL); a negative n, a NULL pointer of a non-empty tensor or an
 * out-of-range beta / eps returns DR_EINVAL before any launch. */
int dr_adam_step_multi(int n_tensors, float* const* p, float* const* g, float* const* m, float* const* v,
                       const int64_t* n, float lr_t, float beta1, float beta2, float eps, const float* lr_t_dev,
                       void* stream);

/* Step counter on the device (Keras optimizer_v2 Adam._prepare_local): *step_dev += 1 and
 * *lr_t_dev = lr * sqrt(1 - beta2^t) / (1 - beta1^t) with t the incremented step (first call: t = 1).         */
int dr_adam_advance(int64_t* step_dev, float lr, float beta1, float beta2, float* lr_t_dev, void* stream);

/* Row-sparse ("lazy") Adam over the rows one batch touched: NOT tf.keras.optimizers.Adam (which decays m, v of
 * every row every step = dr_adam_step over the arena) but tfa.optimizers.LazyAdam -- an opt-in deviation for
 * tables where the dense pass (7 arena sweeps) would dominate the step.
 * Arenas p, g, m, v share one layout: row (slot_offsets[s] + id) * row_stride floats, D embedding floats first and,
 * with DR_EMBED_LIN_IN_ROW, the first-order weight at float D.  g must hold the batch's row gradients already summed
 * over duplicate ids (dr_embed_fm_bwd with scale = 1 into g) and zeros elsewhere; on return the touched rows of g
 * are zero again.  stamp: int32 [total rows], zero-initialised by the caller once; a row is updated exactly once
 * per step no matter how many lookups hit it.  lin_p/g/m/v (nullable together): split-layout first-order arrays
 * [total rows].  step_dev / lr_t_dev: maintained by dr_adam_advance.                                          */
int dr_lazy_adam_rows(const void* ids, int id_bytes, int64_t B, int S, int D, const int64_t* rows,
                      const int64_t* slot_offsets, float* p, float* g, float* m, float* v, int64_t row_stride,
                      int flags, float* lin_p, float* lin_g, float* lin_m, float* lin_v, int32_t* stamp,
                      const int64_t* step_dev, const float* lr_t_dev, float beta1, float beta2, float eps,
                      void* stream);

/* Row-sparse Adam FUSED INTO the backward scatter (one kernel per step; the same tfa-LazyAdam semantics as
 * dr_lazy_adam_rows: rows the batch does not touch keep p, m, v -- on touched rows the update is TensorFlow's ApplyAdam
 * functor exactly).  replaces: the IndexedSlices gradient of the embedding / first-order variables going through
 * tf.keras.optimizers.Adam (examples/train_deepfm_on_movielens_keras.py:44) for the rows of one batch.
 *   state: [total rows, stride] floats, stride = dr_embed_adam_state_stride(D) (a 128-B multiple), zero-initialised once
 *          by the caller; per row [g D | m D | v D | g_w m_w v_w count stamp | pad] (g = gradient accumulator, zero between
 *          steps; count = int32 countdown, zero between steps).
 *   dr_embed_adam_count: count[row] += 1 for every valid lookup of the batch (any time before the backward of the
 *          same batch, e.g. on a side stream while the forward runs).
 *   dr_embed_fm_bwd_adam: same inputs as dr_embed_fm_bwd (ids, saved stack / sum_e, g_logit, g_stack); every lookup
 *          adds its gradient row into state with vector atomics and decrements the row's count; the lookup that takes it
 *          to zero applies m += (g-m)(1-b1), v += (g*g-v)(1-b2), p -= lr_t*m/(sqrt(v)+eps) to the row of the PARAMETER
 *          table (table_ptrs / lin_ptrs, layouts as in dr_embed_fm_fwd) and clears g.  g_bias (nullable) accumulates the
 *          FM bias gradient (sum of g_logit) for a following dr_adam_step.  lr_t_dev: maintained by dr_adam_advance. */
int dr_embed_adam_state_stride(int D);
int dr_embed_adam_count(const void* ids, int id_bytes, int64_t B, int S, int D, const int64_t* rows,
                        const int64_t* slot_offsets, float* state, void* stream);
int dr_embed_fm_bwd_adam(const void* ids, int id_bytes, const int64_t* rows, const int64_t* slot_offsets,
                         const float* stack, const float* sum_e, const float* g_logit, const float* g_stack,
                         int64_t B, int S, int D, int64_t row_stride, int64_t lin_stride, int flags,
                         float* const* table_ptrs, float* const* lin_ptrs, float* state, float* g_bias,
                         const float* lr_t_dev, float beta1, float beta2, float eps, void* stream);

/* The same fused row-sparse Adam made EQUAL to tf.keras.optimizers.Adam (which is dense: in a step that does not touch
 * a row, its m and v still decay and the row still moves by its decayed momentum).  Each state block also holds the
 * step stamp of the row's last update (float index 3 D + 4); when a row is touched again the kernel first replays the
 * steps it sat out (dr_embed_adam_prepare, before the forward, so the forward already sees the moved row)
 * -- m -= m(1-b1), v -= v(1-b2), p -= lr_j m / (sqrt(v) + eps) for j = stamp+1 .. t-1, lr_j from the
 * ring `lr_hist` [hist_len] that dr_adam_advance_hist fills (recomputed from lr, beta1, beta2 for steps that fell out of
 * the ring) -- and then applies step t with the batch's gradient.  dr_embed_adam_flush replays the pending steps of
 * EVERY row up to the current step: call it before the tables are read outside the trainer (evaluation, checkpoint).
 * With it, parameters equal those of dr_adam_step applied densely every step (tests: float64 ApplyAdam oracle). */
int dr_adam_advance_hist(int64_t* step_dev, float lr, float beta1, float beta2, float* lr_t_dev,
                         float* lr_hist, int hist_len, void* stream);
/* Per step, BEFORE the forward of the batch (it replaces dr_embed_adam_count): counts the batch's lookups per row and
 * replays the pending steps (stamp, t-1] of every row the batch touches, so that the forward reads the parameters
 * tf.keras Adam's dense update would have left there. */
int dr_embed_adam_prepare(const void* ids, int id_bytes, int64_t B, int S, int D, const int64_t* rows,
                          const int64_t* slot_offsets, int64_t row_stride, int64_t lin_stride, int flags,
                          float* const* table_ptrs, float* const* lin_ptrs, float* state,
                          const int64_t* step_dev, const float* lr_hist, int hist_len, float lr, float beta1,
                          float beta2, float eps, void* stream);
int dr_embed_fm_bwd_adam_tf(const void* ids, int id_bytes, const int64_t* rows, const int64_t* slot_offsets,
                            const float* stack, const float* sum_e, const float* g_logit, const float* g_stack,
                            int64_t B, int S, int D, int64_t row_stride, int64_t lin_stride, int flags,
                            float* const* table_ptrs, float* const* lin_ptrs, float* state, float* g_bias,
                            const int64_t* step_dev, const float* lr_t_dev, const float* lr_hist, int hist_len,
                            float lr, float beta1, float beta2, float eps, void* stream);
int dr_embed_adam_flush(const int64_t* rows, const int64_t* slot_offsets, int S, int D, int64_t total_rows,
                        int64_t row_stride, int64_t lin_stride, int flags, float* const* table_ptrs,
                        float* const* lin_ptrs, float* state, const int64_t* step_dev, const float* lr_hist,
                        int hist_len, float lr, float beta1, float beta2, float eps, void* stream);

/* The same TensorFlow-equal Adam for the layer API (optimizers.RowSparseAdam), where a forward may run without a
 * backward and the gradient of a lookup comes in several layouts.  Same state blocks (dr_embed_adam_state_stride), same
 * clock (dr_adam_advance_hist), same replay and kCatchUpMax cap as above.  Lookups are ids [n] with slot i % S.
 *   dr_embed_adam_catch_up  before a forward (training or evaluation, with step_dev = the last completed step t):
 *                           replays the pending steps (stamp, t] of every row the lookups read.  It counts nothing,
 *                           so a forward that no backward follows leaves no state behind.
 *   dr_embed_adam_rows_tf   after dr_adam_advance_hist moved step_dev to t and dr_embed_adam_count counted the same
 *                           lookups: step t on every row they touch.  The gradient row of lookup (b, s) is read at
 *                           g_emb + b * g_ld + s * g_slot (16-B aligned; multiples of 4 floats, each 0 or at least
 *                           D: a stride of 0 broadcasts one row), its first-order
 *                           gradient at g_lin + b * gl_ld + s * gl_slot.  g_lin is NULL exactly when the table has no
 *                           first-order weights (lin_ptrs NULL and no DR_EMBED_LIN_IN_ROW); then no first-order slot is
 *                           touched.  row_splits (nullable, [B + 1], row_splits[0] = 0, row_splits[B] = n) makes the
 *                           lookups the members of B bags of one slot (S = 1, mean combiner): each valid member takes its
 *                           bag's gradient row / the bag's valid count and its first-order gradient at scale 1.  Without
 *                           it, n = B * S.  Duplicate lookups of a row are summed before the update; ids < 0 or >= rows
 *                           take none.
 * Bad sizes, strides or flags, D outside {4, 8, ..., 128} or a null pointer return DR_EINVAL before any launch;
 * a misaligned g_emb / state DR_EALIGN. */
int dr_embed_adam_catch_up(const void* ids, int id_bytes, int64_t n, int S, int D, const int64_t* rows,
                           const int64_t* slot_offsets, int64_t row_stride, int64_t lin_stride, int flags,
                           float* const* table_ptrs, float* const* lin_ptrs, float* state, const int64_t* step_dev,
                           const float* lr_hist, int hist_len, float lr, float beta1, float beta2, float eps,
                           void* stream);
int dr_embed_adam_rows_tf(const void* ids, int id_bytes, int64_t n, int64_t B, int S, const int64_t* row_splits,
                          const int64_t* rows, const int64_t* slot_offsets, const float* g_emb, int64_t g_ld,
                          int64_t g_slot, const float* g_lin, int64_t gl_ld, int64_t gl_slot, int D,
                          int64_t row_stride, int64_t lin_stride, int flags, float* const* table_ptrs,
                          float* const* lin_ptrs, float* state, const int64_t* step_dev, const float* lr_t_dev,
                          const float* lr_hist, int hist_len, float lr, float beta1, float beta2, float eps,
                          void* stream);

/* The same tf.keras-equal Adam (examples/train_deepfm_on_movielens_keras.py:44 tf.keras.optimizers.Adam(),
 * examples/train_fm_on_movielens_estimator.py:51 tf.train.AdamOptimizer(0.01)) on ROW-SHARDED tables (owner(r) = r mod
 * world, local row r div world), the optimizer of ShardedDeepFMTrainStep(optimizer="adam_rows_tf").  Every cross-rank
 * access is a plain store (mark) or a vector red.add (the backward into the owners' gradient arenas) that nothing reads
 * before the ranks meet at a barrier; all Adam arithmetic runs on the owner, in its own memory.  Per rank: a gradient
 * arena in the shard's own layout (row_stride, first-order weight in the row with DR_EMBED_LIN_IN_ROW or trailing at
 * lin_offset floats from the base), an int32 touch array [local_rows], an int32 row list [local_rows] + device count, and
 * state blocks [local_rows, dr_embed_adam_state_stride(D)] (dr_embed_adam_flush runs on them with S = 1).  One step t
 * (step_dev after dr_adam_advance_hist):
 *   dr_shard_adam_mark    touch_bases[owner][local] = t for every valid lookup (global ids through slot_offsets / rows
 *                         over `world` peer touch arrays; the NCCL exchange passes its received local ids with world 1,
 *                         S = 1, rows = {local_rows}, slot_offsets = {0}; -1 padding is skipped).  Barrier.
 *   dr_shard_adam_prepare the owner lists its rows with touch == t (list, count: device-resident, no host sync) and
 *                         replays their pending steps (stamp, t-1], as dr_embed_adam_prepare.  Barrier, forward, backward
 *                         into the gradient arenas (scale 1 / world), barrier.
 *   dr_shard_adam_apply   step t on every listed row from its gradient row, which it zeroes; stamp = t, count = 0.
 * world outside [1, 64], D outside {4, 8, ..., 128} or a null pointer return DR_EINVAL before any launch. */
int dr_shard_adam_mark(const void* ids, int id_bytes, int64_t n, int S, const int64_t* slot_offsets,
                       const int64_t* rows, int world, int32_t* const* touch_bases, const int64_t* step_dev,
                       void* stream);
int dr_shard_adam_prepare(int32_t* touch, int64_t local_rows, int32_t* list, int32_t* count, int D,
                          int64_t row_stride, int64_t lin_offset, int flags, float* shard, float* state,
                          const int64_t* step_dev, const float* lr_hist, int hist_len, float lr, float beta1,
                          float beta2, float eps, void* stream);
int dr_shard_adam_apply(const int32_t* list, const int32_t* count, int64_t local_rows, int D, int64_t row_stride,
                        int64_t lin_offset, int flags, float* shard, float* grad, float* state,
                        const int64_t* step_dev, const float* lr_t_dev, float beta1, float beta2, float eps,
                        void* stream);

/* ---- 8(f) #2  id pipeline: raw feature value -> int64 row id, bit-exact with TensorFlow's columns.
 * categorical_column_with_hash_bucket = FarmHash Fingerprint64(bytes of str(value)) mod num_buckets
 * (tf.strings.to_hash_bucket_fast).  Device entries take device pointers; strings travel as one byte
 * buffer + offsets [n+1].  Integer features are hashed through their decimal string, as TF does.
 * The *_host twins run the same code on the CPU for features that arrive as host strings (TFRecord parse);
 * they take host pointers and need no GPU.                                                              */
int dr_hash_bucket_i64(const int64_t* values, int64_t n, int64_t num_buckets, int64_t* out_ids, void* stream);
int dr_hash_bucket_bytes(const uint8_t* bytes, const int64_t* offsets, int64_t n, int64_t num_buckets,
                         int64_t* out_ids, void* stream);
int dr_hash_bucket_i64_host(const int64_t* values, int64_t n, int64_t num_buckets, int64_t* out_ids);
int dr_hash_bucket_bytes_host(const uint8_t* bytes, const int64_t* offsets, int64_t n, int64_t num_buckets,
                              int64_t* out_ids);
uint64_t dr_fingerprint64_host(const uint8_t* s, int64_t len);
/* categorical_column_with_vocabulary_list on integer keys: keys_sorted [vocab_size] ascending,
 * vocab_index[j] = position of keys_sorted[j] in the user's list; a value not in the list -> default_id
 * (TF default -1 => zero embedding row, all-zero indicator).                                            */
int dr_vocab_lookup_i64(const int64_t* values, int64_t n, const int64_t* keys_sorted, const int64_t* vocab_index,
                        int64_t vocab_size, int64_t default_id, int64_t* out_ids, void* stream);
/* crossed_column (replaces tf.feature_column.crossed_column = tf.sparse.cross_hashed, example
 * train_wdl_on_movielens_estimator.py:37-47).  K keys (2 <= K <= 16); values / value_offsets / row_splits are HOST
 * arrays of K pointers (device pointers for dr_cross_hash, host pointers for the _host twin):
 *   values[k]         int64 values, or the bytes of strings when value_offsets[k] != NULL ([n+1] byte offsets);
 *   row_splits[k]     [B+1] splits of a multi-valued key, NULL when the key has one value per example.
 * A single-valued key drops its ignore values (empty string, -1); a multi-valued key keeps every value, as TensorFlow
 * keeps a SparseTensor's.  Each combination of one kept value per key (last key fastest)
 * gives id = (FingerprintCat64 chain from hash_key over Fingerprint64(string) / raw int64) mod num_buckets.
 *   out_splits == NULL         every key single-valued: out_ids[b] = the cross of b, -1 if a key has no kept value;
 *   out_splits, out_ids NULL   out_splits[0] = 0, out_splits[b+1] = number of crosses of b (caller takes the cumsum);
 *   both given                 the crosses of b are written to out_ids[out_splits[b] ..].                        */
int dr_cross_hash(int K, const void* const* values, const int64_t* const* value_offsets,
                  const int64_t* const* row_splits, int64_t B, uint64_t hash_key, int64_t num_buckets,
                  int64_t* out_splits, int64_t* out_ids, void* stream);
int dr_cross_hash_host(int K, const void* const* values, const int64_t* const* value_offsets,
                       const int64_t* const* row_splits, int64_t B, uint64_t hash_key, int64_t num_buckets,
                       int64_t* out_splits, int64_t* out_ids);

/* Wide part of Wide & Deep: tf.feature_column.linear_model over indicator / crossed columns
 * (estimator/models/ranking/wide_and_deep.py:31-33) and tf.train.FtrlOptimizer on it (train_wdl_on_movielens_estimator.py
 * :65-69).  state: 16-B aligned [total_rows + 1, 4] records {w, z, n, g} (weight, FTRL linear and accumulator slots,
 * batch gradient); record total_rows is the bias.  rows / slot_offsets [S] (device): slot s owns rows
 * [slot_offsets[s], + rows[s]).  ids [B, S] int64 single-valued lookups; n_bags (<= DR_WIDE_MAX_BAGS) multi-valued
 * slots replace their column of ids: bag_slots / bag_ids / bag_splits are HOST arrays (device pointers to flat ids and
 * [B+1] splits).  An id outside [0, rows[s]) contributes nothing; duplicates count.
 *   dr_wide_fwd   logit[b] = bias + sum of w over the lookups of b.
 *   dr_wide_bwd   g[row] += g_logit[b] per lookup; g[bias] += sum_b g_logit[b] (float atomics).
 *   dr_wide_ftrl  each touched row (and the bias) applies ApplyFtrl with learning_rate_power = -0.5 once:
 *                 n' = n + g^2; z += g - (sqrt(n') - sqrt(n)) / lr * w;
 *                 w = |z| > l1 ? (sign(z) l1 - z) / (sqrt(n') / lr + 2 l2) : 0; n = n'; then g = 0.
 *                 Untouched rows are not written: equal to TensorFlow's dense update while w is the function of
 *                 (z, n) the last update wrote (true from w = z = 0).  DR_EINVAL for lr <= 0, l1 < 0 or l2 < 0.   */
#define DR_WIDE_MAX_BAGS 16
int dr_wide_fwd(const float* state, int64_t total_rows, const int64_t* rows, const int64_t* slot_offsets,
                const int64_t* ids, int64_t B, int S, int n_bags, const int* bag_slots, const int64_t* const* bag_ids,
                const int64_t* const* bag_splits, float* logit, void* stream);
int dr_wide_bwd(float* state, int64_t total_rows, const int64_t* rows, const int64_t* slot_offsets,
                const int64_t* ids, int64_t B, int S, int n_bags, const int* bag_slots, const int64_t* const* bag_ids,
                const int64_t* const* bag_splits, const float* g_logit, void* stream);
int dr_wide_ftrl(float* state, int64_t total_rows, const int64_t* rows, const int64_t* slot_offsets,
                 const int64_t* ids, int64_t B, int S, int n_bags, const int* bag_slots, const int64_t* const* bag_ids,
                 const int64_t* const* bag_splits, float lr, float l1, float l2, void* stream);

/* Multi-valued slot (VarLenFeature, e.g. "Genres" movielens.py:122): ids [nnz] + row_splits [B+1].
 *   out[b, :] = combine_j table[ids[j], :D]  over the VALID ids (0 <= id < rows) of bag b;
 *   DR_COMBINER_MEAN divides by the number of valid ids (safe_embedding_lookup_sparse: ids < 0 are pruned
 *   first), SQRTN by its square root, SUM by 1; a bag without a valid id gives zeros.
 *   The indicator-column (first-order) term of such a slot is DR_COMBINER_SUM with D = 1.
 * bwd: grad_table[id, :D] += scale * g_out[b, :] / den(b) for every valid id (duplicates accumulate);
 *   scale = 1 for plain gradients, -lr for fused sparse SGD.  row_stride / out_stride / g_stride are row
 *   pitches in floats (>= D): out may be a [B, 32]-pitched scratch "table" in the fused row layout, which
 *   dr_embed_fm_fwd then reads as slot s with ids = 0..B-1 (this is how a multi-valued slot joins the fused
 *   gather + FM launch; its backward goes through the same scratch).                                     */
int dr_embed_bag_fwd(const float* table, int64_t rows, int64_t row_stride, const void* ids, int id_bytes,
                     const int64_t* row_splits, int64_t B, int D, int combiner, float* out, int64_t out_stride,
                     void* stream);
int dr_embed_bag_bwd(const void* ids, int id_bytes, const int64_t* row_splits, int64_t B, int D, int combiner,
                     const float* g_out, int64_t g_stride, int64_t rows, int64_t row_stride, float* grad_table,
                     float scale, void* stream);

/* FNN's tower input (estimator/models/ranking/fnn.py:53-82): concat([bias, w_1 .. w_S, e_1 .. e_S]) in one gather.
 *   Row layout: P = round_up(1 + S, 4), ld = P + S*D; column 0 = *bias, columns 1..S = w_s, columns 1+S..P-1 = 0,
 *   embedding s at [P + s*D, P + (s+1)*D).  Every embedding segment starts 16-B aligned and ld % 4 == 0.
 *   table_ptrs / lin_ptrs / rows / ids / id_bytes / row_stride / lin_stride / flags: as dr_embed_fm_fwd; with
 *   DR_EMBED_LIN_IN_ROW (the fused row layout) w is float D of the row and lin_ptrs may be NULL, otherwise
 *   lin_ptrs is required.  An id < 0 or >= rows[s] gives a zero embedding and a zero w.
 *   bias : device [1], read on the device.  out : [B, ld], 16-B aligned.
 * bwd: for every valid lookup (b, s): grad_table s [id, :D] += scale * g_x[b, P + s*D ...], and its first-order
 *   weight (float D of the row, or grad_lin_ptrs[s][id * lin_stride]) += scale * g_x[b, 1 + s].  Column 0 and the
 *   pad are not read.  scale = 1 with zeroed gradient arenas gives the dense gradient, scale = -lr with the
 *   pointers aliasing the parameters a fused sparse SGD step.
 * Both: DR_EINVAL for a null pointer, D % 4 != 0 or D outside [4, 128], ld != P + S*D, bad strides or flags;
 *   DR_EALIGN for a row buffer (out / g_x) that is not 16-B aligned; DR_ENOTSUP for B*S >= 2^31.  B = 0 is a no-op. */
int dr_fnn_input_fwd(const float* const* table_ptrs, const float* const* lin_ptrs, const int64_t* rows,
                     const void* ids, int id_bytes, int64_t row_stride, int64_t lin_stride, int flags,
                     const float* bias, int64_t B, int S, int D, int64_t ld, float* out, void* stream);
int dr_fnn_input_bwd(const void* ids, int id_bytes, const int64_t* rows, const float* g_x, int64_t B, int S, int D,
                     int64_t ld, int64_t row_stride, int64_t lin_stride, int flags, float* const* grad_table_ptrs,
                     float* const* grad_lin_ptrs, float scale, void* stream);

/* ---- 8(f) #4  input format: TFRecord file of serialized tf.train.Example (datasets/movielens.py:54-62 writer
 * schema, :116-125 tf.io.parse_example reader).  HOST entry points (no GPU needed), the native replacement of
 * tf.data.TFRecordDataset + tf.io.parse_example for this path; their outputs are exactly what the id pipeline above
 * consumes (packed strings + offsets, int64 values, row_splits for VarLenFeature).
 *   dr_crc32c_host / dr_masked_crc32c_host   CRC-32C (Castagnoli) and TFRecord's masked form rotr(c,15)+0xa282ead8.
 *   dr_tfrecord_index   scans `buf`: returns the number of records (or a negative DR_E*), fills rec_off / rec_len
 *                       (payload position and length) for the first `cap` records; verify_crc checks both CRCs.
 *   dr_example_parse_feature   feature `name` of n records -> columnar.  kind 0 = int64_list (values int64),
 *                       1 = bytes_list (bytes + value_offsets [total_values+1]), 2 = float_list (values float).
 *                       row_splits [n+1]: values of record r are [row_splits[r], row_splits[r+1]) -- a
 *                       FixedLenFeature([]) has exactly one, a VarLenFeature any number, an absent feature none.
 *                       Two-pass: with values == bytes == NULL only row_splits / *total_values / *total_bytes are
 *                       written, then the caller allocates and calls again.
 *   dr_vocab_lookup_bytes_host   categorical_column_with_vocabulary_list on strings (position, OOV -> default_id). */
uint32_t dr_crc32c_host(const uint8_t* data, int64_t n);
uint32_t dr_masked_crc32c_host(const uint8_t* data, int64_t n);
int64_t dr_tfrecord_index(const uint8_t* buf, int64_t nbytes, int verify_crc, int64_t* rec_off, int64_t* rec_len,
                          int64_t cap);
int dr_example_parse_feature(const uint8_t* buf, const int64_t* rec_off, const int64_t* rec_len, int64_t n,
                             const char* name, int kind, int64_t* row_splits, void* values, uint8_t* bytes,
                             int64_t* value_offsets, int64_t* total_values, int64_t* total_bytes);
/* dr_example_parse_batch: the same for nfeat features in ONE walk per record (what the dataset classes use):
 * names / kinds [nfeat]; row_splits / values / bytes / value_offsets are arrays of nfeat pointers with the per-feature
 * meaning above (values entry for int64 / float features, bytes + value_offsets entries for string features, unused
 * entries NULL); total_values / total_bytes [nfeat].  Sizing pass: values == bytes == value_offsets == NULL.      */
int dr_example_parse_batch(const uint8_t* buf, const int64_t* rec_off, const int64_t* rec_len, int64_t n, int nfeat,
                           const char* const* names, const int* kinds, int64_t* const* row_splits,
                           void* const* values, uint8_t* const* bytes, int64_t* const* value_offsets,
                           int64_t* total_values, int64_t* total_bytes);
/* Host threads used by dr_example_parse_batch on large batches (tf.data num_parallel_calls): 1 = serial (default),
 * 0 = min(hardware threads, 8), n = n threads.  The output does not depend on it.                              */
int dr_set_host_threads(int n);
int dr_vocab_lookup_bytes_host(const uint8_t* bytes, const int64_t* offsets, int64_t n, const uint8_t* vocab_bytes,
                               const int64_t* vocab_offsets, int64_t vocab_size, int64_t default_id, int64_t* out_ids);

/* ---- 8(f) #3  row-wise top-k (factorized_top_k.py:58-62,196-226,330-334 tf.math.top_k):
 * out_vals [nq,k] descending, out_idx [nq,k] int32 column indices, ties -> lower index first.
 * scores is [nq, nc] with row pitch ld floats.  k > nc is rejected like TF ("input must have at least k
 * columns").                                                                                            */
int dr_topk_rows(const float* scores, int64_t nq, int64_t nc, int64_t ld, int k, float* out_vals,
                 int32_t* out_idx, void* stream);

/* Companions of the selection (keras/models/retrieval/factorized_top_k.py):
 *   dr_take_long_axis   _take_long_axis :26-41: out[i,j] = arr[i, indices[i,j]] for 4- or 8-byte elements (scores,
 *                       int32/int64 identifiers); ld = row pitch in elements, ld == 0 = ONE shared row, i.e.
 *                       tf.gather(identifiers, indices) (:211,:334).  An index outside [0, ncols) gives 0.
 *   dr_exclude_adjust   _exclude :58-62: adjusted[i,j] = scores[i,j] - [identifiers[i,j] in exclude[i,:]] * penalty
 *                       (penalty = 1.0e5 in the reference); the caller then takes dr_topk_rows of `adjusted`.
 *   dr_rowwise_dot      FactorizedTopK.update_state :487-488: out[i] = sum_d a[i,d] * b[i,d].
 *   dr_column_rank      TopKCategoricalAccuracy over [positive | others] with the true class in column 0:
 *                       rank[i] = #{j : others[i,j] > positive[i]}; in_top_k(k) == rank < k.                    */
int dr_take_long_axis(const void* arr, int elem_bytes, int64_t nq, int64_t ncols, int64_t ld, const int32_t* indices,
                      int k, void* out, void* stream);
int dr_exclude_adjust(const float* scores, const int64_t* identifiers, const int64_t* exclude, int64_t nq, int64_t n,
                      int64_t e, float penalty, float* adjusted, void* stream);
int dr_rowwise_dot(const float* a, const float* b, int64_t n, int D, float* out, void* stream);
int dr_column_rank(const float* positive, const float* others, int64_t nq, int64_t n, int64_t ld, int32_t* rank,
                   void* stream);

/* Scratch for the tensor-core GEMM variant (hi/lo TF32 operand planes).  The caller owns the
 * buffer and keeps it alive until it registers another one (ptr = NULL unregisters).  One
 * workspace per process: GEMM entry points that use it must not run concurrently on two
 * streams.  Without a (large enough) workspace the FFMA variant is used.                  */
int dr_set_workspace(void* ptr, uint64_t bytes);

/* Operand-plane cache of the tensor-core GEMMs.  enable=1: forget all cached planes and start
 * caching -- until the next call every distinct operand buffer is split into TF32 hi/lo planes once
 * and the planes are reused by later GEMMs that read the same buffer (valid only while the buffer
 * contents do not change: bracket ONE forward+backward pass, e.g. at the top of a train step).
 * enable=0: stop caching (every GEMM call splits its own operands; always safe).              */
int dr_gemm_plane_cache(int enable);

/* Developer hook (not reference-facing): set a kernel tuning knob by name, e.g.
 * "embed_fwd_unroll", "embed_block", "embed_bwd_agg", "gemm_splitk".                     */
int dr_tune_set(const char* key, int value);
/* Developer hook: read a knob back (tc_pair, tc_dw_share, gemm_variant, gemm_bn, tc_min_n); DR_EINVAL for other keys. */
int dr_tune_get(const char* key, int* value);

/* Developer hook: C[M,N] = op(A) @ op(B); transA: A stored [K,M]; transB: B stored [N,K].  */
int dr_debug_gemm(const float* A, const float* B, float* C, int64_t M, int64_t N, int64_t K,
                  int transA, int transB, void* stream);

/* Developer hook: the same GEMM with a fused epilogue and C's row pitch ldc (>= N):
 *   epi 0: C = acc;  1: C = act(acc + bias[n]);  2: C += acc (split-K over `splitk` parts, C pre-set by the caller);
 *   3: C = acc * act'(aux0[m, n]) (aux0 has pitch ldc). */
int dr_debug_gemm_epi(const float* A, const float* B, float* C, int64_t M, int64_t N, int64_t K,
                      int transA, int transB, int64_t ldc, int epi, int act, const float* bias,
                      const float* aux0, int splitk, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DEEPREC_B200_H_ */
