/*
 * tsc_learn.h — C ABI of the per-intersection A2C learner kernels in libtsc (sm_90a).
 *
 * Replaces, for R lock-stepped replicas and all A agents at once, the TF1 graphs of the reference:
 *   fc / lstm layers                         agents/utils.py:66-74, 88-116
 *   LstmACPolicy / FPLstmACPolicy forward    agents/policies.py:99-136, 191-211
 *   ACPolicy.prepare_loss + backward         agents/policies.py:41-61, 138-155
 *   OnPolicyBuffer._add_R_Adv                agents/utils.py:202-214
 *   clip_by_global_norm + RMSPropOptimizer   agents/policies.py:54-61  (TF1 semantics: ms starts
 *                                            at 1, epsilon inside the sqrt, no momentum)
 * Two networks per agent (pi and V, agents/policies.py:87-96) = 2A "units"; unit u = 2*agent + net.
 *
 * All pointers are caller-owned DEVICE pointers; `stream` is a cudaStream_t as void*.
 * Every function returns 0 or <0 (message via tsc_last_error()).  The three plain time-batched
 * GEMMs of the update (X.Wx, dZ.Wx^T, X^T.dZ) are NOT in this ABI: the host calls the vendor
 * library for them (DESIGN.md §5) until the tensor-core kernels replace them.
 */
#ifndef TSC_LEARN_H_
#define TSC_LEARN_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Static shape/offset description of the A agents (host struct; arrays are HOST pointers, copied
 * by tscl_create).  Observation row of agent i (envs/env.py:163-205):
 *   [wave (n_wave[i]) | wait (n_wait[i]) | fingerprints (n_fp[i])] at obs_off[i]. */
typedef struct tscl_dims {
  int32_t n_agents;   /* A                                                                 */
  int32_t n_obs;      /* row stride of the observation matrix                              */
  int32_t max_na;     /* padded action dimension (row stride of pi / fingerprints)         */
  int32_t fw, ff, ft; /* fc widths: num_fw, num_fp (0 = no fingerprint branch), num_ft     */
  int32_t h;          /* num_lstm (must be 64)                                             */
  int32_t dx;         /* fw + ff + ft                                                      */
  const int32_t* obs_off;  /* [A]                                                          */
  const int32_t* n_wave;   /* [A]                                                          */
  const int32_t* n_wait;   /* [A]                                                          */
  const int32_t* n_fp;     /* [A]                                                          */
  const int32_t* n_a;      /* [A]                                                          */
  /* offsets (in floats) into the flat parameter / gradient / RMS-slot vectors             */
  const int64_t* off_fcw_w; /* [2A] ragged [n_wave][fw]   */ const int64_t* off_fcw_b; /* [2A] */
  const int64_t* off_fcf_w; /* [2A] ragged [n_fp][ff]     */ const int64_t* off_fcf_b; /* [2A] */
  const int64_t* off_fct_w; /* [2A] ragged [n_wait][ft]   */ const int64_t* off_fct_b; /* [2A] */
  int64_t off_wx;  /* [2A][dx][4h] */
  int64_t off_wh;  /* [2A][h][4h]  */
  int64_t off_bl;  /* [2A][4h]     */
  int64_t off_wo;  /* [2A][h][max_na]  (V units use column 0) */
  int64_t off_bo;  /* [2A][max_na] */
  int64_t n_params;
} tscl_dims;

typedef struct tscl_handle tscl_handle;

int tscl_create(const tscl_dims* dims, int32_t device, tscl_handle** out);
int tscl_destroy(tscl_handle* h);

/* fc front end (agents/policies.py:191-201): X[u][m][0:dx] = relu(fc(...)) for m in [0, M).
 * Row m reads obs + (m / rows_per_t) * stride_t + (m % rows_per_t) * n_obs  (floats). */
int tscl_fc_embed(tscl_handle* h, const float* params, const float* obs, int64_t M, int64_t rows_per_t,
                  int64_t stride_t, float* X, void* stream);

/* FcACPolicy hidden layer (agents/policies.py:236: `h = fc(h, out_type + '_fc', n_fc)`), own register-tiled fp32 GEMM
 * kernels (PolicyLayout(recurrent=False): wx [2A][dx][h], bl [2A][h]):
 *   fwd  H[u][m][:] = relu(X[u][m][:] . wx[u] + bl[u])                                  X [2A][M][dx], H [2A][M][h]
 *   bwd  dH <- dH * (H > 0);  dX = dH . wx^T;  grads.wx += X^T dH;  grads.bl += 1^T dH   (tf.gradients through relu + matmul) */
int tscl_fc_hidden_fwd(tscl_handle* h, const float* params, const float* X, int64_t M, float* H, void* stream);
int tscl_fc_hidden_bwd(tscl_handle* h, const float* params, const float* X, const float* H, float* dH, int64_t M,
                       float* dX, float* grads, void* stream);

/* LSTM over T steps (agents/utils.py:88-116): recurrent GEMM h.Wh + fused cell.
 *   ZG   [2A][T*Rc][4h]  in: X.Wx + b (time-major rows m = t*Rc + r); out: gate activations i,f,o,u
 *   C,H  [2A][T*Rc][h]   out (may be NULL when T == 1 and only states are wanted)
 *   Hprev [2A][T*Rc][h]  out, may be NULL: the masked h_{t-1} each step consumed (operand of dWh)
 *   c0,h0 [2A][ld_state][h] initial state rows r0 .. r0+Rc;  c1,h1: final state (may alias c0,h0, may be NULL)
 *   done [T] float (pre-step done: state is zeroed BEFORE the cell, agents/utils.py:104-105) */
int tscl_lstm_seq_fwd(tscl_handle* h, const float* params, float* ZG, float* C, float* H, float* Hprev,
                      const float* c0, const float* h0, float* c1, float* h1, const float* done, int32_t T,
                      int64_t Rc, int64_t ld_state, int64_t r0, void* stream);

/* Heads for one control step (agents/policies.py:18-26, utils.py:155-157): softmax policy, value,
 * categorical sample with the counter-based RNG keyed (seed, step, replica0 + r, agent).
 *   Hs [2A][R][h] -> pi [R][A][max_na] (zero padded), val [R][A], act [R][A] (may be NULL) */
int tscl_heads(tscl_handle* h, const float* params, const float* Hs, int64_t R, float* pi, float* val,
               int32_t* act, uint64_t seed, int64_t step, int64_t replica0, void* stream);

/* n-step returns (agents/utils.py:202-214): R_t = r_t + gamma*R_{t+1}*(1-done_post_t), Adv = R - v.
 *   rew,val,Rs,Adv [T][R][A]; boot [R][A]; done_post [T] float */
int tscl_returns(tscl_handle* h, const float* rew, const float* val, const float* boot, const float* done_post,
                 float gamma, int32_t T, int64_t R, float* Rs, float* Adv, void* stream);
/* tscl_returns for a sweep of K members of R / K replicas each (K must divide R): replica r discounts with the device
 * float gamma[r / (R / K)].  Each member's rows of Rs / Adv equal tscl_returns run on those rows alone with its gamma. */
int tscl_returns_g(tscl_handle* h, const float* rew, const float* val, const float* boot, const float* done_post,
                   const float* gamma, int32_t K, int32_t T, int64_t R, float* Rs, float* Adv, void* stream);

/* Loss gradients at the heads for all (t, r) of a chunk (agents/policies.py:41-52):
 *   H [2A][M][h], act/Rs/Adv rows m -> base + (m / Rc)*stride_t + (m % Rc)*A
 *   dlog [2A][M][max_na] (out; V units use column 0), dH [2A][M][h] (out)
 *   stats [4] += {policy_loss, value_loss, entropy_loss, count} of agent 0 (agents/policies.py:63-72)
 *   scale = 1 / (n_step * total replicas): mean over the batch and over replicas
 *   h_bf16 (optional): read H from one chunk of the bf16 activation store ([2A][M][h]) instead of `H`
 *   grads (optional): also accumulate the head gradients  dWo += H^T dlog, dbo += sum dlog  into the flat
 *                     gradient vector; `dlog` may then be NULL */
int tscl_heads_loss(tscl_handle* h, const float* params, const float* H, const int32_t* act, const float* Rs,
                    const float* Adv, int64_t M, int64_t Rc, int64_t stride_t, float v_coef, float beta,
                    float scale, float* dlog, float* dH, float* stats, const void* h_bf16, float* grads,
                    void* stream);

/* BPTT through the LSTM (reverse of tscl_lstm_seq_fwd).  ZG holds gate activations on entry and
 * dZ (pre-activation gate gradients) on exit; dH holds head gradients on entry. */
int tscl_lstm_seq_bwd(tscl_handle* h, const float* params, float* ZG, const float* C, const float* dH,
                      const float* c0, const float* done, int32_t T, int64_t Rc, int64_t ld_state, int64_t r0,
                      void* stream);

/* fc front-end backward: grads[...] += obs^T . (dX * (X > 0)) and bias sums, rows as tscl_fc_embed. */
int tscl_fc_bwd(tscl_handle* h, const float* obs, const float* X, const float* dX, int64_t M,
                int64_t rows_per_t, int64_t stride_t, float* grads, void* stream);

/* The same contraction on the tensor cores (wgmma, MN-major bf16 operands, fp32 accumulation in the accumulator tile over
 * 128-row tiles; replaces the SIMT kernel in the training loop).  Pass the activations either as fp32 `X` or as one
 * chunk of the bf16 activation store `x_bf16` ([2A][M][dx]); `variant` must be 0. */
int tscl_fc_bwd_tc(tscl_handle* h, const float* obs, const float* X, const void* x_bf16, const float* dX,
                   const void* dx_bf16, int64_t M, int64_t rows_per_t, int64_t stride_t, float* grads, int32_t variant,
                   void* stream);
/* dX likewise as fp32 `dX` or bf16 `dx_bf16` ([2A][M][dx]). */

/* LSTM weight gradients of one chunk on the tensor cores:  grads.wx += X^T dZ, grads.wh += Hp^T dZ, grads.bl += 1^T dZ
 * (rows m = t * rc + r, M = T * rc; bf16 operands, fp32 accumulation).  X as fp32 `X` or bf16 `x_bf16`
 * ([2A][M][dx]); Hp as fp32 `Hp` ([2A][M][h]) or rebuilt from the bf16 store chunk `h_bf16` ([2A][T][rc][h]) as
 * (1 - done[t]) * (t > 0 ? H[t-1] : h0[u][r0 + r]).  `variant` must be 0. */
int tscl_wgrad_tc(tscl_handle* h, const float* dZ, const void* dz_bf16, const float* X, const void* x_bf16,
                  const float* Hp, const void* h_bf16, const float* h0, const float* done, int32_t T, int64_t rc,
                  int64_t ld_state, int64_t r0, float* grads, int32_t variant, void* stream);
/* dZ likewise as fp32 `dZ` or bf16 `dz_bf16` ([2A][M][256], written by tscl_lstm_seq_bwd_tc). */

/* BPTT on the tensor cores (wgmma): same contract as tscl_lstm_seq_bwd, with the recurrent product dz.Wh^T as
 * a bf16 MMA (M=128, N=64, K=256) per step; wt_bf16 [2A][32][64][8] comes from tscl_pack_wht (refresh after
 * every optimizer step).  With gates_bf16 / c_bf16 / dz_bf16 and ZG == NULL (the shipping call) each warpgroup runs the
 * recurrence of 64 replica rows in registers: its per-step operands (gates, c, dH: 56 KB) are fetched one step ahead by
 * cp.async.bulk.tensor copies, and dZ leaves by a bulk tensor store, through 3-D tensor maps [2A * T][Rc][cols] built over
 * the caller's arrays (cuTensorMapEncodeTiled via the driver entry point; if they cannot be built the call runs the
 * row-per-thread kernel, which gives the same bits); the arrays must be 16-byte aligned and hold 2A * T * Rc rows. */
int tscl_pack_wht(tscl_handle* h, const float* params, void* wt_bf16, void* stream);
int tscl_lstm_seq_bwd_tc(tscl_handle* h, const void* wt_bf16, float* ZG, const float* C, const float* dH, const float* c0,
                         const float* done, int32_t T, int64_t Rc, int64_t ld_state, int64_t r0,
                         const void* gates_bf16, const void* c_bf16, void* dz_bf16, void* stream);
/* The same kernel with dX = dZ . Wx^T fused into every step (second wgmma product of the same dz tile, M=128, N=dx,
 * K=256, accumulator columns 64..64+dx): wxt_bf16 [2A][32][dx][8] from tscl_pack_wxt (refresh after every
 * optimizer step), dx_bf16 [2A][T*Rc][dx] receives dX as bf16 — one way of replacing the last library GEMM of the update
 * (the shipping one is tscl_dx_tc below)
 * (reference: the tf.gradients chain through agents/utils.py:106, `tf.matmul(x, wx)`).  Both NULL = plain BPTT. */
int tscl_pack_wxt(tscl_handle* h, const float* params, void* wxt_bf16, void* stream);
int tscl_lstm_seq_bwd_tc_dx(tscl_handle* h, const void* wt_bf16, float* ZG, const float* C, const float* dH, const float* c0,
                            const float* done, int32_t T, int64_t Rc, int64_t ld_state, int64_t r0,
                            const void* gates_bf16, const void* c_bf16, void* dz_bf16, const void* wxt_bf16, void* dx_bf16,
                            void* stream);
/* tscl_heads_loss followed by the store-path tscl_lstm_seq_bwd_tc in one kernel: each BPTT step computes its dH from h_t
 * of the bf16 store `h_bf16` and the head weights in `params` with tscl_heads_loss's arithmetic, so dz_bf16 is bit-identical
 * to that pair's; the head weight / bias gradients are added to `grads` and agent 0's loss sums to `stats` (optional) as
 * tscl_heads_loss adds them (up to summation order).  Runs over `n_chunks` consecutive chunks of Rc replicas: gates_bf16 /
 * c_bf16 / h_bf16 / dz_bf16 are [n_chunks][2A][T][Rc][w] (the activation store's layout), chunk i's replicas are
 * r0 + i * Rc .. of c0 ([2A][ld_state][64]), and act / Rs / Adv point at the first chunk's first replica, row (t, r, a) at
 * t * stride_t + r * A + a with r counted over all chunks.  Needs cuTensorMapEncodeTiled and max_na <= 8. */
int tscl_lstm_seq_bwd_tc_heads(tscl_handle* h, const void* wt_bf16, const float* params, const void* gates_bf16,
                               const void* c_bf16, const void* h_bf16, const float* c0, const float* done,
                               const int32_t* act, const float* Rs, const float* Adv, int32_t T, int64_t Rc,
                               int32_t n_chunks, int64_t ld_state, int64_t r0, int64_t stride_t, float v_coef, float beta,
                               float scale, void* dz_bf16, float* stats, float* grads, void* stream);
/* Host-buffer loop, one call per replica range and control step (replaces the reference's per-step numpy hand-over of
 * ob / reward into `model.add_transition`, agents/models.py:222-229, main.py / utils.py:272-286): observations
 * host -> obs_dev (the rollout slot), rewards host -> rew_hist_dev = clip(reward / reward_norm) (0 = off for either),
 * global rewards host -> rew_acc_dev += (episode sum, utils.py:296-305).  *_stage_dev are device scratch of the same
 * size as the host arrays.  Host arrays should be page-locked; everything is enqueued on `stream`. */
int tscl_host_transition(tscl_handle* h, const float* obs_host, float* obs_dev, int64_t obs_floats, const float* rew_host,
                         float* rew_stage_dev, float* rew_hist_dev, int64_t rew_floats, float reward_norm, float reward_clip,
                         const float* grew_host, float* grew_stage_dev, float* rew_acc_dev, int64_t n, void* stream);
/* Same hand-over with the rewards already on the device (the device-resident loop): rew_hist_dev = clip(rew_dev /
 * reward_norm), rew_acc_dev += grew_dev, one launch. */
int tscl_device_transition(tscl_handle* h, const float* rew_dev, float* rew_hist_dev, int64_t rew_floats, float reward_norm,
                           float reward_clip, const float* grew_dev, float* rew_acc_dev, int64_t n, void* stream);
/* The same for a sweep of K members (K divides rew_floats and n): reward element i is member i / (rew_floats / K)'s and
 * is scaled with the device floats reward_norm[k] / reward_clip[k] (0 = off), with tscl_device_transition's arithmetic. */
int tscl_device_transition_g(tscl_handle* h, const float* rew_dev, float* rew_hist_dev, int64_t rew_floats,
                             const float* reward_norm, const float* reward_clip, int32_t K, const float* grew_dev,
                             float* rew_acc_dev, int64_t n, void* stream);
/* cudaMemcpyAsync on a caller-supplied stream; kind 1 = host->device, 2 = device->host, 3 = device->device */
int tscl_memcpy_async(tscl_handle* h, void* dst, const void* src, int64_t bytes, int32_t kind, void* stream);
/* dX = dZ . Wx^T as a stand-alone streaming product (the shipping path; reference: tf.gradients through
 * `tf.matmul(x, wx)`, agents/utils.py:106): dz_bf16 [2A][M][256], wxt_bf16 from tscl_pack_wxt, dx_bf16 [2A][M][dx] out.
 * Warp-specialised wgmma kernel (cp.async loaders -> 128B-swizzled operand stages, double-buffered accumulator tiles, bulk-copy stores).
 * dx must be a multiple of 16, <= 224 for the shared-memory budget. */
int tscl_dx_tc(tscl_handle* h, const void* dz_bf16, const void* wxt_bf16, void* dx_bf16, int64_t M, void* stream);
/* tscl_dx_tc followed by tscl_fc_bwd_tc in one pass, without dX in memory (the shipping path for dx = 128, 160, 192, 224):
 * grads[fc blocks] += obs^T . (bf16(dz_bf16 . Wx^T) * (x_bf16 > 0)) and the bias sums, rows as tscl_fc_bwd_tc.
 * x_bf16 [2A][M][dx] (one chunk of the bf16 activation store), dz_bf16 [2A][M][256], both 16-byte aligned (read through
 * tensor maps); wxt_bf16 from tscl_pack_wxt.  The masked bf16 dX has the bits of the two-call path; only the order of
 * the fp32 sums differs.  M < 2^31 - 128. */
int tscl_dx_fc_bwd_tc(tscl_handle* h, const float* obs, const void* x_bf16, const void* dz_bf16, const void* wxt_bf16,
                      int64_t M, int64_t rows_per_t, int64_t stride_t, float* grads, void* stream);
/* gates_bf16 / c_bf16 (both or neither): read gate activations and c_t straight from one chunk of the bf16
 * activation store instead of ZG / C (ZG is then write-only: it receives dZ).
 * dz_bf16 (optional): also write dZ as bf16 [2A][T*Rc][256]; with all three bf16 pointers ZG may be NULL. */

/* One replica chunk of the bf16 activation store ([2A][T][rc][w] contiguous) -> fp32 work buffers X, ZG (gates),
 * C, H and Hp[t] = (1 - done[t]) * (t > 0 ? H[t-1] : h0[:, r0 + r]).  Every output may be NULL (skipped): the
 * tensor-core kernels read the store themselves. */
int tscl_unpack_store(tscl_handle* h, const void* st_x, const void* st_g, const void* st_c, const void* st_h, float* X,
                      float* ZG, float* C, float* H, float* Hp, const float* h0, const float* done, int32_t T,
                      int64_t rc, int64_t ld_state, int64_t r0, void* stream);

/* Tools only (scripts/profile_policy_phases.py): per-phase clock64 sums of tscl_policy_step_v2 are added to 8 uint64
 * device counters while the pointer is set (NULL = off; a separate instantiation of the kernel, the hot one is unchanged). */
int tscl_debug_policy_prof(void* counters_dev);
/* same for the store-path BPTT kernel: the first 4 of 8 counters (operand wait | smem->regs + cell backward | MMA issue ->
 * wait | dZ store), summed over the warpgroups; NULL switches profiling off */
int tscl_debug_bptt_prof(void* counters_dev);

/* Per-agent clip_by_global_norm(max_norm) + RMSProp step (TF1 semantics).  agent_of [n_params] u8.
 * norms [A] receives the pre-clip global norms. */
int tscl_clip_rmsprop(tscl_handle* h, float* params, float* grads, float* ms, const uint8_t* agent_of,
                      float max_norm, float lr, float alpha, float eps, float* norms, void* stream);

/* ---- fused tensor-core policy forward (wgmma), csrc/tsc_policy_tc.cu -------------------------
 * tscl_pack_weights: per unit, [Wx;Wh] -> bf16 UMMA operand image [(dx+h)/8][4h][8] followed by the
 *   block-diagonal fc image [8][dx][8]; wpack holds 2A such records (call after every optimizer step).
 * tscl_policy_step: one decision for R replicas and all agents in ONE kernel: fc front end, gate GEMM on
 *   the tensor cores (bf16 operands, fp32 accumulation), LSTM cell, heads, softmax, sampling.
 *   Replaces LstmACPolicy.forward / FPLstmACPolicy.forward for a whole batch (agents/policies.py:125-136).
 *   c_in/h_in/c_out/h_out [2A][R][h] (out may alias in); pi [R][A][max_na]; val [R][A]; act [R][A] or NULL;
 *   zdbg [2A][R][4h] raw gate accumulators (debug) or NULL; swap_lbo_sbo: debug switch, pass 0. */
int tscl_pack_weights(tscl_handle* h, const float* params, void* wpack_bf16, void* stream);
int tscl_policy_step(tscl_handle* h, const float* params, const void* wpack_bf16, const float* obs, int64_t R,
                     const float* c_in, const float* h_in, float* c_out, float* h_out, float* pi, float* val,
                     int32_t* act, int32_t done, uint64_t seed, int64_t step, int64_t replica0, float* zdbg,
                     int32_t swap_lbo_sbo, void* stream);

/* v2 of the fused forward: the fc front end runs on the tensor cores as well (observation slice tile x
 * block-diagonal fc weights -> accumulator -> relu/bf16 -> A operand).  Same arguments as tscl_policy_step
 * (without the descriptor debug switch); needs dx % 32 == 0.  wpack must come from tscl_pack_weights. */
int tscl_policy_step_v2(tscl_handle* h, const float* params, const void* wpack_bf16, const float* obs, int64_t R,
                        const float* c_in, const float* h_in, float* c_out, float* h_out, float* pi, float* val,
                        int32_t* act, int32_t done, uint64_t seed, int64_t step, int64_t replica0, float* zdbg,
                        void* st_x, void* st_g, void* st_c, void* st_h, int32_t t, int32_t T, int64_t rc, void* stream);
/* Replica-range form: R rows starting at absolute replica row0 of a batch of ld_state replicas.  Every pointer is the
 * base of the range's slice (obs + row0 * n_obs, c_in + row0 * h, pi + row0 * A * max_na, ...; the st_* pointers stay
 * the bases of the whole store); the per-unit state arrays keep ld_state rows per unit.  ld_state = 0: plain call. */
int tscl_policy_step_v2r(tscl_handle* h, const float* params, const void* wpack_bf16, const float* obs, int64_t R,
                         const float* c_in, const float* h_in, float* c_out, float* h_out, float* pi, float* val,
                         int32_t* act, int32_t done, uint64_t seed, int64_t step, int64_t replica0, float* zdbg,
                         void* st_x, void* st_g, void* st_c, void* st_h, int32_t t, int32_t T, int64_t rc,
                         int64_t ld_state, int64_t row0, void* stream);
/* Population form: one launch for K members of one agent with Rm replicas each (Rm a multiple of 64), rows
 * k*Rm .. (k+1)*Rm - 1 of the shared obs / state / pi / val / act / store arrays belonging to member k.  Member k's
 * parameters are params + k*p_stride (floats) and its packed image wpack + k*wp_stride (bf16 elements, 2A records each);
 * it samples with seeds[k] (device array of K uint64, required also without act: every block reads its
 * member's seed) and replica index r - k*Rm, so its outputs are bit-identical to
 * tscl_policy_step_v2 on its own slice with seed seeds[k] and replica0 = 0.  State [2A][K*Rm][h]; store as in
 * tscl_policy_step_v2 over K*Rm rows, with rc dividing Rm.  Work items are (member, unit, 64-replica tile). */
int tscl_policy_step_v2g(tscl_handle* h, const float* params, int64_t p_stride, const void* wpack_bf16,
                         int64_t wp_stride, const float* obs, int32_t K, int64_t Rm, const float* c_in,
                         const float* h_in, float* c_out, float* h_out, float* pi, float* val, int32_t* act,
                         int32_t done, const uint64_t* seeds, int64_t step, void* st_x, void* st_g, void* st_c,
                         void* st_h, int32_t t, int32_t T, int64_t rc, void* stream);
/* pi-only form of the v2 forward for test-mode evaluation (reference utils.py:Evaluator, LstmACPolicy.forward(.., 'p')):
 * the same kernel restricted to the A pi units (V units are never touched), bit-identical pi / c / h to the pi units of
 * tscl_policy_step_v2.  State is compact: c_in/h_in/c_out/h_out [A][ld_state or R][h] (out may alias in); pi
 * [R][A][max_na]; act [R][A] or NULL.  act_mode 0 = the counter-RNG sample of tscl_policy_step_v2 (seed, step,
 * replica0 + r, agent); 1 = the first maximum of the written pi (np.argmax).  ld_state / row0: replica-range form as in
 * tscl_policy_step_v2r (pointers are the range's slices); ld_state = 0: plain call. */
int tscl_policy_step_pi(tscl_handle* h, const float* params, const void* wpack_bf16, const float* obs, int64_t R,
                        const float* c_in, const float* h_in, float* c_out, float* h_out, float* pi, int32_t* act,
                        int32_t act_mode, int32_t done, uint64_t seed, int64_t step, int64_t replica0, int64_t ld_state,
                        int64_t row0, void* stream);
/* Grouped pi-only form: one launch for K members of one layout (the handle's), for evaluating several trained agents on
 * one simulator.  rows: device array of K + 1 ascending row boundaries, rows[0] = 0, rows[K] = R; member k owns rows
 * rows[k] .. rows[k+1] - 1 (any count >= 1: ragged, no padding) of obs [R][n_obs], pi [R][A][max_na], act [R][A] and the
 * compact state [A][R][h] (out may alias in).  Member k reads params + k*p_stride and wpack + k*wp_stride and samples
 * (act_mode 0) with seeds[k] (device array of K uint64) and its member-local replica r - rows[k]; act_mode 1 = first
 * argmax.  Member k's pi, c, h and act are bit-identical to tscl_policy_step_pi on its own slice with seed seeds[k] and
 * replica0 = 0.  Work items are (member, pi unit, 64-row tile of the member). */
int tscl_policy_step_pi_g(tscl_handle* h, const float* params, int64_t p_stride, const void* wpack_bf16, int64_t wp_stride,
                          const float* obs, int32_t K, const int64_t* rows, int64_t R, const float* c_in, const float* h_in,
                          float* c_out, float* h_out, float* pi, int32_t* act, int32_t act_mode, int32_t done,
                          const uint64_t* seeds, int64_t step, void* stream);
/* Deterministic action choice for the forwards without a fused pi-only kernel (fc policy, v1 LSTM forward):
 * act[r][a] = first j < n_a[a] with the largest pi[r][a][j]; pi [R][A][max_na], act [R][A]. */
int tscl_argmax_actions(tscl_handle* h, const float* pi, int64_t R, int32_t* act, void* stream);
/* st_x/st_g/st_c/st_h (all or none, may be NULL): bf16 activation store [R/rc][2A][T][rc][dx | 4h | h | h]
 * (replica-chunk major; rc must divide R) written at time index t — the relu'd fc outputs, the gate activations i,f,o,u, c_t and h_t — so that the update can
 * back-propagate through the rollout's own forward pass instead of recomputing it.
 * bf16 elements per unit in the packed weight image: ((dx+h)/8)*4h*8 + 8*dx*8 */

/* ---- IQL Q-network forward for test-mode evaluation, csrc/tsc_q.cu ------------------------------
 * The per-agent networks of the reference's value-based agents (agents/policies.py:341-389, variable names
 * agents/checkpoint.py), all agents and R replicas in one launch:
 *   model 0, LRQPolicy:   q = S.W_q + b_q                               S = the agent's n_s observation floats
 *   model 1, DeepQPolicy: h0 = relu(S[:, :n_s-n_w].W_fcw + b)           width n_fc  (num_fc)
 *                         h1 = relu(S[:, n_s-n_w:].W_fct + b)           width n_ft  (num_fc / 4), agents with n_w > 0
 *                         h  = relu([h0 | h1].W_fc0 + b)                width n_h   (num_h)
 *                         q  = h.W_q + b_q
 * Every tensor is row-major [in][out] at its per-agent offset (in floats) into one flat fp32 parameter vector; offsets of
 * layers a model does not have may be NULL.  fp32 FMAs throughout (no tensor cores), so that argmax ties resolve as in an
 * fp32 host forward.  Limits: max_na <= 8; dqn widths multiples of 16 with n_fc <= 128, n_ft <= 32, n_h <= 64. */
typedef struct tscl_qdims {
  int32_t n_agents;   /* A                                                          */
  int32_t n_obs;      /* row stride of the observation matrix                       */
  int32_t max_na;     /* row stride of q                                            */
  int32_t model;      /* 0 = lr, 1 = dqn                                            */
  int32_t n_fc, n_ft, n_h;  /* dqn layer widths (ignored for lr)                   */
  const int32_t* obs_off;   /* [A] first observation float of agent i               */
  const int32_t* n_s;       /* [A] observation floats of agent i (wave | wait)      */
  const int32_t* n_w;       /* [A] trailing wait floats of agent i (dqn: q_fct input) */
  const int32_t* n_a;       /* [A]                                                  */
  const int64_t* off_fcw_w; /* [A] [n_s-n_w][n_fc]  */ const int64_t* off_fcw_b; /* [A] [n_fc] */
  const int64_t* off_fct_w; /* [A] [n_w][n_ft]      */ const int64_t* off_fct_b; /* [A] [n_ft] */
  const int64_t* off_fc0_w; /* [A] [n_fc (+n_ft)][n_h] */ const int64_t* off_fc0_b; /* [A] [n_h] */
  const int64_t* off_q_w;   /* [A] [n_s or n_h][n_a] */ const int64_t* off_q_b;   /* [A] [n_a] */
  int64_t n_params;
} tscl_qdims;

typedef struct tscl_qhandle tscl_qhandle;

int tscl_q_create(const tscl_qdims* dims, int32_t device, tscl_qhandle** out);
int tscl_q_destroy(tscl_qhandle* h);
/* One decision of IQL.forward(obs, mode='act', stochastic) (agents/models.py:347-363) for R replicas:
 *   obs [R][n_obs] -> q [R][A][max_na] (zero padded), act [R][A].
 *   mode 0: act = the first maximum of q (np.argmax; policy types 'default' and 'deterministic', utils.py:221-225).
 *   mode 1: qs / np.sum(qs) and np.random.choice(n_a, p=qs): s = sum of q in index order, p_j = q_j / s, both fp32; the
 *           inverse CDF of p at the counter-hash uniform of tscl_heads keyed (seed, step, replica0 + r, agent): the first
 *           j with u < p_0 + .. + p_j, else n_a - 1.  A row where np.random.choice would raise (some p_j negative or not
 *           finite: mixed signs, s = 0 or non-finite) gets action 0, and bad_flag (int64, caller-initialised to -1, may
 *           be NULL) receives, as an unsigned atomic minimum, (replica0 + r) << 40 | (step & 0xFFFFFF) << 16 | agent: the
 *           failure the one-replica protocol, playing the replicas in order, meets first.  All-negative q is valid.
 * Replica-range form: pass obs + r0 * n_obs, q + r0 * A * max_na, act + r0 * A, R = n and replica0 = r0. */
int tscl_q_step(tscl_qhandle* h, const float* params, const float* obs, int64_t R, float* q, int32_t* act, int32_t mode,
                uint64_t seed, int64_t step, int64_t replica0, int64_t* bad_flag, void* stream);
/* Grouped form: one launch for K members of one Q layout (the handle's).  rows: device array of K + 1 ascending row
 * boundaries, rows[0] = 0, rows[K] = R; member k owns rows rows[k] .. rows[k+1] - 1 (ragged, any count >= 1) of obs, q
 * and act, reads params + k*p_stride and keys its mode-1 draws with seeds[k] (device, K uint64) and its member-local
 * replica r - rows[k].  bad_flags: NULL or a device array of K int64 (caller-initialised to -1); member k's failed
 * samples go into bad_flags[k] with its own key, member-local replica << 40 | (step & 0xFFFFFF) << 16 | agent, so the
 * member is the array index.  Member k's q, act and bad_flags[k] are bit-identical to tscl_q_step on its own slice with
 * seed seeds[k] and replica0 = 0.  CTAs cover (tile group, agent, member). */
int tscl_q_step_g(tscl_qhandle* h, const float* params, int64_t p_stride, const float* obs, int32_t K, const int64_t* rows,
                  int64_t R, float* q, int32_t* act, int32_t mode, const uint64_t* seeds, int64_t step,
                  int64_t* bad_flags, void* stream);

/* ---- IQL training (IQL.explore / add_transition / backward, agents/models.py:305-376), same handle ----------------
 * Replay ring of one rank's R replicas, slot-major, capacity B: s / s1 [B][R][n_obs] fp32, a [B][R][A] int8,
 * r [B][R][A] fp32 (already normalised and clipped), done [B][R] u8.  The learner owns the write position.
 *
 * Explore forward: act = the first maximum of q, replaced by floor(n_a * u2) (multiply-shift) when u < eps, u and u2
 * from the counter hash keyed (seed, step, replica0 + r, agent) (u2 from a second, salted stream).  Also writes act as
 * int8 into ring_a [R][A] and copies the observation rows into ring_s [R][n_obs] (either may be NULL). */
int tscl_q_explore(tscl_qhandle* h, const float* params, const float* obs, int64_t R, float* q, int32_t* act, float eps,
                   uint64_t seed, int64_t step, int64_t replica0, float* ring_s, int8_t* ring_a, void* stream);
/* random.sample(range(size), batch) for every (agent, replica): idx [A][R][batch] (int32), Floyd's algorithm with
 * multiply-shift draws keyed (seed, update, round, replica0 + r, agent, draw).  size >= batch. */
int tscl_q_sample(tscl_qhandle* h, int64_t R, int32_t batch, int32_t size, uint64_t seed, int64_t update, int32_t round,
                  int64_t replica0, int32_t* idx, void* stream);
/* One round of the TD loss for all agents: the rows idx[a][r][*] of the ring (pointers to slot 0), tq = done ? r :
 * r + gamma max q(s1), loss = inv_n sum (q(s)[a] - tq)^2 over this rank's rows.  grad [n_params + 3 A] receives the
 * weight gradients (flat layout) followed by three per-agent tails: the loss sums, inv_n sum q(s)[a] and inv_n sum tq;
 * reduced in a fixed order (bit-reproducible).  Summed over ranks, the tails are the global means. */
int tscl_q_td(tscl_qhandle* h, const float* params, const float* ring_s, const float* ring_s1, const int8_t* ring_a,
              const float* ring_r, const uint8_t* ring_done, const int32_t* idx, int64_t R, int32_t batch, float gamma,
              float inv_n, float* grad, void* stream);
/* Per agent: tf.clip_by_global_norm(max_grad_norm) of grad and the TF1 Adam step (b1 0.9, b2 0.999, eps 1e-8) with
 * lr_t = lr sqrt(1 - b2^t) / (1 - b1^t); loss_out [A] = grad's loss sums, norm_out [A] = the pre-clip norms.
 * rec_out (optional) [A][4]: per agent (loss, mean q, mean tq, pre-clip norm), the round's summaries. */
int tscl_q_adam(tscl_qhandle* h, float* params, const float* grad, float* adam_m, float* adam_v, float lr_t,
                float max_grad_norm, float* loss_out, float* norm_out, float* rec_out, void* stream);
/* IQL.add_transition's reward and done into one ring slot: ring_r [R][A] = clip(rew / reward_norm), ring_done [R] = done,
 * and rew_acc [R] += grew [R] (rew_acc may be NULL). */
int tscl_q_transition(tscl_qhandle* h, const float* rew, int64_t R, float reward_norm, float reward_clip, float* ring_r,
                      const float* grew, float* rew_acc, uint8_t* ring_done, int32_t done, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TSC_LEARN_H_ */
