/*
 * xb200.h - C-ABI of the H100-native rollout->update hot path for agi-brain/xuance (v1.4.4 @ 4f0b05b).
 *
 * The reference has NO native/FFI layer (SURVEY.md section 8b): its hot path is Python classes resolved
 * through registries.  This header is therefore the boundary a maintainer would bind from those classes
 * (ctypes stubs in INTEGRATION.md); every entry point cites the reference code it replaces.
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless the name ends in _host
 *   - `stream` is a cudaStream_t passed as void*; every call is asynchronous on that stream, allocates
 *     nothing, and returns 0 on success, a negative XB_E* code for a rejected argument, or a positive
 *     cudaError_t if the launch failed
 *   - row-major layouts; [N,T,...] buffers are the reference's `create_memory` layout
 *     (xuance/common/memory_tools.py:12-40) so that flat slot = env*T + step = the index handed to sample()
 *   - scalar fields (actions of a Discrete space, rewards, values, terminals, old_logp, returns, advantages)
 *     are float32, exactly as the reference stores them (memory_tools.py:15; SURVEY appendix B #1)
 */
#ifndef XB200_H_
#define XB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XB_OK 0
#define XB_EINVAL (-1)   /* bad size / null pointer */
#define XB_EALIGN (-2)   /* pointer or row size not aligned as the entry point requires */
#define XB_ERANGE (-3)   /* argument outside the supported range (documented per call) */

/* observation output formats of xb_gather_obs */
#define XB_OBS_U8 0        /* byte copy (bit-exact gather)                                          */
#define XB_OBS_F32_NHWC 1  /* float32 = u8/255.0 (correctly rounded division), same element order   */
#define XB_OBS_F32_NCHW 2  /* float32 = u8/255.0, channel planes (HWC -> CHW per row)               */
#define XB_OBS_BF16_NHWC 3 /* bfloat16(round-to-nearest-even of u8/255.0f), same element order      */
#define XB_OBS_F16_NHWC 4  /* float16 (rn) of u8/255.0f, same element order                         */

int xb_version(void);
const char *xb_error_string(int code);
/* sm_count, compute capability of the current device; returns cudaError on failure */
int xb_device_info(int *sm_count, int *cc_major, int *cc_minor);

/* ---------------------------------------------------------------- K1: rollout / replay store ---------
 * Replaces store_element(): `memory[:, ptr] = data`  (memory_tools.py:43-61), as used by
 * DummyOnPolicyBuffer.store :232-240, DummyOffPolicyBuffer.store :364-372, PerOffPolicyBuffer.store :537-543.
 * rows:    dst[N, T, row_bytes] (bytes)  <- src[N, row_bytes]   at step t      (row_bytes % 4 == 0)
 * scalars: dst[F, N, T] (float32)        <- src[F, N]           at step t      (F may be 0)
 * One launch does both; pass rows_dst = NULL to store scalars only. */
int xb_rollout_store(void *rows_dst, const void *rows_src, int64_t row_bytes,
                     float *scal_dst, const float *scal_src, int F,
                     int N, int T, int t, void *stream);
/* xb_rollout_store with a per-row step: row n goes to step step[n] (device int32[N]); rows whose step is outside
 * [0, T) are not written.  The per-env episode staging of MARL_OnPolicyBuffer_RNN, where each env sits at its own
 * episode step (memory_tools_marl.py:461-470). */
int xb_rollout_store_at(void *rows_dst, const void *rows_src, int64_t row_bytes,
                        float *scal_dst, const float *scal_src, int F,
                        int N, int T, const int32_t *step, void *stream);

/* ---------------------------------------------------------------- K2: GAE / returns scan -------------
 * Replaces DummyOnPolicyBuffer.finish_path (memory_tools.py:242-265) for ALL envs and ALL path segments of a
 * rollout in one launch.  rew/val/term/adv/ret are [N,T] float32.  seg_end[N,T] (uint8) marks the last step
 * of each finished path, bootstrap[N,T] holds the `val` passed to finish_path at that step, covered[N] is the
 * number of leading steps of env i that belong to finished paths (steps >= covered[i] get adv = ret = 0, as in
 * the reference where they are never written).
 *   use_gae=1:  delta_t = r_t + (1-d_t)*gamma*V_{t+1} - V_t ;  A_t = delta_t + (1-d_t)*gamma*lam*A_{t+1}
 *               ret_t = A_t + V_t   (float32; warp-level scan of the affine maps, so +-few ulp of the loop)
 *   use_gae=0:  ret_t = r_t + gamma*ret_{t+1} (float64 scan, as scipy.lfilter), A_t = r_t + gamma*V_{t+1} - V_t */
int xb_gae_scan(const float *rew, const float *val, const float *term,
                const uint8_t *seg_end, const float *bootstrap, const int32_t *covered,
                float *adv, float *ret, int N, int T, float gamma, float lam, int use_gae, void *stream);

/* K2 for the multi-agent on-policy buffer (MARL_OnPolicyBuffer.finish_path, memory_tools_marl.py:208-236): rows are
 * (env, agent) pairs, [N,T] fields as for xb_gae_scan, start[N] / covered[N] (int32, nullable = 0 / T): only steps in
 * [start, covered) are written.  With a ValueNorm state (running_mean, running_mean_sq, debiasing_term: device
 * scalars, all or none) the stored values and, for use_gae, the bootstrap are denormalised with the state as it is
 * when the kernel runs (float32, value_norm.py:65-75); without one they are used as stored.
 *   use_gae=1: delta_t = r_t + (1-d_t)*gamma*V'_{t+1} - V'_t; A_t = delta_t + (1-d_t)*gamma*lam*A_{t+1} in float64
 *              (warp scan of affine maps), ret_t = float32(A_t + V'_t)
 *   use_gae=0: ret_t = float32(r_t + (1-d_t)*gamma*ret_{t+1}) step by step, ret at the segment end's successor = the
 *              raw bootstrap
 *   both:      adv_t = ret_t - V'_t in float32.
 * Every path is float32 as above.  The reference computes a path whose bootstrap is the Python float 0.0 (a terminal
 * step) in float64 (np.append promotes it): its non-GAE returns are not rounded step by step and its advantages
 * denormalise in float64 - a few ulp from this (DESIGN.md section 4). */
int xb_gae_scan_vn(const float *rew, const float *val, const float *term, const uint8_t *seg_end, const float *bootstrap,
                   const int32_t *start, const int32_t *covered, float *adv, float *ret, int N, int T, double gamma,
                   double lam, int use_gae, const float *running_mean, const float *running_mean_sq,
                   const float *debiasing_term, void *stream);

/* ---------------------------------------------------------------- K3: minibatch gather ---------------
 * Replaces sample_batch(): `memory[(env_idx, step_idx)]` (memory_tools.py:64-84) as used by
 * DummyOnPolicyBuffer.sample :267-287 and the replay buffers' sample().  idx[B] are flat slots (env*T+step);
 * idx == NULL means identity (rows 0..B-1), which turns xb_gather_obs into the u8 -> float preprocessing of
 * AC_CNN_Atari.forward / Basic_CNN.forward (xuance/torch/rl_models/representations/cnn.py:45-50,98-102).
 * xb_gather_rows: dst[B,row_bytes] <- src[idx[b]]            (row_bytes % 4 == 0; bulk-async path if % 16 == 0)
 * xb_gather_obs : dst[B, H*W*C] in `format` <- u8 src rows; H*W*C % 16 == 0; NCHW needs C == 4, W % 4 == 0. */
int xb_gather_rows(const void *src, const int64_t *idx, int64_t B, int64_t row_bytes, void *dst, void *stream);
int xb_gather_obs(const uint8_t *src, const int64_t *idx, int64_t B, int H, int W, int C,
                  void *dst, int format, void *stream);

/* Gathers F float32 fields fields[F, slots] at idx[B] into out[F, B]; if adv_field >= 0 that field is
 * replaced by (x - mean) / (std + 1e-8) with the POPULATION std over the B gathered values
 * (memory_tools.py:280-282).  stats_out[2] receives (mean, std).  scratch: >= xb_scratch_doubles() doubles
 * plus one trailing int32 counter, zeroed once by the caller (the kernels re-zero it).
 * world-size > 1 is handled above the ABI (all-reduce of the partial sums). */
int64_t xb_scratch_doubles(void);
int xb_gather_scalars(const float *fields, int64_t slots, const int64_t *idx, int64_t B, int F,
                      float *out, int adv_field, float *stats_out, double *scratch, void *stream);
/* adv[b] <- (adv[b] - stats[0]) / (stats[1] + 1e-8) with GIVEN statistics: the second half of memory_tools.py:281-282 for a
 * minibatch that is sharded over ranks (its global mean / population std are all-reduced once per epoch). */
int xb_adv_normalize(float *adv, int64_t B, const float *stats, void *stream);

/* ---------------------------------------------------------------- K4: fused PPO-Clip loss fwd+bwd ----
 * Replaces ppo_learner.py:46-60 plus the autograd backward of those lines down to (logits, value):
 *   logp = log_softmax(logits)[a]; ratio = exp(logp - old_logp)
 *   a_loss = -mean(min(clamp(ratio,1-eps,1+eps)*adv, adv*ratio)); c_loss = mean((v-ret)^2); e = mean(H)
 *   loss = a_loss - ent_coef*e + vf_coef*c_loss
 * Writes dlogits[B,A] = dloss/dlogits, dvalue[B] = dloss/dvalue (means over B_total >= B rows so a
 * rank-local shard of a global minibatch produces correctly scaled gradients) and
 * stats[8] = {a_loss, c_loss, entropy, mean(v), clip_fraction, loss, 0, 0} * (B/B_total weighting applied,
 * i.e. sums over the local rows divided by B_total).  actions are float32 (reference quirk).  A <= 64.
 * loss_kind 0 = PPO-Clip (above); 1 = plain policy gradient a_loss = -mean(adv*logp) (old_logp unused): A2C
 * (a2c_learner.py:46-52) with adv = advantages, PG (pg_learner.py:44-47) with adv = returns and vf_coef = 0. */
int xb_ppo_loss_fwd_bwd(const float *logits, const float *value, const float *actions,
                        const float *old_logp, const float *adv, const float *ret,
                        int64_t B, int A, int64_t B_total, float clip_range, float vf_coef, float ent_coef,
                        int loss_kind, float *dlogits, float *dvalue, float *stats, double *scratch, void *stream);

/* ---------------------------------------------------------------- K4G: fused Gaussian PPO loss fwd+bwd -
 * ppo_learner.py:46-60 (and a2c_learner.py:46-52, pg_learner.py:44-47 with loss_kind 1) for a DiagGaussianDistribution
 * (modules/distributions.py:165-197): Normal(mu, exp(log_std)), log_prob and entropy summed over the D components:
 *   logp_b = sum_j [-(x-mu)^2/(2 sigma^2) - log_std_j - log sqrt(2 pi)]  (j in index order)
 *   H_b    = sum_j [1/2 + log(2 pi)/2 + log_std_j]
 * ratio, clamp, minimum, tie split, clamp boundary, loss_kind, B_total scaling and stats[8] exactly as K4.
 * Writes dmu[B,D], dvalue[B] and dlog_std[D] = the sum over the local rows divided by B_total (a SUM all-reduce of
 * the shards gives the global gradient).  mu / actions [B,D] float32, log_std [D]; 1 <= D <= 64 (else XB_ERANGE).
 * ws: caller workspace of >= xb_ppo_gauss_ws_doubles(B, D) doubles (D * min(ceil(B/256), 2048); 64 * 2048 doubles
 * always suffice) for the per-block column partials of dlog_std, which are added in block order: dlog_std is
 * bit-identical from launch to launch.  ws_doubles is its size (XB_EINVAL if too small); scratch as for K4. */
int64_t xb_ppo_gauss_ws_doubles(int64_t B, int D);
int xb_ppo_gauss_loss_fwd_bwd(const float *mu, const float *log_std, const float *value, const float *actions,
                              const float *old_logp, const float *adv, const float *ret, int64_t B, int D,
                              int64_t B_total, float clip_range, float vf_coef, float ent_coef, int loss_kind,
                              float *dmu, float *dlog_std, float *dvalue, float *stats, double *scratch, double *ws,
                              int64_t ws_doubles, void *stream);

/* ---------------------------------------------------------------- K4P: fused PPG auxiliary loss fwd+bwd -
 * ppg_learner.py:114-148 (update_auxiliary_critic) plus the autograd backward of its loss down to the network outputs:
 *   aux_loss = MSE(v.detach(), aux_v); kl_loss = mean(KL(pi_new || pi_old)); value_loss = MSE(v, R)
 *   loss = aux_loss + kl_beta * kl_loss + value_loss
 * dvalue[B] = 2 (v - R) / B_total, daux[B] = 2 (aux_v - v) / B_total (aux_loss reaches aux_v only), means over
 * B_total >= B rows as K4, so the SUM of the shards' outputs is the global result.  stats[8] = {aux_loss, kl_loss,
 * value_loss, loss, mean(v), 0, 0, 0}.  scratch as for K4.  One warp per row; no allocation; graph-capturable.
 * xb_ppg_aux_loss_fwd_bwd (Categorical): logits / old_logits [B, A] raw (each side is log-softmax normalised in the
 *   kernel, as Categorical(logits=) does), 1 <= A <= 64 (else XB_ERANGE).  dlogits = kl_beta * dKL/dlogits with torch's
 *   zero-probability rules (a term is +inf where q = 0 and 0 where p = 0, and those terms pass no gradient; a -inf logit
 *   on either side makes its row's gradient NaN, as autograd's 0 * inf does).  logits, old_logits and dlogits are NULL
 *   together: then only value_loss is formed (update_critic, ppg_learner.py:90-112: critic-loss = stats[2]).
 *   aux_value and daux are NULL together (aux_loss = 0).
 * xb_ppg_aux_gauss_loss_fwd_bwd (DiagGaussian): Normal(mu, exp(log_std)) against Normal(old_mu, exp(old_log_std)),
 *   mu / old_mu [B, D], log_std / old_log_std [D], 1 <= D <= 64 (else XB_ERANGE); kl_loss is the mean over B_total * D
 *   terms.  dmu [B, D]; dlog_std [D] = the sum over the local rows (the term depends on the column only: formed as B
 *   times it in double, bit-identical).  Every pointer is required. */
int xb_ppg_aux_loss_fwd_bwd(const float *logits, const float *old_logits, const float *value, const float *aux_value,
                            const float *ret, int64_t B, int A, int64_t B_total, float kl_beta, float *dlogits,
                            float *dvalue, float *daux, float *stats, double *scratch, void *stream);
int xb_ppg_aux_gauss_loss_fwd_bwd(const float *mu, const float *log_std, const float *old_mu, const float *old_log_std,
                                  const float *value, const float *aux_value, const float *ret, int64_t B, int D,
                                  int64_t B_total, float kl_beta, float *dmu, float *dlog_std, float *dvalue,
                                  float *daux, float *stats, double *scratch, void *stream);

/* ---------------------------------------------------------------- K4M: fused MAPPO loss fwd+bwd -------
 * Replaces mappo_learner.py:55-113 (one parameter-sharing group, feed-forward actor and critic, Discrete actions) plus
 * the autograd backward of those lines down to (logits, value).  One row = one agent at one env step.
 * xb_mappo_prepare    : block[4] (float64) = {sum mask, sum ret, sum ret^2, 0} over the R local rows (deterministic
 *                       two-level reduction); SUM-all-reduce it when the minibatch is sharded.
 * xb_value_norm_update: ValueNorm.update + running_mean_var (xuance/torch/utils/value_norm.py:29-52) in float32, in
 *                       torch's operation order: x <- x*beta + m*(1-beta) for running_mean / running_mean_sq with the
 *                       batch moments m = block[1] / R_total, block[2] / R_total (float64 quotients rounded to float32),
 *                       debiasing_term <- d*beta + (1-beta); mean = rm / max(d, 1e-5), var = max(rmsq / max(d, 1e-5) -
 *                       mean^2, 1e-2); writes the state in place and mean_std[2] = {mean, sqrt(var)}.  One thread.
 * xb_mappo_loss_fwd_bwd: logits[R,A] with avail[R, avail_ld] (uint8, nullable; 0 = unavailable: the logit counts as
 *                       -1e10 and its gradient is exactly 0, actor_head.py:40); M = prep[0] is the GLOBAL sum of the
 *                       agent mask:
 *     a_loss = -sum(min(ratio*adv, clip(ratio, 1-eps, 1+eps)*adv) * mask) / M       (K4's tie and clamp rules)
 *     target = vn ? (ret - vn[0]) / vn[1] : ret                                        (vn: mean_std, nullable)
 *     L(d)   = huber_delta > 0 ? HuberLoss(delta)(d) : d^2
 *     value_clip_range > 0: lc = max(L(v - target), L(v_old + clamp(v - v_old, -c, c) - target))  (ties split 1/2,
 *                           clamp inclusive);  else lc = L(v - target)
 *     c_loss = sum(lc * mask) / M;  e = sum(H * mask) / M;  loss = a_loss + vf_coef*c_loss - ent_coef*e
 * Writes dlogits[R,A], dvalue[R] and stats[8] = {a_loss, c_loss, e, predict_value = sum(v) / R_total (unmasked, as the
 * reference logs it), loss, 0, 0, 0}, each the local rows' share (a SUM all-reduce of the shards gives the global
 * value).  M = 0 gives 0/0 = NaN statistics and gradients, as in the reference.  actions are float32; A <= 64 (else
 * XB_ERANGE); old_value may be NULL when value_clip_range <= 0.  scratch as for K4. */
int xb_mappo_prepare(const float *mask, const float *ret, int64_t R, double *block, double *scratch, void *stream);
int xb_value_norm_update(float *running_mean, float *running_mean_sq, float *debiasing_term, const double *block,
                         int64_t R_total, double beta, float *mean_std, void *stream);
int xb_mappo_loss_fwd_bwd(const float *logits, const uint8_t *avail, int avail_ld, const float *actions,
                          const float *old_logp, const float *adv, const float *value, const float *old_value,
                          const float *ret, const float *mask, const float *vn, const double *prep, int64_t R, int A,
                          int64_t R_total, float clip_range, float value_clip_range, float huber_delta, float vf_coef,
                          float ent_coef, float *dlogits, float *dvalue, float *stats, double *scratch, void *stream);

/* ---------------------------------------------------------------- K4V: fused VDAC / IAC loss fwd+bwd --
 * Replaces vdac_learner.py:53-126 and iac_learner.py:206-254 (one parameter-sharing group, Discrete actions) plus the
 * autograd backward of those lines down to (logits, value), with the value mixing and its agent reduction fused in.
 * Rows are agent steps in the episode buffer's (b, i, t) order, r = (b*n + i)*T + t, R = B*n*T (T = 1: feed-forward
 * batches).  prep and vn come from xb_mappo_prepare / xb_value_norm_update (K4M), unchanged.
 *     a_loss = -sum(adv * log pi(a) * mask) / M;   e = sum(H * mask) / M;   M = prep[0], the GLOBAL sum of the mask
 *     masked logits (avail[r, a] == 0) count as -1e10 and get exactly 0 gradient (actor_head.py:40), as in K4M
 *     c_loss = sum(lc(pred_r) * mask) / M with K4M's value term lc (vn target, Huber or square, inclusive clamp, ties
 *              split 1/2);   loss = a_loss + vf_coef*c_loss - ent_coef*e
 * The prediction pred_r of row r depends on mix_mode:
 *     0 independent (IAC): pred_r = value[r]; dvalue[R].
 *     1 VDN: value[R] holds V_i; V_tot(b, t) = sum_i V_i (agents in index order); dvalue[R] gets dV_i = dV_tot(b, t).
 *     2 external mixer (QMIX): value[B*T] is V_tot(b, t) at b*T + t; dvalue[B*T] = dL/dV_tot.
 *     row_order (modes 1, 2): 0 pairs V_tot(b, t) with rows (b, i, t) for every i; 1 reproduces the reference's
 *     use_rnn pairing, where row r reads V_tot at index floor(r / n) of the b*T + t order (DESIGN.md section 4); the two
 *     coincide at T = 1.  dV_tot sums the n rows paired with it, in a fixed order.
 * stats[8] = {a_loss, c_loss, e, predict_value = sum_r pred_r / R_total (unmasked, as the reference logs it: for VDAC the
 * mean of V_tot repeated n times), loss, 0, 0, 0}, each the local rows' share (a SUM all-reduce of the shards gives the
 * global value).  No float atomics: the outputs are bit-identical across launches.  M = 0 gives NaN, as in the
 * reference.  1 <= A <= 64 and 1 <= n <= 32 (else XB_ERANGE); R must be a multiple of n*T; actions are float32;
 * old_value may be NULL when value_clip_range <= 0.  scratch as for K4. */
int xb_vdac_loss_fwd_bwd(const float *logits, const uint8_t *avail, int avail_ld, const float *actions, const float *adv,
                         const float *value, const float *old_value, const float *ret, const float *mask,
                         const float *vn, const double *prep, int64_t R, int A, int n, int T, int mix_mode,
                         int row_order, int64_t R_total, float value_clip_range, float huber_delta, float vf_coef,
                         float ent_coef, float *dlogits, float *dvalue, float *stats, double *scratch, void *stream);

/* ---------------------------------------------------------------- K4C: COMA critic input, loss fwd+bwd, acting --
 * Replaces coma_learner.py:53-137, the critic-input assembly of centralized_critics.py:259-286 and the epsilon-mixed
 * acting of actor_critic.py:279-295 / coma_agents.py:226-258 (one parameter-sharing group, Discrete actions).  Rows are
 * agent steps in the episode buffer's (b, i, t) order, r = (b*n + i)*T + t, R = B*n*T.  Actions are float32 integers.
 * xb_coma_critic_input: out[R, S + F + n*A] with row r = [state[b, t, 0..S) | feat[r, 0..F) | joint one-hot of the n
 *     agents' actions at (b, t), agent-major, with agent i's own A-block zeroed] from state [B,T,S], feat [R,F] and
 *     actions [B,n,T].  Copies and 0 / 1 only, so the rows are bit-exact; an action outside [0, A) sets no bit.  Its
 *     backward is the feature slice of the output gradient (no kernel).  1 <= A <= 64, 1 <= n <= 32 (else XB_ERANGE).
 * xb_coma_loss_fwd_bwd: logits[R,A] with avail[R, avail_ld] (uint8, nullable: use_actions_mask), q[R,A] the critic's
 *     Q, eps[1] (DEVICE scalar: a captured graph stays valid while epsilon decays), M = prep[0] from xb_mappo_prepare
 *     (the GLOBAL sum of the mask):
 *     p = softmax(z), z = logits with unavailable entries at -1e10;  q_mix = (1 - eps) p + eps / A;
 *     pi = q_mix * av / sum(q_mix * av)  (av = 1 without avail);  baseline = sum_a pi_a Q_a;
 *     adv = Q[a] - baseline (detached);  loss_a = -sum(adv * log pi[a] * mask) / M;
 *     loss_c = sum(((Q[a] - ret) * mask)^2) / M
 *     dlogits[R,A] = d loss_a / d logits, exactly 0 at unavailable entries; a taken action with pi[a] = 0 gives
 *     log pi[a] = -inf and NaN at the row's available entries, as autograd of the reference does.
 *     dq[R,A] = d loss_c / d Q, nonzero only at the taken action.
 *     stats[8] = {loss_a, loss_c, advantage = sum(adv) / R_total (unmasked, as the reference logs it), 0, 0, 0, 0, 0},
 *     each the local rows' share (a SUM all-reduce of the shards gives the global value).  No float atomics: outputs
 *     are bit-identical across launches.  M = 0 gives NaN, as in the reference.  1 <= A <= 64 (else XB_ERANGE).
 *     scratch as for K4.
 * xb_coma_act: the acting distribution over logits[N,A]: pi = q_mix / sum(q_mix) with eps[1] on the device (eps NULL:
 *     no mix, the reference's test_mode).  uniforms != NULL: a = min{i : u < pi_0 + .. + pi_i} (the last index with
 *     pi_i > 0 if rounding leaves the total below u); else the first arg-max of pi.  After the mix an unavailable action
 *     has probability eps / A and can be drawn, as in the reference.  Outputs (each nullable, at least one):
 *     actions_f32[N], actions_i32[N], logp[N] = log pi[a].  A <= 64 (else XB_ERANGE). */
int xb_coma_critic_input(const float *state, const float *feat, const float *actions, int B, int n, int T, int S, int F,
                         int A, float *out, void *stream);
int xb_coma_loss_fwd_bwd(const float *logits, const uint8_t *avail, int avail_ld, const float *q, const float *actions,
                         const float *ret, const float *mask, const float *eps, const double *prep, int64_t R, int A,
                         int64_t R_total, float *dlogits, float *dq, float *stats, double *scratch, void *stream);
int xb_coma_act(const float *logits, const uint8_t *avail, int avail_ld, const float *eps, const float *uniforms, int N,
                int A, float *actions_f32, int32_t *actions_i32, float *logp, void *stream);

/* ---------------------------------------------------------------- K5: prioritized-replay trees -------
 * Replaces SumSegmentTree/MinSegmentTree (xuance/common/segtree_tool.py:4-220) and their use in
 * PerOffPolicyBuffer (memory_tools.py:505-598).  One (sum,min) pair PER ENV, float32 nodes, heap layout
 * tree[env][2*cap] (node 1 = root, leaves at cap..2cap-1); parents are fl32(l+r) / min(l,r).
 * insert : leaf[ptr] = max_prio[env]^alpha in both trees for every env           (:545-548)
 * sample : per env, k stratified draws: p_total = sum(0,size-1) with the reference's association order,
 *          mass_j = fl(fl(u_j*seg) + fl(j*seg)), find_prefixsum_idx; weights = p_j/p_min computed as the
 *          reference does (:563-572); u[N,k] float32 uniforms supplied by the caller
 *          outputs: step_out[N,k] int64, flat_out[N*k] int64 (= env*S + step), w_out[N,k] float64
 * update : leaf = p^alpha (p==0 -> 1e-8), later duplicates win, parents recomputed, max_prio updated (:588-598) */
/* out[i] = x[i]^y evaluated exactly as glibc 2.39 powf does (the routine numpy's float32 ** python-float calls, i.e.
 * what memory_tools.py:547,596 evaluate); exported so the parity tests can check the restatement on its own. */
int xb_powf_libm(const float *x, float y, float *out, int64_t n, void *stream);
int xb_per_insert(float *sum_tree, float *min_tree, float *max_prio, int N, int cap, int ptr, float alpha,
                  void *stream);
int xb_per_sample(const float *sum_tree, const float *min_tree, const float *u, int N, int cap, int size,
                  int k, int64_t S, float size_pow_neg_beta,
                  int64_t *step_out, int64_t *flat_out, double *w_out, void *stream);
int xb_per_update(float *sum_tree, float *min_tree, float *max_prio, const int64_t *idx, const float *prio,
                  int N, int cap, int k, float alpha, void *stream);

/* ---------------------------------------------------------------- K6: DQN TD target + loss fwd+bwd ---
 * Replaces dqn_learner.py:41-46 / perdqn_learner.py:44-50: predictQ = Q[b, a_b]; y = r + gamma*(1-d)*max_a Q'
 * loss = mean((predictQ - y)^2); dq[B,A] = dloss/dQ; td[B] = y - predictQ; stats[4] = {loss, mean predictQ,0,0}
 * (sums over local rows / B_total).  q_sel != NULL selects double-Q (ddqn_learner.py:39-44): q_sel[B,A] are the EVAL
 * network's values at the next observation, y uses q_next[b, argmax_a q_sel[b,a]] instead of the max. */
int xb_dqn_td_fwd_bwd(const float *q_eval, const float *q_next, const float *q_sel, const float *actions, const float *rew,
                      const float *term, int64_t B, int A, int64_t B_total, float gamma,
                      float *dq, float *td, float *stats, double *scratch, void *stream);

/* ---------------------------------------------------------------- K6Z: C51 / QR-DQN head tail + loss ---
 * z [B, A, N] float32 row-major is a head's raw output viewed as rows x actions x atoms (C51 logits) or quantiles
 * (QR).  Supported: 2 <= N <= 64 atoms / quantiles, 1 <= A <= 256 actions; anything else (and N < 2, where the
 * reference divides by zero) is XB_EINVAL, as are NULL required pointers and B <= 0.  One warp per row.
 * greedy: replaces deep_q_network.py:202-203 / 230-231 (C51: supports != NULL, Q = sum_i supports_i*softmax(z)_i) and
 *         :289-290 / 317-318 (QR: supports == NULL, Q = mean_i z_i) under no_grad.  Writes actions[B] int64, the first
 *         maximal index as torch.argmax; optional q[B, A] and (C51 only, else XB_EINVAL) probs[B, A, N].
 * c51   : replaces c51_learner.py:38-51 and its autograd to the eval logits.  Target action = the greedy action of
 *         z_next (the same device routine as greedy); Tz = clamp(rew + (gamma*z)*(1 - ter), v_min, v_max);
 *         target_i = sum_j p'_j * clamp(1 - |Tz_j - z_i| / delta_z, 0, 1); p = softmax(z_eval[b, a_b]);
 *         loss = mean_b -sum_i target_i*log(p_i + 1e-8).  Writes dlogits[B, A, N] (the taken row
 *         p*(g - sum p*g), g_i = ((-1/B_total)*target_i)/(p_i + 1e-8); the other rows 0), target_actions[B]
 *         int64, the optional target_dist[B, N] (the projected target, as the reference hands it to on_update_end;
 *         NULL skips it) and stats[4] = {Qloss, 0, 0, 0}.  supports[N] is the model's tensor.
 * qrdqn : replaces qrdqn_learner.py:40-48 and its autograd.  Target action = argmax_a mean(z_next[b, a]);
 *         y = rew + (gamma*theta')*(1 - ter); loss = mse(y, z_eval[b, a_b]) over B_total*N.  Writes dq[B, A, N]
 *         (2*(theta - y)/(B_total*N) on the taken row, 0 elsewhere), target_actions[B], stats[4] = {Qloss,0,0,0}.
 * Both losses: actions are float32 as stored; a row whose action is not in [0, A) gets zero gradient and makes Qloss
 * NaN.  Tz, the projection weights and the QR backup are bit-identical to torch's float32 expressions.  B_total >= B
 * rows scale the means (a SUM all-reduce of shards gives the global values); scratch as for K4. */
int xb_dist_greedy(const float *z, const float *supports, int64_t B, int A, int N, int64_t *actions, float *q,
                   float *probs, void *stream);
int xb_c51_loss_fwd_bwd(const float *z_eval, const float *z_next, const float *supports, const float *actions,
                        const float *rew, const float *ter, int64_t B, int A, int N, int64_t B_total, float gamma,
                        float v_min, float v_max, float delta_z, float *dlogits, int64_t *target_actions,
                        float *target_dist, float *stats, double *scratch, void *stream);
int xb_qrdqn_loss_fwd_bwd(const float *z_eval, const float *z_next, const float *actions, const float *rew,
                          const float *ter, int64_t B, int A, int N, int64_t B_total, float gamma, float *dq,
                          int64_t *target_actions, float *stats, double *scratch, void *stream);

/* ---------------------------------------------------------------- K9: QMIX selection / mixing / TD ----
 * Replaces, for one parameter-sharing group with use_rnn=True (episodes padded to T, `filled` mask):
 * select  : qmix_learner.py:42-66 + iql_learner.py:57-59 - gather Q(o_t, a_t) from the eval net outputs
 *           q_all[B,n,T+1,A], the double-Q / max next value from the target outputs q_tgt at step t+1, both
 *           multiplied by agent_mask*filled and written agent-minor [B*T, n] (the layout Q_tot concatenates,
 *           value_factorization.py:137-142); also filled_sum[0] = sum(filled).  actions/masks are float32.
 *           avail (nullable; use_actions_mask, iql_learner.py:60-81 + value_factorization.py:86-89): uint8
 *           [B,n,T+1,avail_ld], unavailable actions count as -1e10 in the double-Q arg-max over the eval values
 *           and in the target values of step t+1.
 *           select_bwd scatters d(q_eval_taken) back into a zeroed dq_all.
 * mix     : QMIX_Mixer.forward epilogue (q_mix_head.py:81-94) on precomputed hypernet outputs:
 *           hidden = elu(q . |w1_raw|[n,H] + b1) ; q_tot = hidden . |w2_raw| + b2   (n <= 16), and its backward
 *           (abs' = sign, elu' = exp) producing dq, dw1_raw, db1, dw2_raw (db2 = dq_tot).
 * td      : qmix_learner.py:34-35,76-84 masked TD loss; writes dq_tot and stats[2] = {loss_Q, mean(q_tot)}.
 *           filled_sum[0] and rows_total >= B*T are the GLOBAL sum(filled) and row count, so a rank-local shard
 *           writes its share of the global-minibatch gradient and statistics (sums over local rows / global count). */
int xb_qmix_select_fwd(const float *q_all, const float *q_tgt, const float *actions, const float *agent_mask,
                       const float *filled, const uint8_t *avail, int avail_ld, int B, int n, int T, int A,
                       int double_q, float *q_eval_taken, float *q_next_taken, float *filled_sum, double *scratch,
                       void *stream);
int xb_qmix_select_bwd(const float *d_taken, const float *actions, const float *agent_mask, const float *filled,
                       int B, int n, int T, int A, float *dq_all, void *stream);
int xb_qmix_mix_fwd(const float *q, const float *w1_raw, const float *b1, const float *w2_raw, const float *b2,
                    int64_t R, int n, int H, float *q_tot, void *stream);
int xb_qmix_mix_bwd(const float *dq_tot, const float *q, const float *w1_raw, const float *b1, const float *w2_raw,
                    int64_t R, int n, int H, float *dq, float *dw1_raw, float *db1, float *dw2_raw, void *stream);
int xb_qmix_td(const float *q_tot, const float *q_tot_next, const float *rewards, const float *terminals,
               const float *filled, const float *filled_sum, int B, int n, int T, float gamma, int64_t rows_total,
               float *dq_tot, float *stats, double *scratch, void *stream);

/* ---------------------------------------------------------------- K9W: Weighted QMIX selection / loss --
 * Replaces, for one parameter-sharing group with use_rnn=True, wqmix_learner.py:27-129 (_forward_transitions) and
 * :141-199 (the weighted loss of update) plus their autograd backward down to the agent-network outputs.  Layouts as K9:
 * q_all / q_cent / q_cent_tgt / q_tgt [B,n,T+1,A] (eval, central, target central and target agent networks), actions /
 * agent_mask [B,n,T] and filled [B,T] float32, avail (nullable) uint8 [B,n,T+1,avail_ld], non-zero = available.
 * select_fwd: per (b,i,t), m = agent_mask*filled, g_t = the first maximal index of q_all at t with unavailable actions
 *           at -1e10 (value_factorization.py:86-91); the next action is g_{t+1} when double_q, else the UNMASKED first
 *           argmax of q_tgt at t+1 (q_tgt may be NULL when double_q; the reference's use_rnn branch never masks it).
 *           Writes, agent-minor [B*T, n]: q_eval_taken = q_all[t, a_t]*m, q_cent_taken = q_cent[t, g_t]*m,
 *           q_next_cent = q_cent_tgt[t+1, next]*m; greedy[B,n,T] = g_t (int32, saved for the backward);
 *           agree[B*T] = all_i (g_t == a_t and m != 0) (uint8, CW-QMIX's condition_1: a dead or padded agent clears it);
 *           filled_sum[0] = sum(filled).  One thread per (b,t) row.
 * select_bwd: dq_all[b,i,t,a_t] = d_eval[row,i]*m and dq_cent[b,i,t,g_t] = d_cent[row,i]*m into pre-zeroed outputs; either
 *           (d_eval, dq_all) or (d_cent, dq_cent) may be a NULL pair, not both.
 * loss    : r = mean_i rewards, d = all_i terminals (as xb_qmix_td); y = r + (1-d)*gamma*q_ff_next; td = q_tot - y;
 *           w = alpha, or 1 where td < 0 (mode XB_WQMIX_OW) / where agree or y > q_ff (XB_WQMIX_CW; agree required);
 *           loss_Qmix = sum(w*td^2*filled)/filled_sum, loss_central = sum((q_ff-y)^2*filled)/filled_sum.  Writes
 *           dq_tot = 2*w*td*filled/filled_sum, dq_ff = 2*(q_ff-y)*filled/filled_sum (y and w carry no gradient) and
 *           stats[4] = {loss_Qmix, loss_central, loss, predictQ = sum(q_tot)/rows_total}.  filled_sum[0] and rows_total >=
 *           B*T are GLOBAL, so the SUM of the shards' outputs is the global result; deterministic two-level reduction,
 *           scratch as for K4.
 * All three: B, n, T, A >= 1 and non-NULL required pointers (else XB_EINVAL); n <= 16, the K9 mixer's limit (else
 * XB_ERANGE).  No allocation; graph-capturable. */
#define XB_WQMIX_OW 0
#define XB_WQMIX_CW 1
int xb_wqmix_select_fwd(const float *q_all, const float *q_cent, const float *q_cent_tgt, const float *q_tgt,
                        const float *actions, const float *agent_mask, const float *filled, const uint8_t *avail,
                        int avail_ld, int B, int n, int T, int A, int double_q, float *q_eval_taken,
                        float *q_cent_taken, float *q_next_cent, int32_t *greedy, uint8_t *agree, float *filled_sum,
                        double *scratch, void *stream);
int xb_wqmix_select_bwd(const float *d_eval, const float *d_cent, const float *actions, const int32_t *greedy,
                        const float *agent_mask, const float *filled, int B, int n, int T, int A, float *dq_all,
                        float *dq_cent, void *stream);
int xb_wqmix_loss_fwd_bwd(const float *q_tot, const float *q_ff, const float *q_ff_next, const float *rewards,
                          const float *terminals, const float *filled, const uint8_t *agree, const float *filled_sum,
                          int B, int n, int T, int mode, float alpha, float gamma, int64_t rows_total, float *dq_tot,
                          float *dq_ff, float *stats, double *scratch, void *stream);

/* ---------------------------------------------------------------- K9C: Deep Coordination Graphs (DCG / DCG_S) --
 * Replaces, for one parameter-sharing group with use_rnn=True, dcg_learner.py:39-88 (act: max-plus belief propagation
 * and masked arg-max), :90-104 (q_dcg) and the loss of :161-215 plus its autograd backward down to the head outputs.
 * Layouts: utility outputs f [B,n,T1,A]; payoff outputs pay [2][B,E,T1,A*A], the two orientations ([h_from,h_to] and
 * [h_to,h_from], coordination_graph.py:90-101) `payoff_ld` elements apart; edges_from / edges_to int32 [E] (the
 * graph's edge order); avail (nullable) uint8 [B,n,T1,avail_ld], non-zero = available; actions (taken) [B,n,T] float32
 * and filled [B,T] as K9.  F_e[i][j] = float32((P0[i*A+j] + P1[j*A+i]) / 2), u_v = f_v / n and F_e / E in float64.
 * greedy : instance r = b*T + t reads step t0 + t (training: T1 = T+1, t0 = 1; acting: T = T1 = 1, t0 = 0).
 *          U = (u + 0) + 0, messages m_fwd = m_bwd = 0; n_iter times (none when E = 0), Jacobi:
 *            m_fwd'[e][j] = max_i ((U[from_e][i] - m_bwd[e][i]) + F_e[i][j]),
 *            m_bwd'[e][i] = max_j ((U[to_e][j] - m_fwd[e][j]) + F_e[i][j]),
 *            normalize: m -= (sum_a m[a], summed in action order from 0) / A,
 *            U[v] = (u_v + sum_{e: to_e = v} m_fwd[e]) + sum_{e: from_e = v} m_bwd[e], both sums in edge order from 0;
 *          actions[r, v] (int32 [B*T, n]) = the first maximal index of U[v] with unavailable actions at -1e10;
 *          U_out (nullable) float64 [B*T, n, A] = the final U.  Every operation is one IEEE operation in the order
 *          above (no FMA contraction; divisions correctly rounded), so a float64 restatement is bit-exact.
 *          One CTA per instance; shared memory 8*(n*A + 2*E*A + E) bytes, plus 8*E*A*A for a table of F_e formed
 *          once per instance when n_iter > 1 and the total stays within 48 KB (the same values either way).
 * q_fwd  : per (b,t) row, q_eval = (sum_v u_v[a_v]) + (sum_e F_e[a_from][a_to]) from f_eval / p_eval at step t and
 *          the taken actions, q_next the same from f_tgt / p_tgt at step t+1 and greedy [B*T, n]; sums in order from
 *          0; the payoff sum is dropped unless use_payoff (the reference's E == 0 or n_msg_iterations == 0 rule).
 *          float64 outputs [B*T]; filled_sum[0] = sum(filled).  Heads are [B,n,T+1,A] / [2][B,E,T+1,A*A].
 * td     : Q = q_eval (+ V(s)), Q' = q_next (+ V(s')) for DCG_S (v, v_next and dv all given or all NULL);
 *          r = mean_i rewards (float32), d = all_i terminals, y = r + ((1-d)*gamma in float32)*Q'; td = (Q - y)*filled;
 *          dq = 2*td*filled/filled_sum (float64 [B*T]), dv = float(dq); stats[2] = {loss_Q = sum(td^2)/filled_sum,
 *          predictQ = sum(Q)/rows_total (padded rows included)}.  filled_sum and rows_total >= B*T are GLOBAL, so the
 *          SUM of the shards' outputs is the global result; deterministic two-level reduction, scratch as for K4.
 * q_bwd  : into pre-zeroed df [B,n,T+1,A] and dp [2][B,E,T+1,A*A] (dp_ld apart; NULL unless use_payoff):
 *          df[b,v,t,a_v] = float(dq/n); dp0[b,e,t,a_from*A+a_to] = dp1[b,e,t,a_to*A+a_from] = float(dq/E)/2.
 * All four: n >= 1, A >= 1, E >= 0 and the required pointers (else XB_EINVAL); n <= 32, A <= 64, E <= 512 and the
 * greedy's shared memory within 227 KB (else XB_ERANGE).  No allocation; graph-capturable. */
#define XB_DCG_MAX_AGENTS 32
#define XB_DCG_MAX_ACTIONS 64
#define XB_DCG_MAX_EDGES 512
#define XB_DCG_MAX_SMEM (227 * 1024)
int xb_dcg_greedy(const float *f, const float *payoff, int64_t payoff_ld, const int32_t *edges_from,
                  const int32_t *edges_to, const uint8_t *avail, int avail_ld, int B, int T, int T1, int t0, int n,
                  int A, int E, int n_iter, int normalize, int32_t *actions, double *U_out, void *stream);
int xb_dcg_q_fwd(const float *f_eval, const float *p_eval, int64_t p_eval_ld, const float *f_tgt, const float *p_tgt,
                 int64_t p_tgt_ld, const float *actions, const int32_t *greedy, const float *filled,
                 const int32_t *edges_from, const int32_t *edges_to, int B, int n, int T, int A, int E, int use_payoff,
                 double *q_eval, double *q_next, float *filled_sum, double *scratch, void *stream);
int xb_dcg_td_fwd_bwd(const double *q_eval, const double *q_next, const float *v, const float *v_next,
                      const float *rewards, const float *terminals, const float *filled, const float *filled_sum, int B,
                      int n, int T, float gamma, int64_t rows_total, double *dq, float *dv, float *stats,
                      double *scratch, void *stream);
int xb_dcg_q_bwd(const double *dq, const float *actions, const int32_t *edges_from, const int32_t *edges_to, int B,
                 int n, int T, int A, int E, int use_payoff, float *df, float *dp, int64_t dp_ld, void *stream);

/* ---------------------------------------------------------------- K9Q: QTRAN (QTRAN_base / QTRAN_alt) --
 * Replaces, for one parameter-sharing group with use_rnn=True, qtran_learner.py:199-371 (update_rnn) except the Q_jt
 * and V_jt MLPs (cuBLAS through torch), with the action-encoding part of Q_tran / Q_tran_target
 * (value_factorization.py:354-442, q_mix_head.py:191-211 and :264-292) and the autograd backward of all of it.
 * Layouts as K9: heads q_all / q_tgt [B,n,T+1,A]; actions, agent_mask (m), rewards, terminals [B,n,T] and filled (f)
 * [B,T] float32; avail (nullable) uint8 [B,n,T+1,avail_ld], non-zero = available; rows r = b*T + t, R = B*T.
 * Unavailable actions count as -1e10 in every arg-max; every arg-max and arg-min takes the first extreme index.
 * select : greedy [B,n,T+1] int32 = the masked arg-max of q_all at every step; next [B,n,T] int32 = greedy at t+1 when
 *          double_q, else the arg-max of q_tgt at t+1 with the step-(t+1) mask (q_tgt may be NULL when double_q);
 *          filled_sum[0] = sum(filled).
 * encode_fwd: D = H + A; for agent i of row r, u_i = [h[b,i,t]*m, onehot(a_i)] (the one-hot is not masked) and
 *          e_i = W2 relu(W1 u_i + b1) + b2 (the one-hot product is the column W1[:, H+a_i]).  h [B,n,T+1,H] is read at
 *          steps 0..T-1, the state [B,T+1,S] at step state_t0 + t (0 or 1), the actions from exactly one of act_f
 *          (float32) and act_i (int32), [B,n,act_T], act_T >= T.  W1, W2 [D,D], b1, b2 [D] (nn.Linear layout).
 *          mode XB_QTRAN_BASE: x[r] = [state, sum_i e_i], width S+D;  XB_QTRAN_ALT: x[r*n+i] = [state,
 *          (n-1) e_i, onehot_n(i)], width S+D+n: e_i added n-1 times, as q_mix_head.py:283-285 computes it (the
 *          mask drops one repeat of agent i's own encoding, not agent i).  Sums run in agent order.
 *          Actions must lie in [0, A) (the reference's F.one_hot raises otherwise); an action outside it contributes no
 *          one-hot column here, and to xb_qtran_loss_fwd_bwd it is an out-of-bounds index.  pre (nullable) [R,n,D] = W1 u_i + b1.
 *          Shared memory 4*(2*D*D + 4*D + n*D) bytes.
 * encode_bwd: dx as x (the state and id columns carry no gradient); ge_j = dx's encoding columns of row r (base) or
 *          those of agent-row (r,j) added n-1 times (alt); dz_j = (W2^T ge_j) * (pre > 0); dh[b,j,t] = m * W1[:, :H]^T dz_j
 *          (step T written as zero); dW1 = sum dz_j u_j^T (the one-hot columns a scatter by action), db1 = sum dz_j,
 *          dW2 = sum ge_j relu(pre_j)^T, db2 = sum ge_j.  The weight gradients are partial sums over fixed chunks of
 *          max(128, ceil(R*n/1024)) agent-rows in row order, then added in chunk order: bit-identical from launch to
 *          launch.  work holds xb_qtran_encode_bwd_work(B, n, T, H, A) = 2*R*n*D + chunks*(2*D*D + 2*D) floats
 *          (XB_EINVAL if work_floats is smaller): ge and dz1 for every agent-row plus at most 1024 partials, about
 *          9 MB at B = 32, T = 60, n = 5, H = 64, A = 12 and linear in R*n (2.1 GB at B = 1024, T = 60, n = 32, A = 64,
 *          the same order as alt's x there).
 * loss   : r = mean_i rewards, d = all_i terminals (as xb_qmix_td); Q_tot = sum_i q_all[t, a_i]*m and Q_tot_g =
 *          sum_i q_all[t, g_i]*m (g = greedy at t), in agent order; V = v [R].
 *          base: qjt, qjt_greedy, qjt_next [R]; y = r + (1-d)*gamma*qjt_next; td = (qjt - y)*f; eo = (Q_tot_g -
 *          qjt_greedy + V)*f; en = min(Q_tot - qjt + V, 0)*f; den = filled_sum.
 *          alt: qjt, qjt_greedy, qjt_next [R*n, A]; per (r,i): y = r + (1-d)*gamma*qjt_next[r,i,next_i]; td =
 *          (qjt[r,i,a_i] - y)*f; eo = (Q_tot_g - qjt_greedy[r,i,g_i] + V)*f; en = min_a (q_all[i,t,a] + sum_{j != i}
 *          q_all[j,t,a_j]*m_j - qjt[r,i,a] + V)*f over the unmasked row; den = n*filled_sum.
 *          Each loss is sum(term^2)/den.  Writes dqjt (TD only: qjt is detached in opt and nopt; alt writes whole rows),
 *          dv [R], and scatters the opt and nopt gradients into pre-zeroed dq_all [B,n,T+1,A] (taken, greedy and, for
 *          alt, the arg-min entries; coinciding entries add).  stats[5] = {loss_td, loss_opt, loss_nopt, loss =
 *          loss_td + lambda_opt*loss_opt + lambda_nopt*loss_nopt, Q_joint = sum of the taken qjt / (rows_total, times n
 *          for alt), padded rows included}.  filled_sum and rows_total >= R are GLOBAL, so the SUM of the shards'
 *          outputs is the global result; deterministic two-level reduction, scratch as for K4.
 * All: B, n, T, A (and S, H for the encoder) >= 1, mode in {BASE, ALT} and the required pointers (else XB_EINVAL);
 * n <= 32, A <= 64, H <= 64 (else XB_ERANGE).  No allocation; graph-capturable. */
#define XB_QTRAN_BASE 0
#define XB_QTRAN_ALT 1
#define XB_QTRAN_MAX_AGENTS 32
#define XB_QTRAN_MAX_ACTIONS 64
#define XB_QTRAN_MAX_HIDDEN 64
int xb_qtran_select(const float *q_all, const float *q_tgt, const uint8_t *avail, int avail_ld, const float *filled,
                    int B, int n, int T, int A, int double_q, int32_t *greedy, int32_t *next, float *filled_sum,
                    double *scratch, void *stream);
int xb_qtran_encode_fwd(int mode, const float *state, int state_t0, const float *h, const float *agent_mask,
                        const float *act_f, const int32_t *act_i, int act_T, const float *w1, const float *b1,
                        const float *w2, const float *b2, int B, int n, int T, int S, int H, int A, float *x,
                        float *pre, void *stream);
int64_t xb_qtran_encode_bwd_work(int B, int n, int T, int H, int A);
int xb_qtran_encode_bwd(int mode, const float *dx, const float *h, const float *agent_mask, const float *act_f,
                        const int32_t *act_i, int act_T, const float *w1, const float *w2, const float *pre, int B,
                        int n, int T, int S, int H, int A, float *dh, float *dw1, float *db1, float *dw2, float *db2,
                        float *work, int64_t work_floats, void *stream);
int xb_qtran_loss_fwd_bwd(int mode, const float *q_all, const float *actions, const int32_t *greedy,
                          const int32_t *next, const float *agent_mask, const float *filled, const float *rewards,
                          const float *terminals, const float *qjt, const float *qjt_greedy, const float *qjt_next,
                          const float *v, const float *filled_sum, int B, int n, int T, int A, float gamma,
                          float lambda_opt, float lambda_nopt, int64_t rows_total, float *dqjt, float *dv,
                          float *dq_all, float *stats, double *scratch, void *stream);

/* Tensor-core forward of the whole mixer (hypernet GEMMs + epilogue in ONE kernel; wgmma with register
 * accumulators, bf16 hi/lo split operands, 3 MMAs per product, fp32 accumulate): q_tot[R] from states[R,S], q[R,n]
 * and the raw Linear parameters of QMIX_Mixer (q_mix_head.py:52-64): w_l1[4] / b_l1[4] are HOST arrays of 4 device
 * pointers to the first-layer weights [32,S] / biases [32] of hyper_w_1, hyper_b_1, hyper_w_2, hyper_b_2 (in that
 * order), wb1[n*32,32] = hyper_w_1[2], wb2[32,32] = hyper_w_2[2], wb2c[1,32] = hyper_b_2[2].  Requires dim_hidden =
 * dim_hypernet_hidden = 32, n <= 8 and the staged operands to fit 220 KB of shared memory (else XB_ERANGE and the
 * caller uses cuBLAS + xb_qmix_mix_fwd).  Forward only: used for the target mixer / inference. */
int xb_qmix_mix_fused_fwd(const float *states, const float *q, const float *const *w_l1_host,
                          const float *const *b_l1_host, const float *wb1, const float *bias_wb1, const float *wb2,
                          const float *bias_wb2, const float *wb2c, const float *bias_wb2c, int64_t R, int S, int n,
                          int H, int HH, float *q_tot, void *stream);

/* ---------------------------------------------------------------- K8: SAC loss stages ----------------
 * Replaces the elementwise/reduction parts of SAC_Learner.update (xuance/torch/learners/policy_gradient/
 * sac_learner.py:52-88).  `alpha` is a DEVICE scalar (exp(log_alpha)).
 * actor : p_loss = mean(alpha*log_pi - min(q1,q2)); writes dlog_pi, dq1, dq2 (torch.min ties split 1/2),
 *         stats[4] = {Ploss, mean(min q), mean(log_pi), 0}
 * critic: backup = r + (1-d)*gamma*(target_q - alpha*log_pi_next); q_loss = mse(q1,backup)+mse(q2,backup);
 *         writes dq1, dq2, backup; stats[2] = {Qloss, 0} */
int xb_sac_actor_loss(const float *log_pi, const float *q1, const float *q2, const float *alpha, int64_t B,
                      int64_t B_total, float *dlog_pi, float *dq1, float *dq2, float *stats, double *scratch,
                      void *stream);
int xb_sac_critic_loss(const float *q1, const float *q2, const float *target_q, const float *log_pi_next,
                       const float *rew, const float *term, const float *alpha, float gamma, int64_t B,
                       int64_t B_total, float *dq1, float *dq2, float *backup, float *stats, double *scratch,
                       void *stream);

/* ---------------------------------------------------------------- K8D: SAC-Discrete loss stages -------
 * Replaces the elementwise/reduction parts of SACDIS_Learner.update (xuance/torch/learners/policy_gradient/
 * sacdis_learner.py:52-75) for a Categorical policy over A actions, 1 <= A <= 64 (else XB_ERANGE).  All matrices are
 * row-major [B, A] float32; `alpha` is a DEVICE scalar.  Per row, as Categorical(logits).probs and the reference's
 * log rule compute them in float32 (actor_critic.py:184-205):
 *   p = softmax(z - logsumexp(z));  log_pi = log(p + 1e-8*[p == 0])  (floored at log(1e-8) only where p is exactly 0;
 *   subnormal p are kept: the library is built with flush-to-zero off)
 * actor : p_loss = mean_b sum_a p*(alpha*log_pi - min(q1,q2)).  Writes dlogits = p*(g - sum_a p*g) / B_total with
 *         g = alpha*log_pi - min(q1,q2) + alpha*p/(p + z) (the softmax backward; entries with p = 0 get exactly 0) and
 *         stats[4] = {Ploss, Qvalue = sum min(q1,q2) / (B_total*A), sum log_pi / (B_total*A), 0}.  No gradient to q1 /
 *         q2 is written: the reference's critic.zero_grad() discards the one its p_loss.backward() leaves there.
 * critic: target = sum_a p'*(min(tq1,tq2) - alpha*log_pi') of the next-state logits and the target critic's values;
 *         backup = r + (1-d)*gamma*target; q_loss = mse(q1[a], backup) + mse(q2[a], backup), a = trunc(actions[b])
 *         (float32 as stored).  Writes backup[B], dq1 / dq2 dense [B, A]: 2*(q_i[a] - backup)/B_total in column a and
 *         0 elsewhere, and stats[2] = {Qloss, 0}.  A row whose action is not in [0, A) (or NaN) selects no column:
 *         its dq rows are all 0 and it adds NaN to Qloss, so a corrupt batch shows in the log without an out-of-bounds
 *         read.
 * Both: B_total >= B rows scale the means (a SUM all-reduce of shards gives the global values); scratch as for K4. */
int xb_sacdis_actor_loss(const float *logits, const float *q1, const float *q2, const float *alpha, int64_t B, int A,
                         int64_t B_total, float *dlogits, float *stats, double *scratch, void *stream);
int xb_sacdis_critic_loss(const float *q1, const float *q2, const float *actions, const float *logits_next,
                          const float *tq1, const float *tq2, const float *rew, const float *term, const float *alpha,
                          float gamma, int64_t B, int A, int64_t B_total, float *dq1, float *dq2, float *backup,
                          float *stats, double *scratch, void *stream);

/* ---------------------------------------------------------------- K8T: DDPG / TD3 stages --------------
 * Replaces the elementwise/reduction parts of DDPG_Learner.update / TD3_Learner.update (xuance/torch/learners/
 * policy_gradient/{ddpg,td3}_learner.py) and the action noise of core/off_policy.py:142-144 and
 * TwinDelayedActorCritic.Qtarget (actor_critic.py:289-296).  float32 throughout; the elementwise outputs are
 * bit-identical to torch's expressions (no FMA contraction); NaN propagates as in torch.clamp / minimum / maximum.
 * perturb: a, noise, out [B, D] row-major, low / high [D].  n = noise*scale; if noise_clip >= 0, n is clamped to
 *          [-noise_clip, noise_clip]; out = clamp(a + n, low[j], high[j]).  `out` may alias `a`.  The noise is a
 *          standard normal tensor the caller draws (torch.randn_like), so the random stream stays torch's.
 * critic: q2, tq2, dq2 all NULL (DDPG, one critic) or all non-NULL (TD3, twin critics); a mix is XB_EINVAL.
 *         t = tq1 or min(tq1, tq2); backup = rew + (gamma*(1 - term))*t; q_loss = sum_i mse(q_i, backup).
 *         Writes backup[B], dq_i = 2*(q_i - backup)/B_total, stats[4] = {Qloss (the per-critic means added in
 *         float32), mean(q1), mean(q2) (0 for DDPG), 0}.
 * actor : DDPG: p_loss = -mean(q1), dq1 = -1/B_total.  TD3 (q2, dq2 non-NULL): p_loss = -mean((q1 + q2)/2) (the row's
 *         half-sum rounded in float32), dq1 = dq2 = (-1/B_total)*0.5.  stats[4] = {Ploss, 0, 0, 0}.
 * Both losses: B_total >= B rows scale the means (a SUM all-reduce of shards gives the global values); scratch as for
 * K4.  XB_EINVAL on NULL pointers, B <= 0, B_total < B or D <= 0. */
int xb_perturb_actions(const float *a, const float *noise, int64_t B, int D, float scale, float noise_clip,
                       const float *low, const float *high, float *out, void *stream);
int xb_ddpg_critic_loss(const float *q1, const float *q2, const float *tq1, const float *tq2, const float *rew,
                        const float *term, float gamma, int64_t B, int64_t B_total, float *dq1, float *dq2,
                        float *backup, float *stats, double *scratch, void *stream);
int xb_ddpg_actor_loss(const float *q1, const float *q2, int64_t B, int64_t B_total, float *dq1, float *dq2,
                       float *stats, double *scratch, void *stream);

/* ---------------------------------------------------------------- K13: GRU sequence kernels ----------
 * The recurrence of a one-layer torch.nn.GRU (gate order r, z, n) over S independent sequences of T steps, as the
 * recurrent representations of MAPPO run it (Basic_RNN, rl_models/representations/rnn.py:9-99).  xg[S, T, 3H] is the
 * projected input x W_ih^T + b_ih (a cuBLAS GEMM the caller runs for all T at once); w_hh[3H, H], b_hh[3H] are torch's
 * weight_hh_l0 / bias_hh_l0; h0[S, H] is nullable (zeros).  Per step, gh = W_hh h + b_hh and
 *     r = sigmoid(xg_r + gh_r), z = sigmoid(xg_z + gh_z), n = tanh(xg_n + r * gh_n), h' = (1 - z) * n + z * h.
 * fwd: writes y[S, T, H] (every h'), hT[S, H] and, when gates != NULL (training), gates[S, T, 4H] = {r, z, n, gh_n}.
 * bwd: from dy[S, T, H] and a nullable dhT[S, H], with the forward's gates, y and h0, writes dxg[S, T, 3H] (the gradient
 *      of xg: dW_ih, db_ih and dx follow by GEMMs / sums), dgh[S, T, 3H] (the gradient of W_hh h + b_hh: dW_hh =
 *      sum dgh^T h_{t-1}, db_hh = sum dgh) and, when dh0 != NULL, dh0[S, H].
 * float32 on the CUDA cores with accurate expf / tanhf; one CTA walks all T steps of 4 sequences with W_hh resident in
 * shared memory.  No atomics: every sequence's result is bit-identical from launch to launch and whichever CTA owns it.
 * 1 <= H <= 64, T >= 1, S >= 1, and NULL required pointers, are XB_EINVAL. */
int xb_gru_seq_fwd(const float *xg, const float *w_hh, const float *b_hh, const float *h0, int64_t S, int T, int H,
                   float *y, float *hT, float *gates, void *stream);
int xb_gru_seq_bwd(const float *dy, const float *dhT, const float *w_hh, const float *gates, const float *y,
                   const float *h0, int64_t S, int T, int H, float *dxg, float *dgh, float *dh0, void *stream);

/* ---------------------------------------------------------------- K13L: LSTM sequence kernels ---------
 * The recurrence of a one-layer torch.nn.LSTM (gate order i, f, g, o) over S independent sequences of T steps, as
 * DRQN's recurrent Q head runs it (RecurrentQValueHead, rl_models/heads/q_head.py:126-175).  xg[S, T, 4H] is the
 * projected input x W_ih^T + b_ih (a cuBLAS GEMM the caller runs for all T at once); w_hh[4H, H], b_hh[4H] are torch's
 * weight_hh_l0 / bias_hh_l0; h0, c0 [S, H] are nullable (zeros).  Per step, with pre = xg + (W_hh h + b_hh),
 *     i = sigmoid(pre_i), f = sigmoid(pre_f), g = tanh(pre_g), o = sigmoid(pre_o), c' = f c + i g, h' = o tanh(c').
 * fwd: writes y[S, T, H] (every h'), hT, cT [S, H] and, when gates != NULL (training), gates[S, T, 5H] = {i, f, g, o, c'}.
 * bwd: from dy[S, T, H] and nullable dhT, dcT [S, H], with the forward's gates and c0, writes dxg[S, T, 4H], the gradient
 *      of the pre-activations.  All four are plain sums of xg and W_hh h + b_hh, so dxg is also the gradient of
 *      W_hh h + b_hh: dW_ih, db_ih, dx, dW_hh = sum dxg^T h_{t-1} and db_hh = sum dxg follow by GEMMs / sums.  When
 *      dh0 / dc0 != NULL, writes dh0, dc0 [S, H].
 * float32 on the CUDA cores with accurate expf / tanhf; one CTA of 4H threads walks all T steps of 4 sequences.  W_hh
 * stays on chip: the first 32 k-entries of each thread's column in registers, the rest in shared memory (192 KB of the
 * 256 KB at H = 128).  No atomics: every sequence's result is bit-identical from launch to launch and whichever CTA
 * owns it.  1 <= H <= 128, T >= 1, S >= 1, and NULL required pointers, are XB_EINVAL. */
int xb_lstm_seq_fwd(const float *xg, const float *w_hh, const float *b_hh, const float *h0, const float *c0, int64_t S,
                    int T, int H, float *y, float *hT, float *cT, float *gates, void *stream);
int xb_lstm_seq_bwd(const float *dy, const float *dhT, const float *dcT, const float *w_hh, const float *gates,
                    const float *c0, int64_t S, int T, int H, float *dxg, float *dh0, float *dc0, void *stream);

/* ---------------------------------------------------------------- K7: flat-bucket optimiser step -----
 * Replaces clip_grad_norm_ + torch.optim.Adam.step on the learner's parameters (ppo_learner.py:61-65;
 * Adam eps=1e-5, no weight decay, no amsgrad) over ONE flat float32 bucket (params/grads/exp_avg/exp_avg_sq
 * are each a single contiguous array - the same bucket the NCCL all-reduce uses).
 * xb_grad_sumsq  : norm_out[0] = sqrt(sum g^2) * grad_scale   (deterministic two-level reduction)
 * xb_adam_step   : g' = g * grad_scale * min(1, max_norm/(norm+1e-6)) (max_norm <= 0: no clip);
 *                  m = m + (g'-m)*(1-b1); v = v*b2 + g'*g'*(1-b2); p -= step_size * m/(sqrt(v)/bc2_sqrt + eps)
 *                  hyper (device, float32[4]) = {step_size = lr/(1-b1^t), bc2_sqrt = sqrt(1-b2^t), unused, unused}
 *                  write_back_grad != 0 stores g' into g (what clip_grad_norm_ leaves in .grad)
 * xb_soft_update : target = target*(1-tau) + tau*source    (SoftActorCritic.soft_update, actor_critic.py:155-158)
 */
int xb_grad_sumsq(const float *g, int64_t n, float grad_scale, float *norm_out, double *scratch, void *stream);
int xb_adam_step(float *p, float *g, float *m, float *v, int64_t n, const float *hyper,
                 float beta1, float beta2, float eps, float max_norm, const float *norm, float grad_scale,
                 int write_back_grad, void *stream);
int xb_soft_update(float *target, const float *source, int64_t n, float tau, void *stream);

/* ---------------------------------------------------------------- K10/K11: device-side rollout glue ---
 * SURVEY.md section 8f-1: what OnPolicyAgent.get_actions does after the network (core/on_policy.py:128-169) and what
 * Agent._process_observation / RunningMeanStd.update do before it (agents/base/agent.py:262-279,
 * common/statistic_tools.py:117-185), each as ONE launch writing straight into device buffers (e.g. the K1 staging
 * rows of the rollout buffer), so that a vector-env step costs one H2D of observations and one D2H of N int32 actions.
 *
 * xb_categorical_act: CategoricalDistribution over logits[N,A] (modules/distributions.py:128-162), A <= 64.
 *   forced_actions != NULL : a_n = (int)forced_actions[n]          (log_prob / entropy of given actions)
 *   else uniforms != NULL  : a_n = min{i : u_n < p_0+..+p_i}, u in [0,1) (stochastic_sample; inverse CDF in index order,
 *                            the last index with p_i > 0 if rounding leaves the total mass below u_n: a category
 *                            of probability zero, e.g. a masked action, is never drawn)
 *   else                   : a_n = first argmax_i p_i               (deterministic_sample)
 *   outputs (each nullable, at least one): actions_f32[N] (the float32 the buffers store), actions_i32[N] (for the
 *   host-side env step), logp[N] = log_softmax(logits)[a], entropy[N] = -sum p log p over p > 0 (finite for -inf logits).
 * xb_gaussian_act: DiagGaussianDistribution(mu[N,D], exp(log_std[D])) (modules/distributions.py:165-197).
 *   forced_actions != NULL : x = forced_actions[N,D]; actions_f32 is not written (log_prob / entropy of given actions)
 *   else noise != NULL     : x = mu + exp(log_std) * noise, noise[N,D] standard normals (stochastic_sample)
 *   else                   : x = mu                                   (deterministic_sample)
 *   outputs (each nullable, at least one): actions_f32[N,D] (e.g. the rollout buffer's staging rows),
 *   logp[N] = sum_j log N(x_j; mu_j, sigma_j), entropy[N] = sum_j (1/2 + log(2 pi)/2 + log_std_j).
 * xb_rms_update_normalize: x[N,D] float32.
 *   update != 0: (mean, var)[D] <- parallel-variance merge with the batch moments, float32 in the reference's operation
 *                order; `count` is the running count BEFORE the merge (host state, Python float in the reference).
 *                The batch sums run row after row, as NumPy reduces axis 0 of an [N, D > 1] batch; for D = 1 NumPy
 *                sums the single column pairwise once N >= 8, so there the moments may differ in the last bits.
 *   out != NULL: out = clip((x - mean) / (sqrt(var) + eps), -clip_range, clip_range) with the UPDATED statistics
 *                (PPO_Agent.train calls obs_rms.update(obs) and then _process_observation(obs), ppo_agent.py:115-116).
 */
int xb_categorical_act(const float *logits, const float *uniforms, const float *forced_actions, int N, int A,
                       float *actions_f32, int32_t *actions_i32, float *logp, float *entropy, void *stream);
int xb_gaussian_act(const float *mu, const float *log_std, const float *noise, const float *forced_actions, int N, int D,
                    float *actions_f32, float *logp, float *entropy, void *stream);
int xb_rms_update_normalize(const float *x, int N, int64_t D, float *mean, float *var, double count, int update,
                            float *out, float clip_range, float eps, void *stream);

/* ---------------------------------------------------------------- K12: tensor-core layers (wgmma / TMA) ----------
 * The pixel encoders' convolutions and hidden layer (NatureCNN of AC_CNN_Atari / Basic_CNN: rl_models/representations/cnn.py:
 * 45-50, 84-101; layers.py:16-65), forward, data gradient and weight gradient, that cuDNN runs as CUDA-core fp32 kernels
 * (85 % of the fp32 PPO update).  Every float32 operand travels as 1-3 bfloat16 "planes" (x = sum of its planes; plane q =
 * bf16 of the residual left by the planes before it: 1 plane is exact for integers <= 256 such as raw uint8 pixels, 2
 * planes are exact to 2^-16, 3 planes to 2^-24); products are accumulated in float32 registers, one accumulator per order of
 * magnitude (plane-index sum), added smallest first in the epilogue.  planes_a <= planes_b; kept products: index sum <
 * planes_b.
 * xb_split_bf16       : x (float32[n]) -> planes[0] = bf16(x), planes[1] = bf16(x - planes[0]), [planes[2] = ...]
 * xb_pack_conv_weight : torch [N, C, KH, KW] float32 (* scale) -> bf16 planes of [N, (kh, kw, c)] (also a Linear over a
 *                       [C,H,W] flatten).  scale = 1/255 folds `observations / 255.0` (cnn.py:98) into the first layer,
 *                       whose A operand is then the raw uint8 pixel as ONE exact bf16 plane.
 * xb_gemm_gather_tc   : D[m,n] = sum_{t,c} in[b, y*sy+dy[t], x*sx+dx[t], c] * W[n, t*C+c] (+bias, ReLU), m = (b,y,x) over
 *                       [B,OY,OX], n < N; in / W as bf16 planes (NHWC, [N,K]); a work item is (128 sites, n_tile columns),
 *                       planes_b * n_tile <= 256, n_tile % 32 == 0, N % n_tile == 0; result as float32 and / or
 *                       planes_out bf16 planes written to columns [out_c0, out_c0+N) of row
 *                       (b*out_H + y*oys+oy0)*out_W + x*oxs+ox0 of a matrix with out_ld elements per row
 *                       (out_ld % 8 == out_c0 % 8 == 0).  C % 8 == 0, (T*C) % 64 == 0, T <= 64; dy / dx are HOST arrays
 *                       (copied into the launch parameters).  relu_mask (nullable, bf16, the output's pixel index in a
 *                       matrix of mask_ld elements per pixel from column mask_c0; mask_ld = 0: addressed exactly like
 *                       the output): result zeroed where mask <= 0 - the ReLU derivative applied to a data gradient,
 *                       mask = plane 0 of the saved activation.  colsum (nullable, float32 [ceil(M/128)][N]): row i =
 *                       column sums of the result rows of M tile i (after bias / ReLU / mask; deterministic) - the
 *                       partials of the bias gradient of the layer whose output gradient this call produces
 *                       (finish with xb_wgrad_reduce(colsum, tiles, N, 1, 1, 1, 1.0, db)).  Forward conv: dy = kh - pad, (sy,sx) = stride; Linear: one tap;
 *                       data gradients: flipped taps over the output gradient, one call per stride phase.
 * xb_wgrad_gather_tc  : weight gradient of the same gathered GEMM: partials[s, (t,c), n] = sum over the sites of split s of
 *                       in[b, y*sy+dy[t], x*sx+dx[t], c] * G[site*g_ld + n]; G = output gradient planes.  Both operands
 *                       are fed MN-major (16-byte units transposed into the core matrices); one work item =
 *                       (128 columns of (t,c), n_tile columns, split).  partials: float32 [splits, T*C, N].  One A plane
 *                       with C = 8, a full tap rectangle in row-major order, N = n_tile = 32 and T*C <= 256 (conv1 over raw
 *                       pixels) runs from TMA input windows instead, one work item per split, with the same partials bit
 *                       for bit; XB_K12_TMA=0 keeps the gathered path.  So does three planes on each side with C = 32 read
 *                       as pixel pairs (a KH x 4 tap rectangle in row-major order, even sx and dx[0], even IW), N = n_tile
 *                       = 64 (conv2 over act1): TMA pair windows, one box per grid row, image and K tile.
 * xb_wgrad_reduce     : dw[N, C, KH, KW] (torch layout) (+)= scale * sum_s partials[s, (kh,kw,c), n], splits added in a fixed
 *                       order; `partials` is scratch: with more than 256 splits groups of rows are folded in place first. */
int xb_split_bf16(const float *x, int64_t n, int planes, void *out /* bf16 [planes, n] */, void *stream);
/* K3 variant that feeds K12: gathers uint8 rows (sample_batch, memory_tools.py:64-84; idx NULL = rows 0..B-1) and writes
 * dst[q, b, :] = plane q of float32(x)/255.0f for q < planes (bf16 [planes, B, row_bytes], planes 2 or 3), or with
 * planes == 1 the raw pixel value as one exact bf16 plane (the 1/255 lives in the packed weights); row_bytes % 16 == 0. */
int xb_gather_obs_planes(const uint8_t *src, const int64_t *idx, int64_t B, int64_t row_bytes, int planes, void *dst,
                         void *stream);
int xb_pack_conv_weight(const float *w, int N, int C, int KH, int KW, int planes, float scale,
                        void *out /* bf16 [planes, N, KH*KW*C] */, void *stream);
/* One operand form of one weight (xb_pack_weights): torch weight w [N, C, KH, KW] float32 (a Linear layer over a flattened
 * [C, H, W] feature map is N x C x H x W) -> bf16 planes out [planes][rows][cols] of scale * w, with
 *   mode 0: rows = N, cols = (kh, kw, c)            the B operand of the forward GEMM (= xb_pack_conv_weight)
 *   mode 1: rows = (kh, kw, c), cols = N            its transpose: the B operand of a Linear layer's data gradient
 *   mode 2: rows = C, cols = (tap, n), tap t = (kh[t], kw[t])   the B operand of one stride phase of a convolution's data
 *                                                    gradient (flipped taps in the order of the launch's chunks) */
#define XB_PACK_MAX_JOBS 16
#define XB_PACK_MAX_TAPS 16
typedef struct XbPackJob {
    const float *w;
    void *out;
    int N, C, KH, KW;
    int mode, n_taps;
    signed char kh[XB_PACK_MAX_TAPS], kw[XB_PACK_MAX_TAPS];
    float scale;
    int planes;
} XbPackJob;
/* Every operand form an encoder needs for one update in ONE launch: jobs is a HOST array (copied into the launch parameters),
 * n_jobs <= XB_PACK_MAX_JOBS.  Replaces one xb_pack_conv_weight / transpose / xb_split_bf16 launch per form. */
int xb_pack_weights(const XbPackJob *jobs, int n_jobs, void *stream);
int xb_gemm_gather_tc(int planes_a, int planes_b, const void *in, int64_t in_plane, const void *w, int64_t w_plane,
                      const float *bias, const void *relu_mask, int64_t mask_ld, int mask_c0, int B, int IH, int IW, int C,
                      int OY, int OX, int sy, int sx, int T, const int8_t *dy, const int8_t *dx, int N, int n_tile, int relu,
                      void *out_planes, int64_t out_plane, int planes_out, float *out_f32, int out_H, int out_W, int oys,
                      int oxs, int oy0, int ox0, int64_t out_ld, int out_c0, float *colsum, void *stream);
/* xb_gemm_gather_tc for a convolution whose input is stored in a PADDED-ROW layout [planes][B * hp_in][W][C] (hp_in rows per
 * image of which the first / last are zero padding), with the A operand fetched by TMA: a work item is box_h consecutive
 * grid rows x box_px sites (<= 128 GEMM rows); chunk i (64 K values = box_c = 64 channels of one pixel; a 32-channel tensor
 * is passed as its 64-channel pixel-pair view) is ONE box per plane at channel c0[i], pixel w0[i] (negative = left padding,
 * zero-filled by the TMA unit), rows tile_row0 * row_step + r0[i] + k * row_step, k < box_h (the tensor is described to the
 * TMA unit as {channel, pixel, row mod row_step, row / row_step, plane}; in_rows must be a multiple of row_step).
 * relu_mask rows are the output's, in a tensor mask_W pixels wide with the pixel index shifted by mask_x0 (mask_W = 0: laid
 * out exactly like the output).  Output sites are indexed over a padded grid too: hp rows per image, rows y0..y1 valid (the
 * others are never written: the caller keeps them zero), row y lands at ((b*out_H + (y-y0)*oys + oy0)*out_W + x*oxs + ox0).
 * W is [planes_b][N][n_chunks*64] in chunk order.  Everything else as xb_gemm_gather_tc. */
int xb_gemm_box_tc(int planes_a, int planes_b, const void *in, int64_t in_plane, int C, int W, int64_t in_rows, int box_c,
                   int box_px, int box_h, int row_step, int n_chunks, const int16_t *c0, const int16_t *w0, const int16_t *r0,
                   const void *w, int64_t w_plane, const float *bias, const void *relu_mask, int mask_W, int mask_x0, int B,
                   int hp, int y0, int y1, int N, int n_tile, int relu, void *out_planes, int64_t out_plane, int planes_out,
                   float *out_f32, int out_H, int out_W, int oys, int oxs, int oy0, int ox0, int64_t out_ld, int out_c0,
                   float *colsum, void *stream);
/* The gathered GEMM with the activation tile RESIDENT in shared memory ("halo" mode): stride-1 gathers over a 64-channel
 * padded-row tensor in [planes][B*hp rows][W pixels][64] (in_rows = B*hp) - a 3x3 convolution, its data gradient, the stride
 * phases of a strided convolution's data gradient.  The sites are the positions of the haloed raster: row R (image R / hp,
 * padded row y = R % hp), column hc = pixel hc + halo_w0 (halo_w0 <= 0, halo_w columns per row; pixels outside [0, W) read
 * as zero); an M tile is 128 consecutive positions and ONE TMA box per plane holds every input its taps read.  Sub-item j
 * (n_sub <= 4: the n tiles of a forward layer or the stride phases of a data gradient) multiplies with rows j*N .. of
 * w [planes_b][n_sub*N][n_chunks*64]; its chunk i reads the site (R + dr[j*n_chunks+i], pixel + dc[..]) - a descriptor
 * offset into the resident tile.  Valid sites of sub-item j: y0 <= y <= sub_y1[j], 0 <= x <= sub_x1[j]; they land at row
 * ((b*out_H + (y-y0)*oys + sub_oy0[j])*out_W + x*oxs + sub_ox0[j]) of the output, columns out_c0 + j*N (same_cols: out_c0 for
 * every sub-item).  n_sub * n_chunks <= 16.  bias / relu / relu_mask (mask_W, mask_x0) / planes / colsum
 * ([ceil(B*hp*halo_w / 128) * n_sub][N]) as xb_gemm_box_tc. */
int xb_gemm_halo_tc(int planes_a, int planes_b, const void *in, int64_t in_plane, int W, int64_t in_rows, int halo_w, int halo_w0,
                    int n_sub, int n_chunks, const int16_t *dr, const int16_t *dc, const void *w, int64_t w_plane,
                    const float *bias, const void *relu_mask, int mask_W, int mask_x0, int B, int hp, int y0,
                    const int16_t *sub_y1, const int16_t *sub_x1, int N, int relu, void *out_planes, int64_t out_plane,
                    int planes_out, float *out_f32, int out_H, int out_W, int oys, int oxs, const int16_t *sub_oy0,
                    const int16_t *sub_ox0, int64_t out_ld, int out_c0, int same_cols, float *colsum, void *stream);
/* Weight gradient of the same convolution with both operands fetched by TMA boxes: `in` as for xb_gemm_box_tc, `g` the
 * output gradient in the padded site layout [planes_b][g_rows][box_px*box_c/64 sites][N]; a chunk of the reduction is box_h
 * grid rows (box_w * box_h <= 64 sites), N % 64 == 0; partials: float32 [splits, n_chunks*64, N] (reduce with xb_wgrad_reduce). */
int xb_wgrad_box_tc(int planes_a, int planes_b, const void *in, int64_t in_plane, int C, int W, int64_t in_rows, int box_c,
                    int box_px, int box_h, int row_step, int n_chunks, const int16_t *c0, const int16_t *w0, const int16_t *r0,
                    const void *g, int64_t g_plane, int64_t g_rows, int N, int splits, float *partials, void *stream);
/* Diagnostics (XB_K12_TIMING=1 in the environment): per CTA of the LAST K12 launch, clock64 cycles of each warp role and of its
 * barrier waits: out_host[cta][12] = {MMA total, MMA wait operands, MMA wait epilogue, MMA wait resident tile, producer total,
 * producer wait ring, producer wait tile buffer, epilogue total, epilogue wait accumulator, ...}.  Synchronises the device. */
int xb_debug_k12_timing(unsigned long long *out_host, int n_ctas);
/* Test hook: the raw shared-memory image (first out_bytes, 0xEE = untouched) after ONE TMA box load of the 4-D tensor map the
 * box mode builds - lets the tests pin the layout (pixel packing, row step, 128-byte swizzle, zero fill) byte for byte. */
int xb_debug_tma_box(const void *in, int64_t in_plane, int planes, int C, int W, int64_t rows, int box_c, int box_px, int box_h,
                     int row_step, int c0, int c1, int c2, int c3, uint32_t expect_bytes, void *out, uint32_t out_bytes,
                     void *stream);
int xb_wgrad_gather_tc(int planes_a, int planes_b, const void *in, int64_t in_plane, const void *g, int64_t g_plane,
                       int64_t g_ld, int B, int IH, int IW, int C, int OY, int OX, int sy, int sx, int T, const int8_t *dy,
                       const int8_t *dx, int N, int n_tile, int splits, float *partials, void *stream);
int xb_wgrad_reduce(float *partials, int splits, int N, int C, int KH, int KW, float scale, float *dw, int accumulate,
                    void *stream);

#ifdef __cplusplus
}
#endif
#endif /* XB200_H_ */
