/* b200rl -- C ABI of the H100 (sm_90a) learner hot path for DI-engine.
 *
 * This is the drop-in boundary: what a binding for the reference's plugin hook (ding/hpc_rl/wrapper.py:86-133,
 * registry :62-73) would call for each of the hot-path operators of ding/rl_utils.  The reference's own boundary is a
 * Python decorator that forwards to an external, un-vendored package (hpc_rll); this library is the compiled code
 * under such a package: plain device pointers, sizes and scalars, no torch types.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to a dense row-major tensor: fp32 (`float`) unless declared `long long`
 *     (the reference's int64 action tensors).  "nullable" pointers select the reference's `None` default.
 *   - trajectory tensors are (T, B[, ...]) with time as the slowest axis, exactly as the reference lays them out.
 *   - hyper-parameters are C doubles (python floats); the library narrows them to fp32 the way torch narrows a
 *     python scalar operand, so products such as gamma*lambda_ are formed in double first.
 *   - `stream` is a cudaStream_t (passed as void*); all work is enqueued on it, nothing synchronises, nothing
 *     allocates.  Outputs are caller-allocated.
 *   - `workspace` is a caller-owned scratch buffer of at least b200rl_workspace_bytes() bytes that must be
 *     zero-filled once when it is created; launches that share a workspace must be ordered on one stream.
 *   - return value: 0 success; > 0 a cudaError_t from the launch; B200RL_ERR_ARG (-1) bad argument;
 *     B200RL_ERR_WORKSPACE (-2) workspace too small for this problem size.
 *   - forward entry points that feed a backward entry point write "saved" tensors the caller keeps alive between
 *     the two calls (the autograd context in the PyTorch binding).
 *   - upstream gradients of the scalar losses are passed as device pointers to single floats (nullable = 0), so a
 *     backward launch never needs a host read.
 *   - forward-written gradients: the forward launch of several losses also writes their gradients for the upstream
 *     gradients the caller EXPECTS -- g_expected, device floats indexed by slot (0 policy, 1 value, 2 entropy, 3 kl), the
 *     loss weights of the training loop -- and records the values it used in g_used.  The backward ("verify") launch
 *     takes the actual upstream gradients: it does nothing when every slot the loss owns is bit-identical to g_used (the
 *     gradients in memory are the right ones), and otherwise recomputes them with the actual values, so the pair is exact
 *     for any upstream gradient.  A null g_used makes the verify launch recompute.  g_hint (nullable) receives the actual
 *     values of the owned slots, for the caller's next forward launch to expect.  Slots a loss does not own read as 0: the
 *     forward launch records them as 0, the verify launch neither compares nor refreshes them.  Each entry point below
 *     names the slots it owns.
 */
#ifndef B200RL_H_
#define B200RL_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define B200RL_API __attribute__((visibility("default")))
#else
#define B200RL_API
#endif

#define B200RL_ERR_ARG (-1)
#define B200RL_ERR_WORKSPACE (-2)

/* library / ABI version (major*100 + minor) and the compute capability the kernels were built for (90 = sm_90a) */
B200RL_API int b200rl_version(void);
B200RL_API int b200rl_built_for_sm(void);
B200RL_API size_t b200rl_workspace_bytes(void);

/* ---- gae: ding/rl_utils/gae.py:25-70 -------------------------------------------------------------------------
 * value, next_value, adv: (T, C); reward, done, traj_flag: (T, C/A)  (A = 1, or the trailing agent dim of the
 * multi-agent case gae.py:56-59).  done / traj_flag nullable (gae.py:51-54: done -> 0, traj_flag -> done).
 * mask_next_value_inplace != 0 reproduces the reference's `next_value *= (1 - done)` side effect (gae.py:61).
 * Bit-exact with the reference loop (separate fp32 mul / add in the same order). */
B200RL_API int b200rl_gae(const float* value, float* next_value, const float* reward, const float* done, const float* traj_flag,
               float* adv, long long T, long long C, long long A, double gamma, double lambda_,
               int mask_next_value_inplace, void* stream);

/* ---- the batch-level pieces around gae in PPOPolicy._forward_learn (ding/policy/ppo.py:274-297), SURVEY section 8f ----
 * adv = gae(value*s, next_value*s, reward, done, traj_flag); unnormalized_return = value*s + adv; value_out = (value*s)/s;
 * return_out = unnormalized_return / s; stats3 = {mean, population variance, count} of unnormalized_return -- the three
 * numbers RunningMeanStd.update (ding/utils/default_helper.py:547-567) needs, instead of the reference's full D2H copy.
 * adv_stats2 = {mean, std(unbiased) + 1e-8} of adv in the same pass -- the `adv_stats` operand of the ppo entry points when
 * the whole batch is one minibatch (ding/policy/ppo.py:304-306); minibatches take theirs from b200rl_adv_stats.
 * value_scale = s = RunningMeanStd.std (0: value_norm off, s = 1 and no scaling).  Every output but adv is nullable.
 * C == 1 (the real learner: ONE sequence of n_sample steps, T <= 24576): one launch of one CTA; the sequence is cut at every
 * traj_flag == 1 and each segment is scanned by its own lane -- bit-identical to the reference loop.  (T, C > 1): the
 * streaming scan of b200rl_gae (value_scale applied on load) plus one elementwise epilogue launch. */
B200RL_API int b200rl_gae_returns(const float* value, float* next_value, const float* reward, const float* done,
                       const float* traj_flag, long long T, long long C, long long A, double gamma, double lambda_,
                       int mask_next_value_inplace, double value_scale, float* adv, float* unnormalized_return,
                       float* value_out, float* return_out, float* stats3, float* adv_stats2, float* workspace,
                       size_t workspace_bytes, void* stream);
/* {mean, std(unbiased) + 1e-8} of x[0..n) as two device floats (ding/policy/ppo.py:304-306: adv.mean(), adv.std() + 1e-8),
 * one launch; pass the result as `adv_stats` to the ppo entry points, or materialise (x - mean) / (std + 1e-8): */
B200RL_API int b200rl_adv_stats(const float* x, long long n, float* stats2, float* workspace, size_t workspace_bytes,
                     void* stream);
B200RL_API int b200rl_normalize(const float* x, const float* stats2, long long n, float* out, void* stream);

/* ---- PPOFPolicy's advantage recompute (ding/policy/ppof.py:160-210) in one call --------------------------------------
 * value, next_value, reward, adv, value_out, return_out: (T, C); done / traj_flag (T, C) nullable as for b200rl_gae.  The
 * inputs are only read.  value_norm selects how the critic's output is decoded before gae and the value / return encoded
 * after it (unnormalized_returns = value + adv, ppof.py:195):
 *   0 'baseline'       value * std, next_value * std on load; value_out = (value * std) / std, return_out = (value * std + adv)
 *                      / std; stats3 = {mean, population variance, count} of return_out -- the array RunningMeanStd.update
 *                      receives (ppof.py:206-208 divides in place).  std > 0.
 *   1 'value_rescale'  value_inv_transform on load (eps = 1e-2); value_out = h(h^-1(value)), return_out = h(h^-1(value) + adv)
 *   2 'symlog'         inv_symlog on load; value_out = symlog(inv_symlog(value)), return_out = symlog(inv_symlog(value) + adv)
 *   3 'popart'         reward -> (reward - mu) / sigma on load, popart_mu / popart_sigma one device float each (read on the
 *                      device); value_out = value, return_out = value + adv
 * adv_stats2 = {mean, std(unbiased) + 1e-8} of adv as for b200rl_gae_returns.  Every output but adv is nullable.
 * C == 1 and T <= 24576 (every PPOF call): one launch.  Otherwise one element-wise decode launch ('value_rescale' / 'symlog':
 * value and next_value into scratch[0, 2 T C); 'popart': reward into scratch[0, T C); 'baseline' needs none: the scan scales
 * on load), the streaming scan of b200rl_gae, and one element-wise epilogue launch; scratch may be null on the one-launch path
 * and for 'baseline'.  B200RL_ERR_ARG before any launch for an unknown value_norm, std <= 0 in 'baseline', a missing mu /
 * sigma in 'popart' or a missing scratch. */
B200RL_API int b200rl_gae_returns_norm(const float* value, const float* next_value, const float* reward, const float* done,
                            const float* traj_flag, long long T, long long C, double gamma, double lambda_,
                            int value_norm, double std, const float* popart_mu, const float* popart_sigma, float* adv,
                            float* value_out, float* return_out, float* stats3, float* adv_stats2, float* scratch,
                            float* workspace, size_t workspace_bytes, void* stream);

/* ---- symlog / inv_symlog: ding/rl_utils/value_rescale.py:37-66, element-wise over n floats -------------------------------
 * mode 0: y = sign(x) * log(|x| + 1);  mode 1: y = sign(x) * (exp(|x|) - 1)  (sign(NaN) = sign(-0) = 0, as torch.sign).
 * The backward is torch's autograd of those expressions for the upstream gradient g:
 *   mode 0: dx = ((g * sign(x)) / (|x| + 1)) * sign(x);  mode 1: dx = ((g * sign(x)) * exp(|x|)) * sign(x)
 * plus sign's zero gradient, so dx = +0 where x = 0.  n == 0 launches nothing. */
B200RL_API int b200rl_value_map_fwd(int mode, const float* x, long long n, float* y, void* stream);
B200RL_API int b200rl_value_map_bwd(int mode, const float* x, const float* g, long long n, float* dx, void* stream);

/* IMPALAPolicy._reshape_data masking (ding/policy/impala.py:316-322) in one elementwise launch: values (T+1, B), rewards /
 * done (T, B) -> values_out[t] = values[t] * (1 - done[t-1]) (t >= 1), weights_out[t] = 1 - done[t-1] (1 at t = 0),
 * rewards_out = rewards * weights_out.  rewards_out / weights_out nullable: the backward pass masks d/d values with the same
 * launch (values = upstream gradient). */
B200RL_API int b200rl_impala_mask(const float* values, const float* rewards, const float* done, long long T, long long B,
                       float* values_out, float* rewards_out, float* weights_out, void* stream);

/* ---- ppo_error: ding/rl_utils/ppo.py:77-140 (policy :143-230, value :233-275, kl :30-54) -----------------------
 * S samples, G rows per sample (1, or the agent dim of ppo.py:199-200,:206-207), N logits.
 * logit_new/logit_old/logit_pretrained(nullable): (S*G, N); action: (S*G) int64;
 * value_new, value_old, adv, return_, weight(nullable): (S).  dual_clip <= 0 means None; kl_type 1|2|3 = 'k1'|'k2'|'k3'.
 * adv_stats (nullable): {mean, std + 1e-8} of the advantage batch as two device floats (b200rl_adv_stats); when given the
 * kernels use (adv - mean) / (std + 1e-8) -- PPOPolicy's advantage normalisation (ding/policy/ppo.py:304-306) -- on load.
 * factor (nullable, (S)): happo_error's per-sample factor (ding/rl_utils/happo.py:124-130): min(surr1, surr2) is multiplied
 * by it before the dual clip; null = ppo_error.
 * out[0..5] = policy_loss, value_loss, entropy_loss, kl_div, approx_kl, clipfrac  (out has room for 8 floats). */
B200RL_API int b200rl_ppo_fwd(const float* logit_new, const float* logit_old, const float* logit_pretrained,
                   const long long* action, const float* value_new, const float* value_old, const float* adv,
                   const float* return_, const float* weight, long long S, long long G, long long N,
                   double clip_ratio, int use_value_clip, double dual_clip, int kl_type, const float* adv_stats,
                   const float* factor, float* out, float* workspace, size_t workspace_bytes, void* stream);
/* gradients of  g_policy*policy_loss + g_value*value_loss + g_entropy*entropy_loss + g_kl*kl_div  w.r.t.
 * logit_new (S*G, N) and value_new (S); autograd tie rules of torch.min/max/clamp reproduced (ppo.py:208-216,:269-272).
 * With g_used / g_hint (both nullable) it is the verify launch of b200rl_ppo_fwd_grad (forward-written gradients; owned
 * slots: policy, value, entropy, and kl with logit_pretrained); a non-null g_used needs b200rl_ppo_fused_supported. */
B200RL_API int b200rl_ppo_bwd(const float* logit_new, const float* logit_old, const float* logit_pretrained,
                   const long long* action, const float* value_new, const float* value_old, const float* adv,
                   const float* return_, const float* weight, long long S, long long G, long long N,
                   double clip_ratio, int use_value_clip, double dual_clip, int kl_type, const float* adv_stats,
                   const float* factor, const float* g_policy, const float* g_value, const float* g_entropy, const float* g_kl,
                   const float* g_used, float* g_hint, float* grad_logit_new, float* grad_value_new, void* stream);
/* Fused forward: the losses of b200rl_ppo_fwd AND the gradients of b200rl_ppo_bwd for the expected upstream gradients
 * g_expected[0..3], in one pass over the batch -- the forward launch of the forward-written gradients (owned slots as
 * b200rl_ppo_bwd, which is its verify launch; g_used has room for 4 floats).
 * Only available where b200rl_ppo_fused_supported(...) returns 1 (G == 1, N <= 32, 16-byte aligned tensors). */
B200RL_API int b200rl_ppo_fwd_grad(const float* logit_new, const float* logit_old, const float* logit_pretrained,
                        const long long* action, const float* value_new, const float* value_old, const float* adv,
                        const float* return_, const float* weight, long long S, long long G, long long N,
                        double clip_ratio, int use_value_clip, double dual_clip, int kl_type, const float* adv_stats,
                        const float* factor, const float* g_expected, float* g_used, float* out, float* grad_logit_new,
                        float* grad_value_new, float* workspace, size_t workspace_bytes, void* stream);
/* Launch geometry of the tile kernel behind b200rl_ppo_fwd / _fwd_grad / _bwd for S rows of N <= 32 logits on a device
 * with sm_count SMs: geometry3 = {CTAs, ring stages, dynamic shared memory bytes}.  verify_only: the check launch of
 * b200rl_ppo_bwd behind a fused forward.  Host arithmetic only. */
B200RL_API int b200rl_ppo_tile_geometry(long long S, long long N, int has_pretrained, int has_weight, int verify_only,
                                        int sm_count, long long* geometry3);
B200RL_API int b200rl_ppo_fused_supported(const float* logit_new, const float* logit_old, const float* logit_pretrained,
                               const long long* action, const float* value_new, const float* value_old,
                               const float* adv, const float* return_, const float* weight,
                               const float* grad_logit_new, long long G, long long N);

/* ---- q_nstep_td_error / q_nstep_td_error_with_rescale: ding/rl_utils/td.py:649-719, :810-867, nstep_return :230-286
 *      and, on the same kernel: bdq_nstep_td_error (:722-789), q_1step / v_1step / v_nstep (:26-72, :529-617) and the
 *      per-step loop of the recurrent Q-learners (ding/policy/r2d2.py:347-369, ngu.py:343-347) as ONE call.
 * S samples with G rows each (G = 1; the agent dim of the multi-agent branch td.py:700-705; the branches of BDQ):
 * q, next_n_q: (S, G, N); action, next_n_action: (S, G) int64; reward: (nstep, S), or (S) when cum_reward; done: (S);
 * weight nullable (S); value_gamma nullable, stride 0 (0-dim tensor / python scalar) or 1 ((S) tensor);
 * gamma_per_sample nullable: the list-gamma form used by NGU (td.py:275-282).
 * rescale != 0 applies value_inv_transform / value_transform (value_rescale.py:4-34) with eps = rescale_eps.
 * criterion: 0 MSELoss, 1 L1Loss, 2 SmoothL1Loss(beta=criterion_param), 3 HuberLoss(delta=criterion_param), all
 * reduction='none'.  group_mean != 0: td_error_per_sample is (S), the mean over the G rows (td.py:788); else (S, G).
 * seq_len = T > 0 selects the sequence form: S = T*B samples in time-major order, reward (T, nstep, B), gamma_per_sample
 * (B); loss = sum_t mean_b(w*td) / (T + 1e-8) and, when priority_out (B) is given, priority_out[b] = priority_mix *
 * max_t|td| + (1 - priority_mix) * sum_t|td| / (T + 1e-8)  (r2d2.py:364-369).
 * ONE launch writes loss (1), td_error_per_sample, dcrit_saved (S, G) for the backward call, the detached n-step target
 * (target_out, nullable) and -- grad_q_unit (S, G, N), nullable -- d loss / d q for a unit upstream gradient.
 * b200rl_qntd_bwd: grad_q = g_loss * dloss/dq + dtd/dq^T g_td (both upstream gradients nullable = 0; g_td shaped like
 * td_error_per_sample).  skip_if_unit != 0: grad_q already holds grad_q_unit; the launch verifies on the device that
 * *g_loss == 1 (and g_td is null) and returns at once, else it recomputes -- exact for any upstream gradient, no host sync. */
B200RL_API int b200rl_qntd_fwd(const float* q, const float* next_n_q, const long long* action, const long long* next_n_action,
                    const float* reward, const float* done, const float* weight, const float* value_gamma,
                    long long value_gamma_stride, const float* gamma_per_sample, long long S, long long G, long long N,
                    int nstep, double gamma, int cum_reward, int rescale, double rescale_eps, int criterion,
                    double criterion_param, int group_mean, long long seq_len, double priority_mix, float* loss,
                    float* td_error_per_sample, float* dcrit_saved, float* target_out, float* grad_q_unit,
                    float* priority_out, float* workspace, size_t workspace_bytes, void* stream);
B200RL_API int b200rl_qntd_bwd(const float* dcrit_saved, const float* weight, const long long* action, const float* g_loss,
                    const float* g_td, long long S, long long G, long long N, int group_mean, long long seq_len,
                    int skip_if_unit, float* grad_q, void* stream);

/* ---- dqfd_nstep_td_error / dqfd_nstep_td_error_with_rescale: ding/rl_utils/td.py:870-983, :986-1090, and R2D3's per-step
 *      loop over them (ding/policy/r2d3.py:322-388) as ONE call.
 * q, next_n_q, new_n_q_one_step: (S, N); action, next_n_action, next_n_action_one_step: (S) int64; reward: (nstep, S), or
 * (S) when cum_reward; done, done_one_step, is_expert: (S) floats; weight nullable (S); value_gamma as for b200rl_qntd_fwd
 * (n-step target only: the 1-step target uses gamma and reward[0], td.py:953-964; with cum_reward reward[0] is sample 0's
 * reward for every sample, as the reference's broadcast gives it).  rescale, rescale_eps, criterion and criterion_param as
 * for b200rl_qntd_fwd; criterion = -1 computes no TD terms (callers with their own criterion apply it to the targets).
 * Per sample: td_n / td_1 = criterion(q_sa, target), JE = is_expert * (max_j(q_j + margin*[j != a]) - q_sa) with the
 * gradient of the max at the first maximal j (td.py:969-972).  Outputs: loss = sum(w*(ln*td_n + l1*td_1 + ls*JE)) / div,
 * td_error_per_sample = ln*|td_n| + l1*|td_1| + ls*|JE|, loss_statistics[3] = (sum td_n, sum td_1, sum JE) / div, where
 * div = S, or with seq_len = T > 0 (S = T*B samples in time-major order, reward (T, nstep, B)) div = B*(T + 1e-8)
 * (r2d3.py:379-383); priority_out (B) nullable, sequence form only: priority_mix * max_t e + (1 - priority_mix) * sum_t e
 * / (T + 1e-8) on the per-sample errors e, without abs (r2d3.py:353, :386-388).  saved (S, 4) floats, 16-byte aligned: the
 * record b200rl_dqfd_bwd needs.  target_n_out / target_1_out (S) nullable: the detached targets.  grad_q_unit (S, N)
 * nullable: d loss / d q for a unit upstream gradient.
 * b200rl_dqfd_bwd: grad_q for the upstream gradients of the loss, td_error_per_sample (S) and the three statistics (each a
 * device pointer, nullable = 0).  skip_if_unit != 0: grad_q already holds grad_q_unit; the launch verifies on the device
 * that only *g_loss == 1 arrived and returns at once, else it recomputes. */
B200RL_API int b200rl_dqfd_fwd(const float* q, const float* next_n_q, const float* new_n_q_one_step, const long long* action,
                    const long long* next_n_action, const long long* next_n_action_one_step, const float* reward,
                    const float* done, const float* done_one_step, const float* weight, const float* value_gamma,
                    long long value_gamma_stride, const float* is_expert, long long S, long long N, int nstep,
                    double gamma, int cum_reward, int rescale, double rescale_eps, int criterion, double criterion_param,
                    double lambda_n_step_td, double lambda_one_step_td, double lambda_supervised_loss, double margin,
                    long long seq_len, double priority_mix, float* loss, float* td_error_per_sample,
                    float* loss_statistics, float* saved, float* target_n_out, float* target_1_out, float* grad_q_unit,
                    float* priority_out, float* workspace, size_t workspace_bytes, void* stream);
B200RL_API int b200rl_dqfd_bwd(const float* saved, const float* weight, const long long* action, const float* g_loss,
                    const float* g_td, const float* g_loss_statistics_n, const float* g_loss_statistics_1,
                    const float* g_loss_statistics_je, long long S, long long N, double lambda_n_step_td,
                    double lambda_one_step_td, double lambda_supervised_loss, long long seq_len, int skip_if_unit,
                    float* grad_q, void* stream);

/* ---- the TD losses of the entropy-regularised value learners, one forward entry point (csrc/td.cu soft_td_fwd_kernel):
 *      mode 0  m_q_1step_td_error (Munchausen DQN): ding/rl_utils/td.py:75-158
 *      mode 1  q_nstep_sql_td_error (soft Q-learning): td.py:1175-1245, nstep_return :230-286
 *      mode 2  q_v_1step_td_error (discrete SAC critic): td.py:161-219
 * S samples with G rows each (G = 1; the agent dim of mode 2's multi-agent branch, td.py:206-217), R = S*G rows.
 * q: (R, N); action: (R) int64; done: (S) floats; weight nullable (R); reward: (S), mode 1 (nstep, S) or (S) when cum_reward.
 * Mode 0: target_q (R, N) is the target network on the current observation, next_q (R, N) on the next one; target = reward
 *   + alpha*clamp(log_pi[a], -1, 1) + gamma * sum_j pi'_j * (next_q_j - tau*log pi'_j) * (1 - done), with log_pi / pi' the
 *   softmax policies of target_q / tau and next_q / tau (row max taken out first); action_gap (1) = mean over R of top-1 minus
 *   top-2 of target_q; clipfrac (R) = 1 where log_pi[a] lies outside [-1, 1].  N >= 2.
 * Mode 1: next_q = next_n_q (R, N); V' = alpha*logsumexp(next_n_q / alpha) with +inf -> 20, -inf -> -20, written to
 *   record_target_v (R, nullable) before the return is formed; the return is nstep_return's (value_gamma as for
 *   b200rl_qntd_fwd) or, with cum_reward, reward + (value_gamma or gamma**nstep) * V' * (1 - done).
 * Mode 2: next_q = v (R); target = gamma * (1 - done) * v + reward.
 * tau and alpha are divided by as fp32 values (true division).  criterion / criterion_param as for b200rl_qntd_fwd.
 * ONE launch writes loss (1) = sum(w*td) / R, td_error_per_sample (R), dcrit_saved (R), the detached target (target_out,
 * nullable) and -- grad_q_unit (R, N), nullable -- d loss / d q for a unit upstream gradient.  Every target is detached, so
 * the backward is b200rl_qntd_bwd(dcrit_saved, weight, action, g_loss, g_td, R, 1, N, 0, 0, skip_if_unit, grad_q). */
B200RL_API int b200rl_soft_td_fwd(int mode, const float* q, const float* target_q, const float* next_q, const long long* action,
                       const float* reward, const float* done, const float* weight, const float* value_gamma,
                       long long value_gamma_stride, long long S, long long G, long long N, int nstep, double gamma,
                       double tau, double alpha, int cum_reward, int criterion, double criterion_param, float* loss,
                       float* td_error_per_sample, float* dcrit_saved, float* target_out, float* grad_q_unit,
                       float* action_gap, float* clipfrac, float* record_target_v, float* workspace,
                       size_t workspace_bytes, void* stream);

/* ---- dist_nstep_td_error (C51): ding/rl_utils/td.py:413-523; dist_1step_td_error (:294-383) is its nstep = 1 case ---
 * dist, next_n_dist: (B*A, N, n_atom); act, next_n_act: (B*A) int64; reward: (nstep, B); done: (B);
 * weight nullable with stride 0 / 1 over the B*A rows; value_gamma nullable with stride 0 / 1 over B;
 * support: (n_atom) = torch.linspace(v_min, v_max, n_atom) as computed by the caller's torch (td.py:457).
 * bad_flag (int, caller-zeroed, nullable) is set when a selected dist entry is <= 0 (the reference's assert, td.py:513).
 * ONE launch writes loss (1), td_error_per_sample (B*A, unweighted, td.py:519), proj_saved (B*A, n_atom) and --
 * grad_dist_unit (B*A, N, n_atom), nullable -- d loss / d dist for a unit upstream gradient.
 * b200rl_dntd_bwd: g_loss / g_td (R) are the upstream gradients of loss / td_error_per_sample (nullable = 0).  skip_if_unit
 * != 0: grad_dist already holds grad_dist_unit; no-op when *g_loss == 1 and g_td is null, else recomputed. */
B200RL_API int b200rl_dntd_fwd(const float* dist, const float* next_n_dist, const long long* act, const long long* next_n_act,
                    const float* reward, const float* done, const float* weight, long long weight_stride,
                    const float* value_gamma, long long value_gamma_stride, const float* support, long long B,
                    long long A, long long N, int n_atom, int nstep, double gamma, double v_min, double v_max,
                    float* loss, float* td_error_per_sample, float* proj_saved, int* bad_flag, float* grad_dist_unit,
                    float* workspace, size_t workspace_bytes, void* stream);
B200RL_API int b200rl_dntd_bwd(const float* dist, const long long* act, const float* proj_saved, const float* weight,
                    long long weight_stride, const float* g_loss, const float* g_td, long long R, long long N,
                    int n_atom, int skip_if_unit, float* grad_dist, void* stream);

/* ---- generalized_lambda_returns / upgo_returns: ding/rl_utils/td.py:1574-1651, upgo.py:46-68 -------------------
 * value: (T+1, B); reward: (T, B); gammas / lambdas nullable (T, B) tensors overriding the scalars; done nullable.
 * upgo_mode != 0: gamma = 1 and lambda_t = [r_{t+1} + V_{t+2} >= V_{t+1}] (last row 1).  ret: (T, B).  Bit-exact. */
B200RL_API int b200rl_lambda_returns(const float* value, const float* reward, const float* gammas, double gamma,
                          const float* lambdas, double lambda_, const float* done, int upgo_mode, long long T,
                          long long B, float* ret, void* stream);
/* Backward of the lambda-return (the reference function is differentiable; MBSAC / Dreamer back-propagate through it,
 * ding/policy/mbpolicy/mbsac.py:137, mbpolicy/utils.py:75): g_ret (T, B) upstream -> grad_value (T+1, B), and, each
 * nullable, grad_reward (T, B), grad_gammas / grad_lambdas (T, B; need the forward result `ret`).  upgo_mode as above
 * (lambda is recomputed from reward / value; no gradient flows through the comparison). */
B200RL_API int b200rl_lambda_returns_bwd(const float* g_ret, const float* value, const float* reward, const float* ret,
                              const float* gammas, double gamma, const float* lambdas, double lambda_,
                              const float* done, int upgo_mode, long long T, long long B, float* grad_value,
                              float* grad_reward, float* grad_gammas, float* grad_lambdas, void* stream);
/* ---- td_lambda_error: ding/rl_utils/td.py:1539-1571 (scan + loss head fused) -----------------------------------
 * writes loss (1) and dvalue_saved (T+1, B) = d loss / d value for unit upstream gradient */
B200RL_API int b200rl_td_lambda_fwd(const float* value, const float* reward, const float* weight, double gamma, double lambda_,
                         long long T, long long B, float* loss, float* dvalue_saved, float* workspace,
                         size_t workspace_bytes, void* stream);
/* out[i] = (*g) * in[i] -- backward of heads whose forward saved the unit-upstream gradient */
B200RL_API int b200rl_scale(const float* g, const float* in, float* out, long long n, void* stream);

/* ---- upgo_loss head: ding/rl_utils/upgo.py:77-111 (tb_cross_entropy :7-43) --------------------------------------
 * logit: (TB*K, N) with K = 1 for (T,B,N) logits or N2 for (T,B,N2,N); action, mask(nullable): (TB*K);
 * rho, ret (from b200rl_lambda_returns upgo mode), value (= bootstrap_values[:-1]): (TB).
 * grad_logit_unit (nullable, logit's shape): the forward launch also writes d loss / d logit for a unit upstream gradient while
 * each row is still in L1 (one pass over the logits instead of two).  b200rl_upgo_head_bwd with skip_if_unit = 1 and that
 * buffer as grad_logit returns at once when *g_loss == 1 and recomputes otherwise. */
B200RL_API int b200rl_upgo_head_fwd(const float* logit, const long long* action, const float* mask, const float* rho,
                         const float* ret, const float* value, long long TB, long long K, long long N, float* loss,
                         float* adv_saved, float* grad_logit_unit, float* workspace, size_t workspace_bytes, void* stream);
B200RL_API int b200rl_upgo_head_bwd(const float* logit, const long long* action, const float* mask, const float* adv_saved,
                         const float* g_loss, long long TB, long long K, long long N, int skip_if_unit, float* grad_logit,
                         void* stream);

/* tb_cross_entropy alone (upgo.py:7-43): ce (TB) = sum_k mask_k * log softmax(logit)[action]; backward for an upstream
 * gradient g_ce (TB). */
B200RL_API int b200rl_tb_cross_entropy_fwd(const float* logit, const long long* action, const float* mask, long long TB,
                                long long K, long long N, float* ce, void* stream);
B200RL_API int b200rl_tb_cross_entropy_bwd(const float* logit, const long long* action, const float* mask, const float* g_ce,
                                long long TB, long long K, long long N, float* grad_logit, void* stream);

/* ---- vtrace_error_discrete_action: ding/rl_utils/vtrace.py:72-136 (returns :9-29, advantage :32-45, isw.py:55-58)
 * target_output, behaviour_output: (T*B, N); action: (T*B) int64; value: (T+1, B); reward, weight(nullable): (T, B).
 * out3 = policy_loss, value_loss, entropy_loss.  lp_saved / cpg_saved / dv_saved: (T, B) scratch kept for backward. */
B200RL_API int b200rl_vtrace_fwd(const float* target_output, const float* behaviour_output, const long long* action,
                      const float* value, const float* reward, const float* weight, long long T, long long B,
                      long long N, double gamma, double lambda_, double rho_clip_ratio, double c_clip_ratio,
                      double rho_pg_clip_ratio, float* out3, float* lp_saved, float* cpg_saved, float* dv_saved,
                      float* workspace, size_t workspace_bytes, void* stream);
B200RL_API int b200rl_vtrace_bwd(const float* target_output, const long long* action, const float* weight,
                      const float* cpg_saved, const float* dv_saved, const float* g_policy, const float* g_value,
                      const float* g_entropy, long long T, long long B, long long N, float* grad_target_output,
                      float* grad_value, void* stream);

/* vtrace_error_continuous_action (ding/rl_utils/vtrace.py:139-212): Independent(Normal(mu, sigma)) target / behaviour
 * policies, mu / sigma / action (T*B, D) floats; otherwise as b200rl_vtrace_fwd / _bwd (rows kernel -> the shared scan ->
 * backward rows kernel; gradients reach mu_target, sigma_target and value). */
B200RL_API int b200rl_vtrace_continuous_fwd(const float* mu_target, const float* sigma_target, const float* mu_behaviour,
                                 const float* sigma_behaviour, const float* action, const float* value,
                                 const float* reward, const float* weight, long long T, long long B, long long D,
                                 double gamma, double lambda_, double rho_clip_ratio, double c_clip_ratio,
                                 double rho_pg_clip_ratio, float* out3, float* lp_saved, float* cpg_saved, float* dv_saved,
                                 float* workspace, size_t workspace_bytes, void* stream);
B200RL_API int b200rl_vtrace_continuous_bwd(const float* mu_target, const float* sigma_target, const float* action,
                                 const float* weight, const float* cpg_saved, const float* dv_saved, const float* g_policy,
                                 const float* g_value, const float* g_entropy, long long T, long long B, long long D,
                                 float* grad_mu, float* grad_sigma, float* grad_value, void* stream);

/* ---- vtrace_error_discrete_action in one launch: ding/rl_utils/vtrace.py:72-136 (returns :9-29, advantages :32-45,
 * importance weights isw.py:55-58), forward AND gradients (csrc/vtws.cu) -------------------------------------------------
 * Same semantics as b200rl_vtrace_fwd followed by b200rl_vtrace_bwd, but the batch crosses HBM once (96 B per transition at
 * N = 6): column tiles, warp-specialised loader / scanner / consumer warps.  Forward-written gradients: verify = 0 is the
 * forward launch (g_expected, g_used), verify = 1 the verify launch (g_policy, g_value, g_entropy, g_used, g_hint); owned
 * slots: policy, value, entropy.  grad_target_output == null (verify = 0 only): losses only.  out3 is written by the
 * verify = 0 launch only.
 * Two kernels behind the entry point: the streaming column tiles (any T; N <= 14 with weights: the stage ring has to fit two
 * CTAs per SM) and, for the rows they cannot take, resident tiles (the T x 8 | 4-column tile of a CTA fits shared memory twice
 * per SM: IMPALA unroll lengths, any N that fits).  Requires b200rl_vtrace_fused_supported(...) == 1 (one of the two fits,
 * B % 4 == 0, 16-byte aligned tensors).  b200rl_vtrace_set_impl: 0 = automatic (default), 1 = streaming column tiles only,
 * 2 = resident tiles wherever they fit; returns the previous value. */
B200RL_API int b200rl_vtrace_set_impl(int impl);
B200RL_API int b200rl_vtrace_fused_supported(const float* target_output, const float* behaviour_output,
                                  const long long* action, const float* value, const float* reward,
                                  const float* weight, long long T, long long B, long long N,
                                  const float* grad_target_output, const float* grad_value);
B200RL_API int b200rl_vtrace_fwd_grad(const float* target_output, const float* behaviour_output, const long long* action,
                           const float* value, const float* reward, const float* weight, long long T, long long B,
                           long long N, double gamma, double lambda_, double rho_clip_ratio, double c_clip_ratio,
                           double rho_pg_clip_ratio, const float* g_expected, int verify, const float* g_policy,
                           const float* g_value, const float* g_entropy, float* g_used, float* g_hint, float* out3,
                           float* grad_target_output, float* grad_value, float* workspace, size_t workspace_bytes,
                           void* stream);

/* ---- ppo_value_error alone (ppo.py:233-275): loss = 0.5 * mean(w * max((R-v)^2, (R-v_clip)^2)) (or the unclipped form)
 * and, when dvalue_unit != null, d loss / d value_new for a unit upstream gradient (backward = b200rl_scale of it).
 * value_new, value_old, return_, weight (nullable = 1): (S). */
B200RL_API int b200rl_ppo_value_fwd(const float* value_new, const float* value_old, const float* return_,
                         const float* weight, long long S, double clip_ratio, int use_value_clip, float* loss,
                         float* dvalue_unit, float* workspace, size_t workspace_bytes, void* stream);

/* ---- compute_q_retraces: ding/rl_utils/retrace.py:7-56 (ACER's Retrace targets; no gradient, as in the reference) -----------
 * q_values, ratio (T+1 | T, B, N) -- row T of q_values is never read; v_pred (T+1, B); rewards / weights (T, B); actions (T, B)
 * int64; q_retraces (T+1, B).  Bit-identical to the reference loop (same fp32 operations in the same order). */
B200RL_API int b200rl_q_retraces(const float* q_values, const float* v_pred, const float* rewards, const long long* actions,
                      const float* weights, const float* ratio, long long T, long long B, long long N, double gamma,
                      float* q_retraces, void* stream);

/* ---- ACER heads: ding/rl_utils/acer.py:8-57 (policy), :60-83 (value), :86-124 (trust region) -- csrc/acer.cu ---------------
 * M = T * B transitions, un-reduced per-transition outputs (ACERPolicy weights and sums them itself, policy/acer.py:247-270).
 * q_values, target_logit (= log pi), ratio: (M, N); q_retraces, v_pred, actor_loss, bias_correction_loss, critic_loss: (M);
 * actions (M) int64.  Gradients: policy -> target_logit (g_actor / g_bias: upstream (M), nullable = 0); value -> q_values.
 * acer_trust_region: out = g - max(((g . k) - delta) / (k . k), 0) * k with k = exp(avg_logit), row by row. */
B200RL_API int b200rl_acer_policy_fwd(const float* q_values, const float* q_retraces, const float* v_pred,
                           const float* target_logit, const long long* actions, const float* ratio, long long M, long long N,
                           double c_clip_ratio, float* actor_loss, float* bias_correction_loss, void* stream);
B200RL_API int b200rl_acer_policy_bwd(const float* q_values, const float* q_retraces, const float* v_pred,
                           const float* target_logit, const long long* actions, const float* ratio, const float* g_actor,
                           const float* g_bias, long long M, long long N, double c_clip_ratio, float* grad_target_logit,
                           void* stream);
B200RL_API int b200rl_acer_value_fwd(const float* q_values, const float* q_retraces, const long long* actions, long long M,
                          long long N, float* critic_loss, void* stream);
B200RL_API int b200rl_acer_value_bwd(const float* q_values, const float* q_retraces, const long long* actions,
                          const float* g_loss, long long M, long long N, float* grad_q_values, void* stream);
B200RL_API int b200rl_acer_trust_region(const float* actor_gradient, const float* avg_logit, long long M, long long N,
                             double trust_region_value, float* out, void* stream);

/* ---- quantile-regression n-step TD: qrdqn_nstep_td_error (ding/rl_utils/td.py:1098-1166, form 0), iqn_nstep_td_error
 * (:1253-1346, form 1), fqf_nstep_td_error (:1359-1436, form 2) -- csrc/quantile.cu, one kernel, the layouts are strides:
 * theta_i = q[b*q_sb + i*q_si + action_b*q_sa] (i < n_tau), theta'_j from next_n_q likewise (j < n_tau_prime),
 * tau_i = tau[b*tau_sb + i*tau_si] (a stride may be 0); reward (nstep, B), done / weight(nullable) (B), value_gamma nullable
 * with element stride vg_stride (0 = one value).  kappa is used by forms 1 and 2 (td.py:1329,:1341,:1431).
 * Writes loss (scalar), td (B) = the per-sample losses, dtheta (B, n_tau) = d td_b / d theta_i and -- grad_q_unit non-null,
 * q's layout -- d loss / d q for a unit upstream gradient.  b200rl_quantile_td_bwd: grad_q = (g_loss * w_b / B + g_td_b) *
 * dtheta scattered to the chosen action (zeros elsewhere); skip_if_unit = 1: grad_q already holds the unit gradient, the
 * launch returns at once when *g_loss == 1 and g_td is null. */
B200RL_API int b200rl_quantile_td_fwd(const float* q, const float* next_n_q, const long long* action,
                           const long long* next_n_action, const float* reward, const float* done, const float* tau,
                           const float* weight, const float* value_gamma, long long vg_stride, long long B, long long N,
                           long long n_tau, long long n_tau_prime, long long nstep, double gamma, long long q_sb,
                           long long q_si, long long q_sa, long long nq_sb, long long nq_sj, long long nq_sa,
                           long long tau_sb, long long tau_si, int form, double kappa, float* loss, float* td,
                           float* dtheta, float* grad_q_unit, float* workspace, size_t workspace_bytes, void* stream);
B200RL_API int b200rl_quantile_td_bwd(const float* dtheta, const float* weight, const long long* action,
                           const float* g_loss, const float* g_td, long long B, long long N, long long n_tau,
                           long long q_sb, long long q_si, long long q_sa, int skip_if_unit, float* grad_q, void* stream);

/* ---- FQF's fraction loss: fqf_calculate_fraction_loss (ding/rl_utils/td.py:1466-1513) -- csrc/quantile.cu.
 * s_i = q_tau_i[b*qt_sb + i*qt_si + a_b*qt_sa] (i < N-1, A_tau actions), h_k = q_value[b*qv_sb + k*qv_si + a_b*qv_sa]
 * (k < N, A_value actions), quantiles[b*qn_sb + k*qn_si] (k <= N); actions (B) int64, an action out of range reads NaN.
 * g_i = (s_i > (i == 0 ? h_0 : s_{i-1}) ? 1 : -1) * (s_i - h_i) + (s_i < (i == N-2 ? h_{N-1} : s_{i+1}) ? 1 : -1) *
 * (s_i - h_{i+1}); writes loss = mean_b sum_i g_i * quantiles[b, i+1] (scalar), g_saved (B, N-1) and -- non-null --
 * grad_quantiles_unit (B, N+1), contiguous: fp32(1/B) * g_i in column i+1, zero in columns 0 and N.
 * b200rl_fqf_fraction_bwd: grad_quantiles (B, N+1) = (*g_loss * fp32(1/B)) * g_i likewise; skip_if_unit = 1: grad_quantiles
 * already holds the unit gradient, the launch returns at once when *g_loss == 1. */
B200RL_API int b200rl_fqf_fraction_fwd(const float* q_tau_i, const float* q_value, const float* quantiles,
                            const long long* actions, long long B, long long N, long long A_tau, long long A_value,
                            long long qt_sb, long long qt_si, long long qt_sa, long long qv_sb, long long qv_si,
                            long long qv_sa, long long qn_sb, long long qn_si, float* loss, float* g_saved,
                            float* grad_quantiles_unit, float* workspace, size_t workspace_bytes, void* stream);
B200RL_API int b200rl_fqf_fraction_bwd(const float* g_saved, const float* g_loss, long long B, long long N,
                            int skip_if_unit, float* grad_quantiles, void* stream);

/* ---- sibling heads (SURVEY section 8f rank 3), forward + gradients in ONE launch each (csrc/heads.cu) ---------------------
 * Forward-written gradients with verify = 0 / 1 as b200rl_vtrace_fwd_grad (grad_* null, verify = 0 only: losses only).
 * Owned slots: policy, value, entropy; ppo_error_continuous also kl with the pretrained pair.
 * a2c_error (ding/rl_utils/a2c.py:10-44): logit (S, N), action (S) int64, value / adv / return_ / weight(nullable) (S);
 * out3 = policy_loss -mean(logp*adv*w), value_loss mean(w*(return_-value)^2), entropy_loss mean(H*w).
 * ppo_error_continuous (ding/rl_utils/ppo.py:278-374): Independent(Normal(mu, sigma)) policies, mu / sigma / action (S, D)
 * (a 1-D old policy is D = 1), pretrained pair nullable; out6 as b200rl_ppo_fwd.  factor (nullable, (S)) selects
 * happo_error_continuous (ding/rl_utils/happo.py:195-284): min(surr1, surr2) * factor before the dual clip, entropy and
 * approx_kl averaged over the S * D per-dimension terms. */
B200RL_API int b200rl_a2c_fwd_grad(const float* logit, const long long* action, const float* value, const float* adv,
                        const float* return_, const float* weight, long long S, long long N, const float* g_expected,
                        int verify, const float* g_policy, const float* g_value, const float* g_entropy, float* g_used,
                        float* g_hint, float* out3, float* grad_logit, float* grad_value, float* workspace,
                        size_t workspace_bytes, void* stream);
B200RL_API int b200rl_ppo_continuous_fwd_grad(
    const float* mu_new, const float* sigma_new, const float* mu_old, const float* sigma_old, const float* mu_pretrained,
    const float* sigma_pretrained, const float* action, const float* value_new, const float* value_old, const float* adv,
    const float* return_, const float* weight, const float* factor, long long S, long long D, double clip_ratio,
    int use_value_clip, double dual_clip, int kl_type, const float* g_expected, int verify, const float* g_policy,
    const float* g_value, const float* g_entropy, const float* g_kl, float* g_used, float* g_hint, float* out6, float* grad_mu,
    float* grad_sigma, float* grad_value, float* workspace, size_t workspace_bytes, void* stream);
/* a2c_error_continuous (ding/rl_utils/a2c.py:50-88): Independent(Normal(mu, sigma)) policy, mu / sigma / action (S, D) float,
 * value / adv / return_ / weight(nullable) (S); out3 and the backward contract as b200rl_a2c_fwd_grad, gradients reach mu,
 * sigma and value. */
B200RL_API int b200rl_a2c_continuous_fwd_grad(const float* mu, const float* sigma, const float* action, const float* value,
                        const float* adv, const float* return_, const float* weight, long long S, long long D,
                        const float* g_expected, int verify, const float* g_policy, const float* g_value,
                        const float* g_entropy, float* g_used, float* g_hint, float* out3, float* grad_mu, float* grad_sigma,
                        float* grad_value, float* workspace, size_t workspace_bytes, void* stream);

/* ppg_joint_error's behavioural-cloning term (ding/rl_utils/ppg.py:62-67): F.kl_div(logp_new, logp_old, 'batchmean') -- the
 * reference passes the old LOG-probability as the non-log target, so the value is NaN whenever an old log-probability is
 * negative while the gradient (-logp_old / B through log-softmax) is finite; both are reproduced.  dlogit_unit (nullable,
 * (B, N)) = d loss / d logit_new for a unit upstream gradient.  The auxiliary value term is b200rl_ppo_value_fwd. */
B200RL_API int b200rl_ppg_bc_fwd(const float* logit_new, const float* logit_old, const long long* action, long long B,
                      long long N, float* loss, float* dlogit_unit, float* workspace, size_t workspace_bytes, void* stream);

/* ---- fused learner step: gae (gae.py:25-70) followed by ppo_error (ppo.py:77-140) in ONE launch ------------------
 * Semantics are exactly b200rl_gae(value, next_value, reward, done, traj_flag -> adv) followed by b200rl_ppo_fwd_grad
 * (or b200rl_ppo_fwd when g_expected is null) with that adv, S = T*B, G = 1 -- same arithmetic, bit-identical adv.
 * value/next_value/reward/done/traj_flag/adv: (T, B); logits: (T*B, N); action/value_new/value_old/return_/weight: (T*B).
 * The advantage rows are produced newest-first and consumed by the PPO tiles in the same order inside the kernel, so the
 * batch crosses HBM once.  Requires b200rl_gae_ppo_supported(...) == 1: 1 <= N <= 32, B >= 4, B % 4 == 0, 16-byte aligned
 * tensors, and either ceil(T/32) * ceil(B/128) <= 4096 (row tiles) or a ring of two stages fits (column tiles: N <= 21, or
 * N <= 14 with logit_pretrained). */
B200RL_API int b200rl_gae_ppo_supported(const float* value, const float* next_value, const float* reward,
                             const float* done, const float* traj_flag, long long T, long long B,
                             const float* logit_new, const float* logit_old, const float* logit_pretrained,
                             const long long* action, const float* value_new, const float* value_old,
                             const float* return_, const float* weight, long long N, const float* adv,
                             const float* grad_logit_new);
B200RL_API int b200rl_gae_ppo_fwd_grad(const float* value, float* next_value, const float* reward, const float* done,
                            const float* traj_flag, long long T, long long B, double gamma, double lambda_,
                            int mask_next_value_inplace, const float* logit_new, const float* logit_old,
                            const float* logit_pretrained, const long long* action, const float* value_new,
                            const float* value_old, const float* return_, const float* weight, long long N,
                            double clip_ratio, int use_value_clip, double dual_clip, int kl_type,
                            const float* g_expected, float* g_used, float* adv, float* out, float* grad_logit_new,
                            float* grad_value_new, float* workspace, size_t workspace_bytes, void* stream);
/* The same step in data-parallel training (B sharded across ranks, SURVEY section 8e): the six loss scalars out[0..5] are
 * exchanged by launches the step makes anyway -- no extra launch, no collective call, nothing on the critical path.  Step q's
 * loss-finalisation launch stages {q, out[k]} locally; step q+1's streaming kernel (six warps of its first CTA, while they
 * would wait for their first chunk anyway) consumes the entries tagged q-1 of all ranks from this rank's mailbox into
 * out_mean and publishes the staged word to every peer's mailbox over NVLink (one 8-byte store per peer and value; the
 * acknowledgements return while the kernel streams).  out_mean[0..5] = mean over ranks of the latest consumed step (mean of
 * the rank means, ding/utils/pytorch_ddp_dist_helper.py:38-47), two steps behind out; out_mean[8..13] the step before.
 * mailbox_ptrs_dev: device array of `world` (<= 32) mailbox base addresses as seen from THIS process (peer-mapped symmetric
 * memory), each b200rl_p2p_mailbox_floats(world) floats, zero-initialised; seq_dev: 24 32-bit device words and out_mean: 16
 * floats, zero-initialised, owned by this exchange; every rank must make the same sequence of calls.  After the last step
 * b200rl_p2p_drain_mean publishes / consumes the tail: out_mean[0..5] = the LAST step's mean, out_mean[8..13] the one before.
 * Requires the column-tile kernel (b200rl_gae_ppo_supported, B >= 16) and P2P access between the ranks' GPUs. */
B200RL_API int b200rl_gae_ppo_fwd_grad_dp(const float* value, float* next_value, const float* reward, const float* done,
                               const float* traj_flag, long long T, long long B, double gamma, double lambda_,
                               int mask_next_value_inplace, const float* logit_new, const float* logit_old,
                               const float* logit_pretrained, const long long* action, const float* value_new,
                               const float* value_old, const float* return_, const float* weight, long long N,
                               double clip_ratio, int use_value_clip, double dual_clip, int kl_type,
                               const float* g_expected, float* g_used, float* adv, float* out, float* grad_logit_new,
                               float* grad_value_new, const unsigned long long* mailbox_ptrs_dev, int rank, int world,
                               unsigned int* seq_dev, float* out_mean, float* workspace, size_t workspace_bytes,
                               void* stream);
B200RL_API int b200rl_p2p_drain_mean(const unsigned long long* mailbox_ptrs_dev, int rank, int world, int n,
                          unsigned int* seq_dev, float* out_mean, void* stream);
/* Kernels behind the calls above (gae, ding/rl_utils/gae.py:25-70, followed by ppo_error, ding/rl_utils/ppo.py:77-140).
 * Column tiles: a CTA owns 16 batch columns for all T and runs their scan and their
 * ppo_error rows -- no cross-CTA dependency; csrc/colws.cu (warp-specialised loader / scanner / consumer warps on an
 * mbarrier pipeline, cp.async copies).  Chosen when B >= 1024 or T*B <= 16384 and its ring fits two CTAs per SM.  Row tiles:
 * csrc/fused.cu (scan CTAs publish 32-step chunks that the PPO tiles of all CTAs consume); every other supported call.
 * impl: 0 automatic (default), 1 row tiles, 2 column tiles, each where it can take the call; returns the previous setting
 * (or B200RL_ERR_ARG for any other value).  Test hook, process-wide: runs each kernel on every shape. */
B200RL_API int b200rl_gae_ppo_set_impl(int impl);

/* ---- language-model policy losses on vocabulary-scale logits (csrc/vocab.cu) -------------------------------------
 * grpo_policy_error (ding/rl_utils/grpo.py), rloo_policy_error (ding/rl_utils/rloo.py) and the per-token log-probability
 * methods of ding/rl_utils/log_prob_utils.py.  Logits are (rows, V) row-major in the dtype given by `dtype`
 * (B200RL_DTYPE_F32 or B200RL_DTYPE_BF16; every logit pointer of a call in that dtype, 16-byte aligned); all arithmetic is
 * fp32.  Rows are the B*S tokens, row = b*S + s.  action / index: (rows) int64.  weight nullable (B, S) = ones.
 *
 * b200rl_grpo_fwd_grad: logit_new, logit_old, logit_ref (B, S, V), adv (B).  out3 = {loss, approx_kl, clipfrac}:
 *   loss = mean_b(sum_s(w * l) / sum_s(w)), l = -min(r*adv, clamp(r, 1-clip, 1+clip)*adv) + beta*(exp(d) - d - 1),
 *   r = exp(lp_new - lp_old), d = lp_ref - lp_new; approx_kl = mean(lp_old - lp_new); clipfrac = mean(r > 1+clip or
 *   r < 1-clip).  Saved for the backward: lse_new (rows) = logsumexp(logit_new[row]) and dlogp_unit (rows) =
 *   d loss / d lp_new for a unit upstream gradient.  grad_logit_new (nullable = no gradient; dtype of the logits) =
 *   dlogp_unit[row] * (onehot(a) - softmax(logit_new[row])).
 * b200rl_rloo_fwd_grad: as GRPO without logit_ref and beta; the advantage of row b is computed from reward (K, B / K):
 *   (k, j) = (b / (B/K), b % (B/K)), adv = r[k, j] - (sum_k' r[k', j] - r[k, j]) / (K - 1).
 * b200rl_token_logp_fwd: logp (rows) = z[a] - logsumexp(z), lse (rows) saved for the backward.
 * b200rl_token_logp_bwd: grad_logits[row] = g * dlogp[row] * (onehot(a) - softmax(z)), g = *g_scale (nullable = 1).
 *   skip_if_unit != 0: grad_logits already holds the gradient for g = 1 (written by a forward above); the launch returns
 *   at once on the device when *g_scale == 1, else it recomputes -- the backward of GRPO / RLOO, with no host sync.
 * b200rl_token_head_fwd: the GRPO (logp_ref != null, adv) or RLOO (logp_ref null, reward / K) head alone on per-token
 *   log-probabilities (B, S) fp32 that the caller computed; out3 and dlogp_unit as above (backward = b200rl_scale).
 * b200rl_ppo_lm_fwd_grad: ppo_policy_error (ding/rl_utils/ppo.py:143-230) on token rows: logit_new, logit_old,
 *   logit_pretrained (nullable = no KL) (rows, V); adv, weight (rows).  M = rows.  out5 = {policy_loss, entropy_loss,
 *   kl_div, approx_kl, clipfrac}: policy_loss = mean(-sel * w), sel = min(r*adv, clamp(r, 1-clip, 1+clip)*adv) (with
 *   dual_clip > 0 and adv < 0: max(sel, dual_clip*adv)), r = exp(lp_new - lp_old); entropy_loss = mean(H * w) with H the
 *   entropy of softmax(logit_new[row]) (entropy = 0: not computed, 0); kl_div = mean(k(lp_new - lp_pre)), k1 = x,
 *   k2 = x^2 / 2, k3 = exp(-x) - 1 + x (0 without logit_pretrained); approx_kl = mean(lp_old - lp_new); clipfrac =
 *   mean(r > 1+clip or r < 1-clip).  Saved for the backward: lse_new (rows), entropy_row (rows, only with entropy) = H,
 *   dlogp_policy (rows) = (-w / M) * dsel/dr * r and dlogp_kl (rows, only with logit_pretrained) = dk/dx / M.
 *   grad_logit_new (nullable = no gradient; dtype of the logits) = c_act * (onehot(a) - p) - c_ent * p * (log p + H),
 *   p = softmax(logit_new[row]), log p clamped at -FLT_MAX, c_act = g_pol * dlogp_policy + g_kl * dlogp_kl,
 *   c_ent = g_ent * w / M, for the expected upstream gradients g_expected (forward-written gradients; owned slots: policy,
 *   entropy with `entropy`, kl with logit_pretrained; g_expected and g_used hold 4 floats).
 * b200rl_ppo_lm_bwd: the same gradient for the actual upstream gradients g_policy, g_entropy, g_kl (device scalars,
 *   nullable = 0) from the saved rows (entropy_row / dlogp_kl null = no entropy / KL term): one read of logit_new, one
 *   write.  The verify launch of b200rl_ppo_lm_fwd_grad (g_used, g_hint nullable; owned slots: policy, entropy with
 *   entropy_row, kl with dlogp_kl).
 * b200rl_a2c_lm_fwd_grad: a2c_error (ding/rl_utils/a2c.py:10-44) on token rows: logit (rows, V); action, value, adv,
 *   return_, weight (rows) fp32.  M = rows.  out3 = {policy_loss, value_loss, entropy_loss}: policy_loss =
 *   mean(-lp * adv * w), lp = z[a] - logsumexp(z); value_loss = mean((return_ - value)^2 * w); entropy_loss = mean(H * w)
 *   with H the entropy of softmax(logit[row]).  Saved for the backward (all (rows) fp32): lse, entropy_row = H,
 *   dlogp_policy = -adv * w / M and dvalue = -2 * w * (return_ - value) / M.  grad_logit (nullable = no gradient; dtype
 *   of the logits) = c * (onehot(a) - p) - c_ent * p * (log p + H), p = softmax(logit[row]), log p clamped at -FLT_MAX,
 *   c = g_pol * dlogp_policy, c_ent = g_ent * w / M; grad_value (rows) fp32 = g_val * dvalue, given with grad_logit; both
 *   for the expected upstream gradients g_expected (forward-written gradients; owned slots: policy, value, entropy;
 *   g_expected and g_used hold 4 floats).
 * b200rl_a2c_lm_bwd: the same gradients for the actual upstream gradients g_policy, g_value, g_entropy (device scalars,
 *   nullable = 0) from the saved rows.  The verify launch of b200rl_a2c_lm_fwd_grad (g_used, g_hint nullable; owned slots:
 *   policy, value, entropy): it returns at once when all three match g_used; grad_value is rewritten whenever they do not,
 *   and grad_logit (one read of logit, one write) only when the policy or entropy slot differs. */
#define B200RL_DTYPE_F32 0
#define B200RL_DTYPE_BF16 1
B200RL_API int b200rl_grpo_fwd_grad(int dtype, const void* logit_new, const void* logit_old, const void* logit_ref,
                         const long long* action, const float* adv, const float* weight, long long B, long long S,
                         long long V, double clip_ratio, double beta, float* out3, float* lse_new, float* dlogp_unit,
                         void* grad_logit_new, float* workspace, size_t workspace_bytes, void* stream);
B200RL_API int b200rl_rloo_fwd_grad(int dtype, const void* logit_new, const void* logit_old, const long long* action,
                         const float* reward, long long K, const float* weight, long long B, long long S, long long V,
                         double clip_ratio, float* out3, float* lse_new, float* dlogp_unit, void* grad_logit_new,
                         float* workspace, size_t workspace_bytes, void* stream);
B200RL_API int b200rl_token_logp_fwd(int dtype, const void* logits, const long long* index, long long rows, long long V,
                          float* logp, float* lse, void* stream);
B200RL_API int b200rl_token_logp_bwd(int dtype, const void* logits, const long long* index, const float* lse,
                          const float* dlogp, const float* g_scale, int skip_if_unit, long long rows, long long V,
                          void* grad_logits, void* stream);
B200RL_API int b200rl_token_head_fwd(const float* logp_new, const float* logp_old, const float* logp_ref, const float* adv,
                          const float* reward, long long K, const float* weight, long long B, long long S,
                          double clip_ratio, double beta, float* out3, float* dlogp_unit, float* workspace,
                          size_t workspace_bytes, void* stream);
B200RL_API int b200rl_ppo_lm_fwd_grad(int dtype, const void* logit_new, const void* logit_old,
                           const void* logit_pretrained, const long long* action, const float* adv, const float* weight,
                           long long rows, long long V, double clip_ratio, double dual_clip, int kl_type, int entropy,
                           const float* g_expected, float* g_used, float* out5, float* lse_new, float* entropy_row,
                           float* dlogp_policy, float* dlogp_kl, void* grad_logit_new, float* workspace,
                           size_t workspace_bytes, void* stream);
B200RL_API int b200rl_ppo_lm_bwd(int dtype, const void* logit_new, const long long* action, const float* weight,
                      long long rows, long long V, const float* lse_new, const float* entropy_row,
                      const float* dlogp_policy, const float* dlogp_kl, const float* g_policy, const float* g_entropy,
                      const float* g_kl, const float* g_used, float* g_hint, void* grad_logit_new, void* stream);
B200RL_API int b200rl_a2c_lm_fwd_grad(int dtype, const void* logit, const long long* action, const float* value,
                           const float* adv, const float* return_, const float* weight, long long rows, long long V,
                           const float* g_expected, float* g_used, float* out3, float* lse, float* entropy_row,
                           float* dlogp_policy, float* dvalue, void* grad_logit, float* grad_value, float* workspace,
                           size_t workspace_bytes, void* stream);
B200RL_API int b200rl_a2c_lm_bwd(int dtype, const void* logit, const long long* action, const float* weight,
                      long long rows, long long V, const float* lse, const float* entropy_row, const float* dlogp_policy,
                      const float* dvalue, const float* g_policy, const float* g_value, const float* g_entropy,
                      const float* g_used, float* g_hint, void* grad_logit, float* grad_value, void* stream);

/* ---- data-parallel exchange step: one-shot all-reduce (mean) of n <= 8 floats over NVLink peer memory -----------
 * Replaces the small-message NCCL all-reduce of the packed loss scalars (mean of rank means,
 * ding/utils/pytorch_ddp_dist_helper.py:38-47).  mailbox_ptrs_dev: device array of `world` pointers, entry r = the
 * address (in THIS process) of rank r's mailbox of b200rl_p2p_mailbox_floats(world) floats in peer-mapped (symmetric)
 * memory, zero-initialised; seq_dev: device counter, zero-initialised, advanced by every call (all ranks must call in
 * the same order).  out[j] = mean over ranks of local[j], bit-identical on every rank.  One small CTA; graph-capturable. */
B200RL_API int b200rl_p2p_allreduce_mean(const float* local, const unsigned long long* mailbox_ptrs_dev, int rank,
                              int world, int n, unsigned int* seq_dev, float* out, void* stream);
B200RL_API size_t b200rl_p2p_mailbox_floats(int world);

/* ---- calibration probe (not an operator): persistent float4 copy of n_floats (multiple of 4) -------------------- */
B200RL_API int b200rl_probe_copy(const float* src, float* dst, long long n_floats, int ctas_per_sm, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200RL_H_ */
