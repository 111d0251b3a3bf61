/* omnisafe_b200 -- C ABI of the H100-native on-policy SafeRL hot path.
 *
 * The reference (PKU-Alignment/omnisafe) is pure Python: its seam for this path is the set of
 * Python methods listed below, not an FFI.  Each entry point here is what a ctypes binding of the
 * corresponding reference method body would call (see INTEGRATION.md for the stub).  All pointers
 * are DEVICE pointers to contiguous row-major arrays the caller owns; `stream` is a cudaStream_t
 * (NULL = default stream).  Every function returns 0 on success, non-zero on failure;
 * osb_last_error() returns the reason.  No function synchronises the host unless stated.
 * Host-side state (kernel attributes set once, the FOCOPS / P3O scratch scalar, the P2P step counter, the
 * last-error string) is per process: call the entry points from ONE host thread per device, one
 * process per GPU -- the way the reference's `distributed.fork` runs it.
 *
 * Slab layout ("time-major"): per-step scalars are [T][N] (env index contiguous), observations
 * [T][N][O], actions [T][N][A].  Sample k of the reference's env-major order
 * (vector_onpolicy_buffer.py:L125-129, k = i*T + t) lives at slab row t*N + i.
 *
 * Flat parameter vector theta = [actor | reward_critic | cost_critic], each in the reference's
 * named_parameters() order (utils/tools.py:L35-129): actor = log_std[A], W1[64][O], b1[64],
 * W2[64][64], b2[64], W3[A][64], b3[A]; critic = W1, b1, W2, b2, W3[1][64], b3[1].
 */
#ifndef OMNISAFE_B200_H
#define OMNISAFE_B200_H

#ifdef __cplusplus
extern "C" {
#endif

/* ---- plumbing ---------------------------------------------------------------------------- */
const char* osb_last_error(void);
int osb_abi_version(void);

/* Hidden-layer activations (model_cfgs.actor / critic.activation) and real hidden widths (1..64, the networks being
 * zero-padded 64-wide tiles) of the networks the following launches compute, process-wide until changed.  Default:
 * tanh, [64, 64].  Every launch of a network's kernels reads the spec when it is enqueued, so a model sets its own
 * before its launches; a captured graph keeps the spec it was captured with.  Sigmoid and softplus units past a layer's
 * width output +0, so the pads of a narrower network stay exact. */
#define OSB_ACT_TANH 0
#define OSB_ACT_IDENTITY 1
#define OSB_ACT_RELU 2
#define OSB_ACT_SIGMOID 3
#define OSB_ACT_SOFTPLUS 4
int osb_set_net_spec(int actor_act, int critic_act, int a1, int a2, int c1, int c2);
/* kernels launched by this library in this process so far (bench.py counts its timed region with it) */
long long osb_launch_count(void);
int osb_device_info(int device, int* sm_count, int* cc_major, int* cc_minor);

/* ---- dual GAE (segmented reverse scan) ----------------------------------------------------
 * replaces OnPolicyBuffer.finish_path            omnisafe/common/buffer/onpolicy_buffer.py:L148-203
 *          _calculate_adv_and_value_targets('gae')                                     :L299-303
 *          discount_cumsum (fp64 carry)           omnisafe/utils/math.py:L59-82
 * flags bit0 = terminated, bit1 = truncated; a path also ends at t == T-1.  At a path end the
 * bootstrap value is 0 if terminated, else boot_{r,c}[t][i].  disc_ret may be NULL.
 * workspace: osb_gae_workspace_doubles(N) doubles.  sums[4] <- {sum adv_r, sum adv_r^2,
 * sum adv_c, count} over this rank's samples (fp64; all-reduce them across ranks, then call
 * osb_adv_moments). */
int osb_gae_workspace_doubles(int n_envs);
int osb_gae_dual(const float* rew, const float* cost, const float* val_r, const float* val_c,
                 const unsigned char* flags, const float* boot_r, const float* boot_c, int T, int N,
                 double gamma, double lam, double lam_c, double penalty_coef, float* adv_r,
                 float* adv_c, float* tv_r, float* tv_c, float* disc_ret, double* workspace,
                 double* sums, void* stream);
/* osb_gae_dual with the reference's other advantage estimators (onpolicy_buffer.py:L299-331):
 * estimator 0 = 'gae', 1 = 'gae-rtg' (targets = discounted reward-to-go of the penalised path incl.
 * its bootstrap slot), 2 = 'plain' (advantage = one-step delta, targets = reward-to-go), 3 = 'vtrace'
 * (on-policy V-trace, rho = c = 1: targets v_t = V_t + delta_t + gamma (v_{t+1} - V_{t+1}), advantage
 * r_t + gamma v_{t+1} - V_t; fp32 replay of the reference recurrence from an fp64 scan carry).
 * For 1 / 2 disc_ret shares the reward-to-go scan: pass NULL unless penalty_coef == 0. */
int osb_adv_estimate(const float* rew, const float* cost, const float* val_r, const float* val_c,
                     const uint8_t* flags, const float* boot_r, const float* boot_c, int T, int N,
                     double gamma, double lam, double lam_c, double penalty_coef, int estimator,
                     float* adv_r, float* adv_c, float* tv_r, float* tv_c, float* disc_ret,
                     double* workspace, double* sums, void* stream);
/* moments[4] <- {mean_r, std_r + 1e-8, mean_c, 1}: the statistics VectorOnPolicyBuffer.get()
 * standardises with (vector_onpolicy_buffer.py:L131-136, utils/distributed.py:L382-388). */
int osb_adv_moments(const double* sums, int standardize_r, int standardize_c, float* moments,
                    void* stream);
/* out_r = (adv_r - mean_r) / (std_r + 1e-8), out_c = adv_c - mean_c  (what get() returns). */
int osb_adv_standardize(const float* adv_r, const float* adv_c, const float* moments, long long n,
                        float* out_r, float* out_c, void* stream);
/* discount_cumsum over `rows` independent vectors of length `len` (utils/math.py:L59-82);
 * x is fp32 (x_is_f64 = 0) or fp64, out is fp64. */
int osb_discount_cumsum(const void* x, int x_is_f64, int rows, int len, double discount,
                        double* out, void* stream);

/* ---- rollout: fused env step + 3 MLP forwards + sample + slab append ------------------------
 * replaces, per step, ConstraintActorCritic.step  models/actor_critic/constraint_actor_critic.py:L84-109
 *          ActionScale.step / ObsNormalize.step    envs/wrapper.py:L510-514, L231-241
 *          Normalizer.normalize / _push            common/normalizer.py:L88-139
 *          VectorOnPolicyBuffer.store              common/buffer/vector_onpolicy_buffer.py:L96-99
 *          the per-env done loop                   adapter/onpolicy_adapter.py:L114-136
 * Env state arrays: s_raw[2][N][O], final_raw[2][N][O], ep_step[N], episode[N], gstep[N],
 * ep_ret[N], ep_cost[N], ep_len[N], bias[O].  Normaliser state: mean/sumsq/std/mean1/std1 [O],
 * count[2], acc_all[2][O], acc_fin[2][O] (int64 fixed point), fin_count[1], had_fin[1], ticket[1]
 * (all zero-initialised by the caller).  osb_env_reset = OnPolicyAdapter.reset() at epoch start
 * (onpolicy_adapter.py:L80).  osb_rollout_step with t in [0, T) performs step t; t == T is the
 * epoch-end bootstrap launch (critics only).  eps = [N][A] standard-normal draws of this step
 * (parity mode) or NULL (in-kernel Philox keyed by noise_seed / global_step).  precision: 0 = exact
 * fp32 FMA tiles (parity), 1 = TF32 wgmma tiles of 128 envs (O <= 64; falls back to 0 otherwise). */
int osb_env_reset(int O, int A, int max_episode_steps, unsigned seed, unsigned term_threshold,
                  unsigned env_id_offset, float cost_threshold, int obs_normalize, int N,
                  float* s_raw, float* final_raw, int* ep_step, unsigned* episode, unsigned* gstep,
                  float* ep_ret, float* ep_cost, int* ep_len, const float* bias,
                  float* norm_mean, float* norm_sumsq, float* norm_std, float* norm_mean1,
                  float* norm_std1, long long* norm_count, long long* acc_all, long long* acc_fin,
                  int* fin_count, int* had_fin, unsigned* ticket, void* stream);
int osb_rollout_step(int O, int A, int max_episode_steps, unsigned seed, unsigned term_threshold,
                     unsigned env_id_offset, float cost_threshold, int obs_normalize, int N, int T,
                     int t, float* s_raw, float* final_raw, int* ep_step, unsigned* episode,
                     unsigned* gstep, float* ep_ret, float* ep_cost, int* ep_len, const float* bias,
                     float* norm_mean, float* norm_sumsq, float* norm_std, float* norm_mean1,
                     float* norm_std1, long long* norm_count, long long* acc_all,
                     long long* acc_fin, int* fin_count, int* had_fin, unsigned* ticket,
                     float* obs, float* act, float* logp, float* rew, float* cost, float* val_r,
                     float* val_c, float* boot_r, float* boot_c, unsigned char* flags, float* epfin,
                     const float* theta, const float* eps, unsigned noise_seed,
                     unsigned global_step, int precision, void* stream);
/* Whole-epoch rollout in one call: reset, T step launches (eps_all = [T][N][A] or NULL), the
 * epoch-end bootstrap launch and the episode window (= OnPolicyAdapter.rollout,
 * adapter/onpolicy_adapter.py:L58-136).  Philox counter = epoch_index * T + t. */
int osb_rollout_epoch(int O, int A, int max_episode_steps, unsigned seed, unsigned term_threshold,
                      unsigned env_id_offset, float cost_threshold, int obs_normalize, int N, int T,
                      float* s_raw, float* final_raw, int* ep_step, unsigned* episode,
                      unsigned* gstep, float* ep_ret, float* ep_cost, int* ep_len, const float* bias,
                      float* norm_mean, float* norm_sumsq, float* norm_std, float* norm_mean1,
                      float* norm_std1, long long* norm_count, long long* acc_all,
                      long long* acc_fin, int* fin_count, int* had_fin, unsigned* ticket,
                      float* obs, float* act, float* logp, float* rew, float* cost, float* val_r,
                      float* val_c, float* boot_r, float* boot_c, unsigned char* flags, float* epfin,
                      const float* theta, const float* eps_all, unsigned noise_seed,
                      unsigned epoch_index, int W, float* ring, int* meta, double* window_sums,
                      int precision, void* stream);
/* Saute / Simmer mode of the following osb_env_reset / osb_rollout_* calls (SauteAdapter.step / reset,
 * adapter/saute_adapter.py:L135-217; SimmerAdapter.reset, simmer_adapter.py:L97-111): safety = [2][N] device floats (the
 * safety state z by step parity) or NULL for the plain OnPolicyAdapter.  The networks then take O + 1 inputs
 * ([normalised obs | z], theta sized accordingly) and the obs slab rows are O + 1 wide; z starts an epoch at safety_init,
 * z <- (z - cost / safety_budget) / saute_gamma per step, the stored reward is unsafe_reward once z <= 0, z <- 1 at
 * episode ends.  Process-wide until changed. */
int osb_rollout_set_saute(float* safety, float safety_budget, float saute_gamma, float unsafe_reward, float safety_init);
/* EarlyTerminated mode of the following osb_rollout_* calls (EarlyTerminatedAdapter.step,
 * adapter/early_terminated_adapter.py:L56-98, per env): cost_acc = [N] device floats holding the accumulated cost (not cleared
 * by ordinary episode ends) or NULL; once it exceeds cost_limit the step stores reward 0 and terminated = 1, the env is reset
 * and the accumulator cleared.  Process-wide until changed. */
int osb_rollout_set_early_termination(float* cost_acc, float cost_limit);
/* Logger window of the last <= W finished episodes in (step, env) order
 * (common/logger.py:L253-282, adapter/onpolicy_adapter.py:L159-175).  ring[3][W], meta[2] persist
 * across epochs; window_sums[4] <- {sum EpRet, sum EpCost, sum EpLen, count} (fp64). */
int osb_episode_window(const unsigned char* flags, const float* epfin, int T, int N, int W,
                       float* ring, int* meta, double* window_sums, void* stream);
/* ---- evaluation of a saved policy on the synthetic env (Evaluator.evaluate, omnisafe/evaluator.py:L399-490) ---------
 * N envs (seed, env id offset 0), env e runs episodes e, e + N, ... of num_episodes (N <= num_episodes) with the
 * deterministic action (the mean, the bits osb_policy_step gives without eps) and ActionScale.  Per step, as
 * ObsNormalize pushes them: the final observations of envs whose env episode ended, the next observations of every env
 * still running (an env that ended hands back its auto-reset observation), then the observations of the envs reset after
 * the step.  N == 1 resets the env after every episode (the reference calls env.reset()); N > 1 only resets an env whose
 * episode was cut by the cost rule.  Episode sums in fp64: return += reward, cost += cost_criteria^length * cost; early:
 * the episode also ends once that cost >= cost_limit (PPOEarlyTerminated).  safety = [2][N] device floats or NULL:
 * Saute / Simmer, z (column O of the network input) starts every episode at 1, z <- (z - cost / safety_budget) /
 * saute_gamma after every step, the reward is never replaced.  The env and normaliser arrays are those of
 * osb_rollout_step (the normaliser holds the loaded statistics; on return it holds the drifted ones).  Workspace,
 * zeroed by the caller except left[e] = episodes of env e and ctr[0] = N: left, done_eps, len [N] ints, ret, cost [N]
 * doubles, acc_rst [2][O] long longs, ctr [3] ints.  Results: out_ret / out_cost [num_episodes] doubles, out_len ints, in
 * episode order.  act_out = [N][A] floats or NULL: the deterministic action of each env in the last step it ran.
 * Precision 1 / 2 with O (+ 1 with safety) <= 64 run the tensor-core tiles, everything else the fp32 tiles.  On the
 * tensor-core tiles, when the ceil(N / 128) CTAs fit on the SMs and per_step == 0, ONE cooperative launch runs every step
 * with a grid barrier per step and ends when every env has finished; otherwise one launch per step, and the host reads
 * the 4-byte done word ctr[0] (envs still running) every 16 steps -- its only synchronisation.  Both give the same bits. */
int osb_eval_synthetic(int O, int A, int max_episode_steps, unsigned seed, unsigned term_threshold, float cost_threshold,
                       int obs_normalize, int N, int num_episodes, float* s_raw, float* final_raw, int* ep_step,
                       unsigned* episode, unsigned* gstep, float* ep_ret, float* ep_cost, int* ep_len, const float* bias,
                       float* norm_mean, float* norm_sumsq, float* norm_std, float* norm_mean1, float* norm_std1,
                       long long* norm_count, long long* acc_all, long long* acc_fin, int* fin_count, int* had_fin,
                       unsigned* ticket, float* safety, float safety_budget, float saute_gamma, int early,
                       double cost_limit, double cost_criteria, int* left, int* done_eps, double* ret, double* cost,
                       int* len, long long* acc_rst, int* ctr, double* out_ret, double* out_cost, int* out_len,
                       float* act_out, const float* theta, int precision, int per_step, void* stream);
/* Evaluation on a registered env (a user CMDP stepped in PyTorch), same semantics and workspace (acc_rst unused).
 * Per episode schedule: env.reset() -> osb_eval_ext_observe(is_reset = 1, t = -1); for t = 0, 1, ...:
 * osb_eval_ext_act(t) -> env.step(act_env) -> osb_eval_ext_observe(t); then read ctr: ctr[0] == 0 ends the evaluation,
 * ctr[2] > 0 (N == 1: the episode ended and another follows) asks for env.reset() -> osb_eval_ext_observe(is_reset = 1, t).
 * N > 1 relies on the envs resetting themselves (an episode the cost rule cuts: osb_eval_ext_observe_rst below).  osb_eval_ext_act: ObsNormalize, the deterministic forward, act_env[N][A]
 * <- ActionScale onto [act_lo, act_hi] (as osb_ext_act), act_out as above; no slabs.  osb_eval_ext_observe: the fp64
 * sums, Saute z, the cost rule and the episode ends of the running envs; next_obs -> s_raw (the buffer step t + 1
 * reads); ObsNormalize pushes the final rows of running envs (final_obs / final_mask may be NULL), then the next rows
 * of running envs (reset: the rows of envs with episodes left) from fp64 per-tile moments combined in tile order.
 * workspace: osb_eval_ext_workspace_doubles(O, N) doubles, the same size as osb_ext_workspace_doubles (one layout for
 * every fp64 push, so this workspace also serves osb_ext_reset_rows); nonfinite as for osb_ext_observe. */
int osb_eval_ext_workspace_doubles(int O, int N);
int osb_eval_ext_act(int O, int A, int obs_normalize, int N, int t, const float* s_raw, const float* norm_mean,
                     const float* norm_std, const long long* norm_count, const float* safety, const float* theta,
                     const float* act_lo, const float* act_hi, float* act_env, const int* left, const int* ctr,
                     float* act_out, int precision, void* stream);
int osb_eval_ext_observe(int O, int N, int t, int obs_normalize, int is_reset, const float* next_obs, const float* rew,
                         const float* cost, const unsigned char* terminated, const unsigned char* truncated,
                         const float* final_obs, const unsigned char* final_mask, float* s_raw, float* norm_mean,
                         float* norm_sumsq, float* norm_std, long long* norm_count, unsigned* ticket, float* safety,
                         float safety_budget, float saute_gamma, int early, double cost_limit, double cost_criteria,
                         int* left, int* done_eps, double* ret, double* cost_acc, int* len, int* ctr, double* out_ret,
                         double* out_cost, int* out_len, double* workspace, int* nonfinite, void* stream);
/* The cost rule at N > 1 on a registered env with the optional reset_envs(mask) hook (envs/core.py).  Per step:
 * osb_eval_ext_act(t) -> env.step -> osb_eval_ext_observe_rst(t) -> env.reset_envs(rst) -> osb_ext_reset_rows(t) with
 * mask = rst and the returned rows, with no host synchronisation in between.  osb_eval_ext_observe_rst =
 * osb_eval_ext_observe of a step (is_reset = 0), plus rst[N] (one byte per env, written on every call): 1 where the cost
 * rule ended a running env's episode that the env did not end itself (terminated and truncated both 0) and the env has
 * episodes left, else 0.  osb_ext_reset_rows then writes those envs' reset rows into the state buffer step t + 1 reads
 * and pushes them into ObsNormalize as the step's third batch, after its final and next rows (no row set: untouched).
 * t enters osb_eval_ext_act / osb_eval_ext_observe(_rst) / osb_ext_reset_rows only through its parity, so the launches
 * of a block of steps captured into a CUDA graph at an even t replay as any block at an even offset; once ctr[0] == 0
 * every launch leaves the results, the statistics and act_out as they are.
 * osb_eval_ext_prepare performs the one-time host actions of osb_eval_ext_act (kernel attributes, the tensor-core
 * accumulator image) for a network input of On columns (O, + 1 with safety) and N envs; call it before capturing an
 * osb_eval_ext_act launch.  The observe and reset-rows launches need no preparation. */
int osb_eval_ext_observe_rst(int O, int N, int t, int obs_normalize, const float* next_obs, const float* rew,
                             const float* cost, const unsigned char* terminated, const unsigned char* truncated,
                             const float* final_obs, const unsigned char* final_mask, float* s_raw, float* norm_mean,
                             float* norm_sumsq, float* norm_std, long long* norm_count, unsigned* ticket, float* safety,
                             float safety_budget, float saute_gamma, int early, double cost_limit,
                             double cost_criteria, int* left, int* done_eps, double* ret, double* cost_acc, int* len,
                             int* ctr, double* out_ret, double* out_cost, int* out_len, double* workspace,
                             int* nonfinite, unsigned char* rst, void* stream);
int osb_eval_ext_prepare(int On, int A, int N, int precision);
/* Evaluation on a registered env that declares need_time_limit_wrapper / need_auto_reset_wrapper (envs/core.py).  The
 * evaluation applies TimeLimit only (evaluator.py: TimeLimit(time_limit = 1000), never AutoReset), so such an env does
 * not reset itself.  osb_eval_ext_observe_wrapped = osb_eval_ext_observe_rst with the wrapper step: tl_steps[N]
 * (device ints, zero at the first reset) counts the steps of each running env's episode and is cleared at its end; with
 * time_limit > 0 a step is truncated when the count reaches time_limit, whatever the env's truncated says (time_limit =
 * 0: the env's flag).  rst[N] is 1 for every episode end with episodes left: N > 1 resets them through
 * env.reset_envs(rst) -> osb_ext_reset_rows (the reset rows as their own push, as the reference's explicit reset), N == 1
 * through ctr[2] and env.reset() as above.  No final rows are read: each step's rows are the env's own.  Capturable. */
int osb_eval_ext_observe_wrapped(int O, int N, int t, int obs_normalize, const float* next_obs, const float* rew,
                                 const float* cost, const unsigned char* terminated, const unsigned char* truncated,
                                 float* s_raw, float* norm_mean, float* norm_sumsq, float* norm_std,
                                 long long* norm_count, unsigned* ticket, float* safety, float safety_budget,
                                 float saute_gamma, int early, double cost_limit, double cost_criteria, int* left,
                                 int* done_eps, double* ret, double* cost_acc, int* len, int* ctr, double* out_ret,
                                 double* out_cost, int* out_len, double* workspace, int* nonfinite, unsigned char* rst,
                                 int* tl_steps, int time_limit, void* stream);
/* ---- rollout on an external env (a user CMDP stepped in PyTorch) ----------------------------
 * The fused step split at the env boundary.  Per epoch: env.reset() -> osb_ext_reset_ingest; for t in [0, T):
 * osb_ext_act(t) -> env.step(act_env) -> osb_ext_observe(t); then osb_ext_act(T) (epoch-end bootstrap, critics only)
 * and osb_episode_window.  State arrays as for osb_rollout_step: s_raw[2][N][O] and final_raw[2][N][O] by step parity,
 * ep_ret / ep_cost / ep_len [N], the normaliser state (acc_all / acc_fin / fin_count are not used: the observation
 * statistics are combined from fp64 per-tile moments in fixed tile order, so they are exact to fp64 rounding for any
 * observation range and the same on every run).  workspace: osb_ext_workspace_doubles(O, N) doubles, the size every
 * fp64 push of the observe, evaluation-observe and reset-rows calls shares.
 * nonfinite (device int) is set to 1 when an observation (next or final) is not finite; it is never cleared here.
 * osb_ext_act = the network half of osb_rollout_step (same arithmetic in every precision mode, O > 64 under 1 / 2
 * falls back to the fp32 tiles): obs / act / logp / value slabs, bootstrap values of paths truncated at t - 1 (from
 * final_raw with mean1 / std1) and at t == T the epoch-end bootstrap; act_env[N][A] <- ActionScale(act) onto
 * [act_lo, act_hi] (wrapper.py:L510-512, fp32 lo + (hi - lo) * (a + 1) / 2, no clipping); the act slab keeps the
 * unscaled action.  osb_ext_observe: rew / cost / flags / epfin of step t, episode bookkeeping, next obs -> s_raw,
 * rows of final_obs selected by final_mask -> final_raw (both may be NULL: no final observation), ObsNormalize push
 * of the final rows (-> mean1 / std1) then of all rows (wrapper.py:L231-241).  terminated / truncated / final_mask
 * are one byte per env (0 / non-zero). */
int osb_ext_workspace_doubles(int O, int N);
int osb_ext_reset_ingest(int O, int N, int obs_normalize, const float* obs, float* s_raw, float* ep_ret, float* ep_cost,
                         int* ep_len, float* norm_mean, float* norm_sumsq, float* norm_std, float* norm_mean1,
                         float* norm_std1, long long* norm_count, int* had_fin, unsigned* ticket, double* workspace,
                         int* nonfinite, void* stream);
int osb_ext_act(int O, int A, int obs_normalize, int N, int T, int t, unsigned env_id_offset, float* s_raw,
                float* final_raw, float* norm_mean, float* norm_std, float* norm_mean1, float* norm_std1,
                long long* norm_count, float* obs, float* act, float* logp, float* val_r, float* val_c, float* boot_r,
                float* boot_c, unsigned char* flags, const float* theta, const float* eps, unsigned noise_seed,
                unsigned global_step, const float* act_lo, const float* act_hi, float* act_env, int precision,
                void* stream);
int osb_ext_observe(int O, int N, int T, int t, int obs_normalize, const float* next_obs, const float* rew,
                    const float* cost, const unsigned char* terminated, const unsigned char* truncated,
                    const float* final_obs, const unsigned char* final_mask, float* s_raw, float* final_raw,
                    float* ep_ret, float* ep_cost, int* ep_len, float* norm_mean, float* norm_sumsq, float* norm_std,
                    float* norm_mean1, float* norm_std1, long long* norm_count, int* had_fin, unsigned* ticket,
                    float* rew_slab, float* cost_slab, unsigned char* flags, float* epfin, double* workspace,
                    int* nonfinite, void* stream);
/* EarlyTerminated on an external env (early_terminated_adapter.py:L77-87, per env).  osb_ext_observe_early =
 * osb_ext_observe plus the cost-limit rule: cost_acc[N] (device floats, carried across episodes and epochs) += the
 * env's cost; where it exceeds cost_limit the step stores reward 0 (slab and episode return), terminated = 1 and the
 * env's truncated, the accumulator is cleared and trig[N] (one byte per env, written every step) is 1.  An ordinary
 * episode end does not clear the accumulator.  trig_total (device int, or NULL) is zeroed on the stream and receives the
 * number of triggered envs.  The observation rows and their ObsNormalize pushes are those of osb_ext_observe.
 * The caller then resets the triggered envs and hands their observations to osb_ext_reset_rows (same t): rows of
 * obs[N][O] with mask set go to the state buffer step t + 1 reads and are pushed into the observation statistics after
 * the step's pushes (one batch, device-side row count; no masked row leaves the statistics untouched).  mean1 / std1 /
 * had_fin are not changed.  workspace: osb_ext_workspace_doubles(O, N) doubles, as for osb_ext_observe.  Both calls
 * are capturable into a CUDA graph. */
int osb_ext_observe_early(int O, int N, int T, int t, int obs_normalize, const float* next_obs, const float* rew,
                          const float* cost, const unsigned char* terminated, const unsigned char* truncated,
                          const float* final_obs, const unsigned char* final_mask, float* s_raw, float* final_raw,
                          float* ep_ret, float* ep_cost, int* ep_len, float* norm_mean, float* norm_sumsq,
                          float* norm_std, float* norm_mean1, float* norm_std1, long long* norm_count, int* had_fin,
                          unsigned* ticket, float* rew_slab, float* cost_slab, unsigned char* flags, float* epfin,
                          double* workspace, int* nonfinite, float* cost_acc, float cost_limit, unsigned char* trig,
                          int* trig_total, void* stream);
int osb_ext_reset_rows(int O, int N, int t, int obs_normalize, const unsigned char* mask, const float* obs, float* s_raw,
                       float* norm_mean, float* norm_sumsq, float* norm_std, long long* norm_count, unsigned* ticket,
                       double* workspace, int* nonfinite, void* stream);
/* TimeLimit and AutoReset (wrapper.py) for an external env that declares need_time_limit_wrapper /
 * need_auto_reset_wrapper and does not reset itself.  Per step: osb_ext_act(t) -> env.step -> osb_ext_wrapper_step ->
 * reset of the envs in done -> osb_ext_observe_wrapped(t).  osb_ext_wrapper_step, one byte per env: steps[N] (device
 * ints, TimeLimit's _time; zero them at every epoch-start reset) += 1; trunc_out = steps >= time_limit when time_limit
 * > 0 (the env's own truncated is discarded), else the env's truncated; done = terminated | trunc_out; steps = 0 where
 * done.  done_total (device int, or NULL) is zeroed on the stream and receives the number of done envs.
 * osb_ext_observe_wrapped = osb_ext_observe of a step whose final observation is the step's own row: truncated is
 * trunc_out, the rows of step_obs where done is set are the final rows (final_raw, the first ObsNormalize push), and the
 * next row of such an env is its row of reset_obs[N][O] (read only where done is set; NULL when no env is done).  The
 * second push is every env's next row, so the reset rows join the step's batch, as AutoReset inside ObsNormalize does.
 * Both calls are capturable into a CUDA graph. */
int osb_ext_wrapper_step(int N, int time_limit, const unsigned char* terminated, const unsigned char* truncated,
                         int* steps, unsigned char* trunc_out, unsigned char* done, int* done_total, void* stream);
int osb_ext_observe_wrapped(int O, int N, int T, int t, int obs_normalize, const float* step_obs, const float* rew,
                            const float* cost, const unsigned char* terminated, const unsigned char* truncated,
                            const float* reset_obs, const unsigned char* done, float* s_raw, float* final_raw,
                            float* ep_ret, float* ep_cost, int* ep_len, float* norm_mean, float* norm_sumsq,
                            float* norm_std, float* norm_mean1, float* norm_std1, long long* norm_count, int* had_fin,
                            unsigned* ticket, float* rew_slab, float* cost_slab, unsigned char* flags, float* epfin,
                            double* workspace, int* nonfinite, void* stream);
/* CUDA-graph capture of the external-env epoch (for envs whose step is itself capturable).
 * osb_ext_prepare performs every one-time host action of osb_ext_act / osb_ext_act_graph for these dimensions
 * (kernel attributes, the tensor-core accumulator image at its final size); call it before capturing.  An act launch on
 * a capturing stream that would still need one of them fails with OSB_ERR_UNSUPPORTED instead of breaking the capture.
 * osb_ext_act_graph = osb_ext_act with the Philox counter read on the device: *epoch_dev * T + t (unsigned wrap-around,
 * the same value osb_ext_act gets from global_step = epoch * T + t), so a replayed act draws the noise of the epoch the
 * counter holds.  osb_ext_epoch_advance adds 1 to *epoch_dev on the stream (one thread; captured last in an epoch).
 * osb_ext_reset_ingest and osb_ext_observe need no preparation. */
int osb_ext_prepare(int O, int A, int N, int precision);
int osb_ext_act_graph(int O, int A, int obs_normalize, int N, int T, int t, unsigned env_id_offset, float* s_raw,
                      float* final_raw, float* norm_mean, float* norm_std, float* norm_mean1, float* norm_std1,
                      long long* norm_count, float* obs, float* act, float* logp, float* val_r, float* val_c,
                      float* boot_r, float* boot_c, unsigned char* flags, const float* theta, const float* eps,
                      unsigned noise_seed, const unsigned* epoch_dev, const float* act_lo, const float* act_hi,
                      float* act_env, int precision, void* stream);
int osb_ext_epoch_advance(unsigned* epoch_dev, void* stream);
/* RewardNormalize / CostNormalize (envs/wrapper.py:L280-423; Normalizer(shape=(), clip=5),
 * common/normalizer.py:L88-139) applied to one epoch's slab x[T][N] in place, after the rollout: row t
 * is pushed into the running statistics (batch of N) and normalised with the statistics valid right
 * after that push, exactly the reference's per-step sequence.  state: {mean, sumsq, std} (3 floats) and
 * count[1] persist across epochs; workspace: 4 * T floats. */
int osb_scalar_normalize_rows(float* x, int T, int N, float clip, float* state, long long* count,
                              float* workspace, void* stream);

/* ---- policy step on a trained model (no env, no slabs) ------------------------------------------
 * replaces ConstraintActorCritic.step          models/actor_critic/constraint_actor_critic.py:L84-109
 *          GaussianLearningActor.predict / forward / log_prob   models/actor/gaussian_learning_actor.py:L64-139
 *          VCritic.forward                       models/critic/v_critic.py:L75-92
 * B >= 1 rows of already normalised observations obs[B][O] (what the model sees behind ObsNormalize); theta as above
 * with 1 <= A <= 16 and hidden sizes [64, 64].  net_mask bit0 actor, bit1 reward critic, bit2 cost critic (at least
 * one).  Actor: mean[B][A]; act[B][A] = mean + exp(log_std) * eps with eps[B][A] caller-supplied standard-normal draws
 * (Normal.rsample), or act = mean when eps is NULL (deterministic); logp[B] = sum_a Normal(mean, std).log_prob of act,
 * or of act_in[B][A] when act_in is given (act must then be NULL; eps and act_in are exclusive).  mean, act and logp
 * may each be NULL (not written).  Critics: value_r[B] / value_c[B], required when their bit is set.  The arithmetic of
 * osb_rollout_step in each precision: 0 = fp32 FMA tiles (any O), 1 = tf32 wgmma tiles (O <= 512), 2 = bf16x3 wgmma
 * tiles (O <= 64); a tensor-core mode outside its bound runs on the fp32 tiles.  Writes nothing else: no RNG, normaliser
 * or slab state.  Launches of this entry share one accumulator image per device: order them on one stream.
 * osb_policy_prepare performs the one-time host actions (kernel attributes, the accumulator image sized for any B);
 * the first osb_policy_step does them too, and a call on a capturing stream that would still need them fails with
 * OSB_ERR_UNSUPPORTED instead of breaking the capture. */
int osb_policy_prepare(void);
int osb_policy_step(const float* theta, int O, int A, long long B, const float* obs, const float* eps,
                    const float* act_in, int net_mask, int precision, float* mean, float* act, float* logp,
                    float* value_r, float* value_c, void* stream);

/* ---- learner: fused minibatch forward + loss + backward ------------------------------------
 * replaces PolicyGradient._update minibatch body  algorithms/on_policy/base/policy_gradient.py:L369-381
 *          _update_reward_critic/_update_cost_critic/_update_actor                       :L407-524
 *          PPO._loss_pi  base/ppo.py:L35-87;  PPOLag._compute_adv_surrogate  naive_lagrange/ppo_lag.py:L82-102
 *          PolicyGradient._loss_pi  base/policy_gradient.py:L551-588;  CPO._loss_pi_cost  second_order/cpo.py:L182-212
 *          FOCOPS._loss_pi  first_order/focops.py:L62-108
 * Batch tensors are the slabs ([rows] / [rows][O] / [rows][A], row = t*N + i); advantages are the
 * RAW GAE outputs and are standardised on the fly with moments[4] (osb_adv_moments).  A minibatch is
 * the window [mb_start, mb_start+mb_count) of a permutation of [0,total): perm (slab rows, parity
 * mode) or NULL (in-kernel keyed Feistel bijection).  loss_kind: 0 PPO-clip, 1 plain ratio*adv,
 * 2 FOCOPS, 3 cost surrogate, 5 P3O (PPO-clip + kappa * relu(mean(ratio*adv_c) + Jc - limit),
 * penalty_function/p3o.py:L48-125; kappa is passed as focops_lam, Jc - limit as focops_eta; like
 * FOCOPS it runs a forward-only pass first for the minibatch mean).  lagrange: device scalar lambda or NULL (0).  net_mask bit0 actor,
 * bit1 reward critic, bit2 cost critic.  gpart: osb_update_grid_blocks(mb_count) * P floats;
 * stats_part: that many * 3 * 8 floats.  stop_flag (device int, may be NULL): non-zero = no-op. */
int osb_update_grid_blocks(int mb_count);
int osb_minibatch_grad(const float* theta, int O, int A, const float* obs, const float* act,
                       const float* logp, const float* adv_r, const float* adv_c,
                       const float* tv_r, const float* tv_c, const float* mu_old,
                       const float* moments, const int* perm, long long total, unsigned perm_seed,
                       long long mb_start, int mb_count, int loss_kind, float clip,
                       float entropy_coef, float focops_lam, float focops_eta,
                       const float* lagrange, const float* logstd_old, int net_mask, float* gpart,
                       float* stats_part, const int* stop_flag, void* stream);
/* Tensor-core variant of osb_minibatch_grad: the tile GEMMs run as tf32 wgmma with accumulator image
 * accumulators (operands fp32 in 128B-swizzled smem tiles; transposed activations produced by
 * role-swapped MMAs).  Same arguments and outputs; O <= 512, A <= 16.  This is arithmetic mode
 * `precision = 1` of osb_ppo_update_epoch; mode 0 is the exact-fp32 FMA parity path.
 * gpart / stats_part rows: osb_tc_grid_blocks(mb_count, net_mask) -- a third of the device's SMs per network
 * when several networks share the launch, up to all of them (at most 148) when net_mask names a single network. */
int osb_tc_grid_blocks(long long rows, int net_mask);
int osb_minibatch_grad_tc(const float* theta, int O, int A, const float* obs, const float* act,
                          const float* logp, const float* adv_r, const float* adv_c,
                          const float* tv_r, const float* tv_c, const float* mu_old,
                          const float* moments, const int* perm, long long total, unsigned perm_seed,
                          long long mb_start, int mb_count, int loss_kind, float clip,
                          float entropy_coef, float focops_lam, float focops_eta,
                          const float* lagrange, const float* logstd_old, int net_mask, float* gpart,
                          float* stats_part, const int* stop_flag, void* stream);
/* Split-bf16 ("bf16x3") parity-grade tensor-core variant (csrc/update_x3.cu): every GEMM = six bf16 wgmma
 * MMAs over the three bf16 pieces of its fp32 operands, fp32 accumulate; O <= 64, A <= 16, every loss kind. */
int osb_minibatch_grad_x3(const float* theta, int O, int A, const float* obs, const float* act,
                          const float* logp, const float* adv_r, const float* adv_c,
                          const float* tv_r, const float* tv_c, const float* mu_old,
                          const float* moments, const int* perm, long long total, unsigned perm_seed,
                          long long mb_start, int mb_count, int loss_kind, float clip,
                          float entropy_coef, float focops_lam, float focops_eta,
                          const float* lagrange, const float* logstd_old, int net_mask, float* gpart,
                          float* stats_part, const int* stop_flag, void* stream);
/* Full-batch actor pass (KL early stop policy_gradient.py:L383-397; TRPO/CPO line-search
 * evaluations trpo.py:L102-138, cpo.py:L114-171).  mu_store != NULL: write mu(theta) per row.
 * Otherwise out[8] <- {sum_s sum_a KL(old||new), sum ratio*adv, sum ratio*adv_c, sum ratio, count,
 * sum ratio*adv_r, 0, 0} in fp64; rows 0, stride, 2*stride, ...; workspace: 296*8 doubles. */
int osb_actor_eval(const float* theta_actor, int O, int A, const float* obs, const float* act,
                   const float* logp, const float* adv_r, const float* adv_c, const float* mu_old,
                   const float* logstd_old, const float* moments, const float* lagrange,
                   long long total, int stride, float* mu_store, double* workspace, double* out,
                   void* stream);
/* Tensor-core (TF32 wgmma) variant of osb_actor_eval: same arguments / outputs, O <= 512. */
int osb_actor_eval_tc(const float* theta_actor, int O, int A, const float* obs, const float* act,
                      const float* logp, const float* adv_r, const float* adv_c, const float* mu_old,
                      const float* logstd_old, const float* moments, const float* lagrange,
                      long long total, int stride, float* mu_store, double* workspace, double* out,
                      void* stream);
/* One update iteration of PolicyGradient._update (policy_gradient.py:L369-381) as ONE persistent cooperative
 * kernel on bf16x3 tiles (csrc/update_x3.cu): every minibatch = fused forward + loss + backward, fixed-order
 * partial reduction, per-network clip_grad_norm_, clipped-gradient exchange over NVLink peer memory when
 * world > 1 (clip -> average -> step: policy_gradient.py:L437-443, distributed.py:L193-198) and torch-Adam,
 * parameters re-staged in shared memory between minibatches.  perm = slab rows of this iteration or NULL. */
int osb_ppo_update_iter_x3(float* theta, float* grad, float* adam_m, float* adam_v, int* adam_step, int O, int A,
                           const float* obs, const float* act, const float* logp, const float* adv_r,
                           const float* adv_c, const float* tv_r, const float* tv_c, const float* moments,
                           const int* perm, long long total, unsigned perm_seed, int batch_size, int loss_kind,
                           float clip, float entropy_coef, const float* lagrange, int net_mask,
                           float critic_norm_coef, float max_grad_norm, float lr_actor, float lr_critic_r,
                           float lr_critic_c, float* gpart, float* stats_part, float* train_stats,
                           const int* stop_flag, void* peer_buf, void* peer_flag, int world, int rank,
                           int* p2p_error, void* stream);
/* Split-bf16 (parity-grade tensor-core) variant, O <= 64 (csrc/eval_tc.cu). */
int osb_actor_eval_x3(const float* theta_actor, int O, int A, const float* obs, const float* act,
                      const float* logp, const float* adv_r, const float* adv_c, const float* mu_old,
                      const float* logstd_old, const float* moments, const float* lagrange,
                      long long total, int stride, float* mu_store, double* workspace, double* out,
                      void* stream);
/* Fisher-vector product partials (NaturalPG._fvp, base/natural_pg.py:L74-119, analytic
 * Gauss-Newton form; damping is added by osb_reduce_partials).  gpart: blocks * P_actor floats. */
int osb_fvp_grid_blocks(long long total, int stride);
int osb_fvp_partials(const float* theta_actor, const float* vec, int O, int A, const float* obs,
                     long long total, int stride, float* gpart, void* stream);
/* Tensor-core Fisher-vector product (O <= 512): forward-mode tangent pass on tf32 tiles (csrc/fvp_tc.cu; dmu
 * scratch [total][A]) + the actor backward of the tensor-core gradient kernel.
 * gpart: osb_tc_grid_blocks(rows, 1) rows of P_actor floats, rows = ceil(total / stride);
 * stats_scratch: that many * 24 floats.  Reduce with osb_reduce_partials. */
int osb_fvp_partials_tc(const float* theta_actor, const float* vec, int O, int A, const float* obs,
                        long long total, int stride, float* dmu, float* gpart, float* stats_scratch,
                        void* stream);
/* Split-bf16 ("bf16x3") variant of osb_fvp_partials_tc (O <= 64): forward-mode tangent kernel on bf16x3 tiles
 * (csrc/fvp_tc.cu) + the bf16x3 actor backward with the tangent as output gradient: fp32-level F v on the tensor
 * cores.  NaturalPG._fvp, natural_pg.py:L74-119. */
int osb_fvp_partials_x3(const float* theta_actor, const float* vec, int O, int A, const float* obs,
                        long long total, int stride, float* dmu, float* gpart, float* stats_scratch,
                        void* stream);
/* Actor backward with a supplied output gradient (loss kind LOSS_DMU = 6): the backward of actor losses written in
 * PyTorch.  obs [rows][O] (contiguous, normalised), dmu [rows][A] = dL/dmu; gpart <- per-CTA partials of
 * J_mu^T dmu over the actor parameters (log_std entries zero: no sigma^-2 factor, no 1/rows scale, no log_std term),
 * osb_actor_dmu_grid_blocks(rows, O, precision) rows of P_actor floats; stats_scratch: that many * 24 floats.  Reduce
 * with osb_reduce_partials.  precision as osb_ppo_update_epoch: 2 = bf16x3 tiles (O <= 64), 1 = tf32 tiles
 * (O <= 512), otherwise the fp32 tiles -- the tiles osb_actor_eval{_x3,_tc,} of the same precision run forward. */
int osb_actor_dmu_grid_blocks(int rows, int O, int precision);
int osb_actor_dmu_backward(const float* theta_actor, int O, int A, const float* obs, const float* dmu, int rows,
                           int precision, float* gpart, float* stats_scratch, void* stream);
/* Critic backward with a supplied output gradient (LOSS_DMU on a critic): the backward of critic losses written in
 * PyTorch.  theta: the flat [actor | reward critic | cost critic] parameters (P floats); net 1 = reward critic, 2 = cost
 * critic; obs [rows][O] (contiguous, normalised), dv [rows] = dL/dV.  gpart <- per-CTA partials of J_V^T dv,
 * osb_critic_dv_grid_blocks(rows, O, precision) rows of P floats of which the critic's segment (at its offset in theta)
 * is written, as osb_minibatch_grad{,_tc,_x3} write it; stats_scratch: that many * 24 floats.  value [rows] (may be
 * NULL) <- the forward V of the launch.  Reduce with osb_reduce_partials.  The kernels, tiles and CTAs are those of a
 * stepwise update launch of that critic alone over `rows` samples (precision chosen as for osb_actor_dmu_backward), so
 * `value` has the bits of the update kernels' critic forward: with dv = 0 the entry is that forward. */
int osb_critic_dv_grid_blocks(int rows, int O, int precision);
int osb_critic_dv_backward(const float* theta, int O, int A, int net, const float* obs, const float* dv, float* value,
                           int rows, int precision, float* gpart, float* stats_scratch, void* stream);

/* ---- optimiser side --------------------------------------------------------------------------
 * osb_grad_reduce: grad <- sum of CTA partials (+ 2*critic_norm_coef*theta for critics,
 * policy_gradient.py:L431-433); advances adam_step[net]; accumulates train_stats[3][8]
 * ({sum of minibatch mean loss, mean ratio, mean kl, #minibatches, actor: mean entropy bonus -entropy_coef * mean
 * entropy (stats_part slot 5)}).  sumsq_part: 6*osb_optim_blocks.
 * osb_clip_adam: clip_grad_norm_ per network (do_clip) and torch.optim.Adam step (do_adam);
 * multi-rank order = clip -> all-reduce SUM -> grad_scale = 1/world -> Adam (policy_gradient.py:L437-443). */
int osb_optim_blocks(int O, int A);
int osb_grad_reduce(const float* gpart, const float* stats_part, int nblocks, int O, int A,
                    const float* theta, float* grad, float critic_norm_coef, int net_mask,
                    float* sumsq_part, int* adam_step, float* train_stats, const int* stop_flag,
                    void* stream);
int osb_clip_adam(float* grad, float* theta, float* adam_m, float* adam_v, const int* adam_step,
                  const float* sumsq_part, int O, int A, float max_grad_norm, float lr_actor,
                  float lr_critic_r, float lr_critic_c, float grad_scale, float critic_norm_coef,
                  float* train_stats, int do_clip, int do_adam, int net_mask, const int* stop_flag,
                  void* stream);
/* Single-rank fusion of osb_grad_reduce + osb_clip_adam (clip and step) in one cooperative launch. */
int osb_optim_fused(const float* gpart, const float* stats_part, int nblocks, int O, int A,
                    float* theta, float* grad, float* adam_m, float* adam_v, int* adam_step,
                    float critic_norm_coef, float max_grad_norm, float lr_actor, float lr_critic_r,
                    float lr_critic_c, int net_mask, float* sumsq_part, float* train_stats,
                    const int* stop_flag, void* stream);
/* Multi-rank fusion: reduce + clip + one-shot all-reduce over NVLink peer memory + Adam in one
 * cooperative kernel (reference order clip -> average -> step, policy_gradient.py:L437-443,
 * utils/distributed.py:L193-198).  Exchange buffers: every rank osb_p2p_alloc()s [2][P] floats and
 * [2][world] uint32 flags, the 64-byte cudaIpc handles are exchanged by the host, peers
 * osb_p2p_open() them; peer_buf / peer_flag are DEVICE arrays of `world` pointers.  step_id must
 * increase by one per call identically on every rank.  error_flag <- 1 on a peer timeout. */
int osb_p2p_alloc(long long bytes, void** ptr, unsigned char* handle64);
int osb_p2p_open(const unsigned char* handle64, void** ptr);
int osb_optim_fused_p2p(const float* gpart, const float* stats_part, int nblocks, int O, int A,
                        float* theta, float* grad, float* adam_m, float* adam_v, int* adam_step,
                        float critic_norm_coef, float max_grad_norm, float lr_actor,
                        float lr_critic_r, float lr_critic_c, int net_mask, float* sumsq_part,
                        float* train_stats, const int* stop_flag, void* peer_buf, void* peer_flag,
                        int world, int rank, unsigned step_id, int* error_flag, void* stream);
/* Lagrange.update_lagrange_multiplier (common/lagrange.py:L114-136) on the device: Adam step on
 * lambda with grad -(Jc - cost_limit), Jc = window_sums[1]/window_sums[3], clamp to
 * [0, upper_bound] (upper_bound < 0 = none).  state[4] = {lambda, m, v, t}.  nan_flag <- 1 when no
 * episode has finished yet (the reference asserts, naive_lagrange/ppo_lag.py:L74). */
int osb_lagrange_update(const double* window_sums, float cost_limit, float lambda_lr,
                        float upper_bound, float* state, int* nan_flag, void* stream);
/* Lagrange.update_lagrange_multiplier with lambda_optimizer = any other optimiser torch steps on a 0-d
 * fp32 parameter given only lr (common/lagrange.py:L86-97): torch.optim.<kind> with its defaults, as
 * its single-tensor CPU path computes it, then the clamp to [0, upper_bound] (upper_bound < 0 = none).
 * Jc = window_sums[1] / window_sums[3]; an empty window or a NaN Jc sets *nan_flag and leaves state alone.
 * state[OSB_LAMBDA_STATE] (fp32), initialised by the host; s[0] = lambda, s[4] = torch's step count
 * (counted for every kind), unused slots 0:
 *   SGD        -                                 Adagrad    s[1] sum (0)
 *   AdamW      s[1] exp_avg (0), s[2] exp_avg_sq (0)    Adadelta   s[1] square_avg (0), s[2] acc_delta (0)
 *   Adamax     s[1] exp_avg (0), s[2] exp_inf (0)       RMSprop    s[1] square_avg (0)
 *   NAdam      s[1] exp_avg, s[2] exp_avg_sq, s[3] mu_product (1)
 *   RAdam      s[1] exp_avg (0), s[2] exp_avg_sq (0)    Rprop      s[1] prev (0), s[2] step_size (lr)
 *   ASGD       s[1] eta (lr), s[2] mu (1), s[3] ax (0)  Adafactor  s[1] variance (0) */
#define OSB_LAMBDA_STATE 8
#define OSB_LAMBDA_SGD 0
#define OSB_LAMBDA_ADAMW 1
#define OSB_LAMBDA_ADAMAX 2
#define OSB_LAMBDA_NADAM 3
#define OSB_LAMBDA_RADAM 4
#define OSB_LAMBDA_RMSPROP 5
#define OSB_LAMBDA_RPROP 6
#define OSB_LAMBDA_ADAGRAD 7
#define OSB_LAMBDA_ADADELTA 8
#define OSB_LAMBDA_ASGD 9
#define OSB_LAMBDA_ADAFACTOR 10
int osb_lagrange_update_opt(int kind, const double* window_sums, double cost_limit, double lambda_lr,
                            double upper_bound, float* state, int* nan_flag, void* stream);
/* PID-Lagrangian controller step (PIDLagrangian.pid_update, common/pid_lagrange.py:L95-125) in the
 * reference's Python-float (fp64) arithmetic.  pid_state: 64 doubles {integral, EMA(delta), EMA(Jc),
 * penalty, deque length, deque head, -, -, ring[pid_d_delay]}, initialised by the host to
 * {lagrangian_multiplier_init, 0, 0, 0, 1, 0, ..., ring[0] = 0}.  lagrange_state[0] <- (float) penalty.
 * Jc = window_sums[1] / window_sums[3]; an empty window sets *nan_flag. */
int osb_pid_lagrange_update(const double* window_sums, double pid_kp, double pid_ki, double pid_kd,
                            int pid_d_delay, double pid_delta_p_ema_alpha, double pid_delta_d_ema_alpha,
                            int sum_norm, int diff_norm, double penalty_max, double cost_limit,
                            double* pid_state, float* lagrange_state, int* nan_flag, void* stream);
/* kl = eval_out[0]/eval_out[4]; kl_state[4] = {last kl, passes done, stopped, 0}. */
int osb_kl_check(const double* eval_out, float target_kl, int early_stop, int* stop_flag,
                 float* kl_state, void* stream);
/* out[q] = scale * sum_b gpart[b*stride + q] + add_scale * add[q], q < n  (add may be NULL). */
int osb_reduce_partials(const float* gpart, int nblocks, int stride, int n, float scale,
                        const float* add, float add_scale, float* out, void* stream);
/* conjugate_gradients (utils/math.py:L86-132) as device-resident state: x, r, p [n],
 * cg_scalars[4] = {rdotr, converged, iterations, 0}; the caller computes z = F p between steps. */
int osb_cg_init(const float* b, int n, float* x, float* r, float* p, float* cg_scalars, void* stream);
int osb_cg_step(const float* z, int n, float* x, float* r, float* p, float* cg_scalars,
                float residual_tol, float eps, void* stream);
int osb_dot(const float* a, const float* b, int n, float* out, void* stream);

/* ---- epoch driver + NCCL -------------------------------------------------------------------
 * One epoch of PolicyGradient._update (policy_gradient.py:L345-405) issued from C: old-policy
 * snapshot, update_iters passes of minibatch steps (grad -> reduce -> clip -> [all-reduce] ->
 * Adam), full-batch KL after each pass, device-side early stop.  comm = handle from osb_nccl_init
 * (or NULL for a single rank).  With peer_buf / peer_flag (device arrays of `world_size` cudaIpc-mapped
 * pointers, see osb_p2p_alloc) the per-step gradient exchange is the fused one-shot NVLink kernel
 * osb_optim_fused_p2p instead of NCCL; NCCL then only carries the per-pass KL scalar. */
int osb_ppo_update_epoch(float* theta, float* grad, float* adam_m, float* adam_v, int* adam_step,
                         int O, int A, const float* obs, const float* act, const float* logp,
                         const float* adv_r, const float* adv_c, const float* tv_r,
                         const float* tv_c, float* mu_old, float* logstd_old, const float* moments,
                         const int* perm, long long total, unsigned perm_seed, int batch_size,
                         int update_iters, int loss_kind, float clip, float entropy_coef,
                         float focops_lam, float focops_eta, const float* lagrange, int net_mask,
                         float critic_norm_coef, float max_grad_norm, float lr_actor,
                         float lr_critic, float target_kl, int kl_early_stop, float* gpart,
                         float* stats_part, float* sumsq_part, float* train_stats, double* eval_ws,
                         double* eval_out, int* stop_flag, float* kl_state, int precision,
                         void* comm, int world_size, void* peer_buf, void* peer_flag, int rank,
                         int* p2p_error, void* stream);
/* NCCL via dlopen(libpath) of the libnccl.so.2 torch already loaded (distributed.py:L142-228). */
int osb_nccl_unique_id(const char* libpath, unsigned char* id128);
int osb_nccl_init(const char* libpath, const unsigned char* id128, int nranks, int rank,
                  void** comm_out);
int osb_nccl_allreduce(void* comm, void* buf, long long count, int is_f64, void* stream);
int osb_nccl_destroy(void* comm);

/* ---- diagnostics ---------------------------------------------------------------------------
 * One tf32 wgmma GEMM D = A * B^T (both operands K-major; a_mn / b_mn must be 0) on a single warpgroup;
 * out[128][N] is the dump of the accumulator lanes.  Pins the descriptor / swizzle / lane conventions the
 * tensor-core MLP tiles rely on (tests/test_umma_gpu.py). */
int osb_umma_selftest(const float* A, const float* B, int M, int N, int K, int a_mn, int b_mn,
                      float* out, void* stream);

/* Split-bf16 ("bf16x3") building blocks of the parity-grade tensor-core mode (csrc/x3.cuh):
 * one single-warpgroup GEMM D = A * B^T with A [M][K], B [N][K] (row-major fp32 in global memory), each operand
 * staged as three bf16 tiles (SW128 or SW32) consumed K-major or MN-major; out[128][N] = dump of the
 * accumulator lanes (tests/test_x3_gpu.py).  (M, N, K, a_mn, b_mn, b_ones) must be one of the GEMM shapes the
 * kernels issue (csrc/x3_selftest.cu); any other shape is refused. */
int osb_x3_selftest(const float* A, const float* B, int M, int N, int K, int a_mn, int b_mn, int a_sw,
                    int b_sw, int b_ones, float* out, void* stream);
/* The row-half products of the bf16x3 update kernel (gemm_x3_rows, csrc/x3.cuh): D = A * B^T with A [128][K] consumed
 * K-major and B [N][K], issued as one m64 block per row half over the whole K (K = 64: two wgmma chains whose fp32 sum
 * is stored) into out[128][N], and as the M = 128 product in column-half phases (the second adding to the image) into
 * out_phases[128][N]; the two must agree bit for bit (tests/test_update_rowhalf_gpu.py).  (N, K, b_mn) must be one of
 * the shapes the update kernel issues. */
int osb_x3_rows_selftest(const float* A, const float* B, int N, int K, int b_mn, int a_sw, int b_sw, float* out,
                         float* out_phases, void* stream);
int osb_x3_debug_buffer(long long* buf);
/* development aid: clock64 stamps of CTA 0 of the streaming GAE kernel (tools/gae_stage_times.py); NULL turns it off */
int osb_gae_debug_buffer(long long* buf);
/* same for the persistent rollout kernel (tools/rollout_stage_times.py) */
int osb_rollout_debug_buffer(long long* buf);

#ifdef __cplusplus
}
#endif
#endif /* OMNISAFE_B200_H */
