/*
 * b200rl.h -- C ABI of libb200rl.so: the H100-native (sm_90a) implementation of rllab's
 * data-parallel hot path (lock-step lane rollout, process_samples, VPG / TRPO update).
 *
 * The reference (rll/rllab @ ba78e4c) has NO native boundary on this path: the path is pure Python over
 * Theano-compiled functions, pybox2d (SWIG) and libmujoco131 (ctypes, rllab/mujoco_py/mjlib.py:17-60).
 * Each entry point below therefore cites the reference *Python* interface it replaces; the ctypes stub a
 * maintainer adds on the reference side is shown in INTEGRATION.md.
 *
 * Conventions
 *   - every function returns 0 on success, a negative B200RL_E* code otherwise; b200rl_last_error() returns
 *     a thread-local human-readable message for the last failure.
 *   - all pointers are DEVICE pointers unless the name ends in _host; the caller owns every buffer, the
 *     library borrows them until the work queued on `stream` completes; no allocation inside hot calls.
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream); calls are asynchronous.
 *   - lane layout (structure of arrays, time-major): obs [O][T][N], act/mean [A][T][N], rew/adv/ret/base
 *     [T][N] float32, flags [T][N] uint8 (bit0 = env done, bit1 = last sample of its path), tstep [T][N]
 *     uint16 (index of the sample inside its path).  N = lanes on this GPU, T = steps per lane.
 *   - flat policy parameter layout (rllab core/lasagne_powered.py:16-20): [W0 (O,h1) row-major, b0, W1 (h1,h2),
 *     b1, Wout (h2,A), bout, log_std (A)];  P = O*h1+h1 + h1*h2+h2 + h2*A+A + A.  Master copy float64,
 *     kernels read a float32 shadow.
 *   - reductions are two-stage and order-deterministic: per-block float64 partials in `ws`, then a fixed-order
 *     finalize; results are SUMS over this GPU's samples already multiplied by the `scale` argument
 *     (pass 1/B_global so that an NCCL all-reduce(sum) over ranks yields the global mean).
 */
#ifndef B200RL_H_
#define B200RL_H_

#ifdef __cplusplus
extern "C" {
#endif

#define B200RL_VERSION 100

#define B200RL_OK 0
#define B200RL_EINVAL (-1)       /* bad argument / unsupported shape */
#define B200RL_ECUDA (-2)        /* CUDA runtime error (message has the cudaError string) */
#define B200RL_EUNSUPPORTED (-3) /* env kind / network size not compiled in */

/* env kinds (reference classes): examples/point_env.py, rllab/envs/box2d/cartpole_env.py,
 * GymEnv("Pendulum-v0") (rllab/envs/gym_env.py), rllab/envs/mujoco/swimmer_env.py, hopper_env.py;
 * every kind includes the NormalizedEnv action map of rllab/envs/normalized_env.py:78-92. */
#define B200RL_ENV_POINT 0
#define B200RL_ENV_CARTPOLE 1
#define B200RL_ENV_PENDULUM 2
#define B200RL_ENV_SWIMMER 3
#define B200RL_ENV_HOPPER 4
#define B200RL_ENV_CARTPOLE_SWINGUP 5 /* rllab/envs/box2d/cartpole_swingup_env.py (same Box2D model as CartpoleEnv) */
#define B200RL_ENV_DOUBLE_PENDULUM 6 /* rllab/envs/box2d/double_pendulum_env.py (models/double_pendulum.xml.mako) */
#define B200RL_ENV_HALF_CHEETAH 7 /* rllab/envs/mujoco/half_cheetah_env.py (vendor/mujoco_models/half_cheetah.xml) */
/* GymEnv("CartPole-v0") over gym 0.7.4: Discrete(2) actions.  The action float of env_step is the action index; the
 * Gaussian b200rl_rollout rejects it, b200rl_rollout_categorical drives it. */
#define B200RL_ENV_GYM_CARTPOLE 8

#define B200RL_NOISE_UNIFORM 0
#define B200RL_NOISE_NORMAL 1

#define B200RL_LOSS_TRPO 0 /* -mean(exp(logp_new-logp_old)*adv)   rllab/algos/npo.py:72-82 */
#define B200RL_LOSS_VPG 1  /* -mean(logp*adv)                     rllab/algos/vpg.py:91     */
#define B200RL_LOSS_KL 2   /* mean KL(old || new): only as the gradient pass of b200rl_update_f64 (FiniteDifferenceHvp) */

#define B200RL_FLAG_DONE 1
#define B200RL_FLAG_END 2
#define B200RL_FLAG_CUT 4    /* set with END on a path cut by the end of the lane buffer (neither done nor max length) */
#define B200RL_FLAG_MASKED 8 /* set by b200rl_process_samples(drop_cut_paths) on every sample of a dropped path */

/* number of float64 slots in the process_samples statistics block (see b200rl_process_samples) */
#define B200RL_PS_NSUM 16
#define B200RL_PS_NMAX 4

const char* b200rl_last_error(void);
int b200rl_version(void);
/* Number of CUDA kernels this library has launched in this process (bench.py reports the per-step delta). */
unsigned long long b200rl_kernel_launches(void);
/* FP32 roofline microbenchmark (no memory traffic): queues one kernel of num_SMs*8 blocks x 256 threads, each thread
 * running iters x 16 independent float2 FMA chains; *fma_out_host = scalar FMAs executed.  The caller times it (CUDA
 * events) -- bench.py reports the policy passes against this measured FP32 peak. */
int b200rl_bench_ffma2(int iters, float* sink, long long* fma_out_host, void* stream);
/* SM count of the current device (grid sizing helper for callers that size workspaces). */
int b200rl_device_sms(int* sms_out);

/* Static description of an env kind.  lb/ub: wrapped action bounds (host arrays of act_dim floats) --
 * Env.action_space / observation_space of rllab/envs/base.py:43-62. */
int b200rl_env_info(int env_kind, int* obs_dim, int* act_dim, int* state_dim, int* reset_dim, int* noise_kind,
                    float* lb_host, float* ub_host);

/* *n_out = number of discrete actions of an env kind (its action space is Discrete(n)), 0 for a Box action space. */
int b200rl_env_num_actions(int env_kind, int* n_out);

/* Number of policy parameters P for (O, h1, h2, A); <0 if the network size is not compiled in. */
long long b200rl_policy_num_params(int obs_dim, int h1, int h2, int act_dim);

/* Counter-based Philox4x32-10 noise, the generator the fused rollout uses internally:
 * out[row][k][n] for row in [row0,row0+rows), k < K, n < N;  value = f(seed, iter, stream_id, lane0+n, row, k).
 * stream_id 0 = action noise eps (normal), 1 = reset noise (kind of the env).  Replaces the np.random draws of
 * gaussian_mlp_policy.py:128,135 and of the envs' reset(). */
int b200rl_fill_noise(float* out, int rows, int row0, int K, int N, long long lane0, int noise_kind,
                      unsigned int seed, unsigned int iter, int stream_id, void* stream);

/* Env.reset for N lanes (rllab/envs/base.py:26-33; vec_env_executor.py:28-31).  reset_raw [K][N] raw noise or NULL
 * (then Philox(seed, iter, stream 1, row)).  Writes state [S][N] and obs [O][N]. */
int b200rl_env_reset(int env_kind, int N, float* state, float* obs_out, const float* reset_raw,
                     unsigned int seed, unsigned int iter, int row, long long lane0, void* stream);

/* Env.step for N lanes (rllab/envs/base.py:6-24).  normalized != 0: actions [A][N] are the policy's raw actions and
 * go through NormalizedEnv.step (normalized_env.py:78-92) first; normalized == 0: actions are handed to the wrapped
 * env unchanged.  Writes obs_out [O][N], rew_out [N], done_out [N]; state is advanced in place (no auto-reset here:
 * the caller decides, as vec_env_executor.py:14-26 does). */
int b200rl_env_step(int env_kind, int N, int normalized, float* state, const float* actions, float* obs_out,
                    float* rew_out, unsigned char* done_out, void* stream);

/* GaussianMLPPolicy.get_actions (rllab/policies/gaussian_mlp_policy.py:132-137): obs [O][n] ->
 * act_out, mean_out [A][n], log_std_out [A] (after the min_std clamp).  eps [A][n] or NULL (Philox). */
int b200rl_policy_get_actions(const float* params_f32, int obs_dim, int h1, int h2, int act_dim, float min_std,
                              const float* obs, long long n, const float* eps, unsigned int seed, unsigned int iter,
                              int row, long long lane0, float* act_out, float* mean_out, float* log_std_out,
                              void* stream);

/* Fused rollout: T lock-step steps of N lanes = BatchSampler.obtain_samples (rllab/algos/batch_polopt.py:22-34)
 * -> rollout (rllab/sampler/utils.py:6-43) with the vectorized auto-reset semantics of
 * sandbox/rocky/tf/envs/vec_env_executor.py:14-26.  eps [T][A][N] / reset_raw [T+1][K][N] inject noise (tests),
 * NULL = in-kernel Philox.  log_std_out [A]. */
int b200rl_rollout(int env_kind, const float* params_f32, int h1, int h2, float min_std, int N, int T,
                   int max_path_length, const float* eps, const float* reset_raw, unsigned int seed,
                   unsigned int iter, long long lane0, float* obs, float* act, float* mean, float* rew,
                   unsigned char* flags, unsigned short* tstep, float* log_std_out, void* stream);

/* BaseSampler.process_samples numeric core (rllab/sampler/base.py:48-93): LinearFeatureBaseline.predict
 * (linear_feature_baseline.py:19-23,40-43) with weights w [2O+4] float64 (NULL = zeros), GAE advantages and
 * discounted returns (special.discount_cumsum), plus the reductions behind the tabular statistics.
 * sums_out [B200RL_PS_NSUM] float64 (all-reduce SUM across ranks):
 *   0 sum adv, 1 sum adv^2, 2 count B, 3 n_paths, 4 sum ret@path start, 5 sum undisc. return, 6 sum undisc^2,
 *   7 sum ret, 8 sum ret^2, 9 sum base, 10 sum base^2, 11 sum (ret-base), 12 sum (ret-base)^2
 * maxs_out [B200RL_PS_NMAX] float64 (all-reduce MAX): 0 max undisc, 1 -min undisc, 2 -min adv, 3 max adv
 * drop_cut_paths != 0 = the reference's whole_paths=True (batch_polopt.py:30-34: samplers only return whole paths): a
 * path cut by the end of the lane buffer (B200RL_FLAG_CUT) is dropped -- its samples get B200RL_FLAG_MASKED in `flags`
 * (in/out), adv = 0, and are left out of every sum above (sums_out[2] is then the number of VALID samples, the divisor
 * every later pass reads through its `count` argument); 0 keeps the cut path as a truncated path (whole_paths=False,
 * truncate_paths, parallel_sampler.py:129-155).
 * ws: float64 workspace of at least b200rl_ws_doubles() entries. */
int b200rl_process_samples(int obs_dim, int N, int T, const float* obs, const float* rew, unsigned char* flags,
                           const unsigned short* tstep, const double* w, double discount, double gae_lambda,
                           int drop_cut_paths, float* adv, float* ret, float* base, double* sums_out, double* maxs_out,
                           double* ws, void* stream);

/* b200rl_process_samples with a baseline the caller has already written into `base` [T][N] float32 (read only): the
 * LinearFeatureBaseline predict is skipped, the GAE scan and the statistics are the same kernels.  Used by baselines
 * predicted by their own kernels (GaussianMLPBaseline.predict, gaussian_mlp_baseline.py:38-40, via b200rl_vf_forward). */
int b200rl_process_samples_base(int obs_dim, int N, int T, const float* obs, const float* rew, unsigned char* flags,
                                const unsigned short* tstep, const float* base, double discount, double gae_lambda,
                                int drop_cut_paths, float* adv, float* ret, double* sums_out, double* maxs_out,
                                double* ws, void* stream);

/* center_advantages / shift_advantages_to_positive (rllab/algos/util.py:7-12) in place over B samples, from the
 * (already all-reduced) sums/maxs of b200rl_process_samples; masked samples (flags, may be NULL) keep adv = 0. */
int b200rl_center_advantages(float* adv, long long B, const unsigned char* flags, const double* sums,
                             const double* maxs, int center, int positive, void* stream);

/* LinearFeatureBaseline.fit normal equations (linear_feature_baseline.py:26-33): with d = 2O+4 and
 * f = [features, ret], writes gram_out [(d+1)*(d+2)/2] float64 = upper triangle (row-major, i<=j) of sum f f^T
 * over this GPU's samples.  The d x d solve (np.linalg.lstsq on d<=44 unknowns) is done by the caller. */
int b200rl_lfb_gram(int obs_dim, long long B, const float* obs, const unsigned short* tstep, const float* ret,
                    const unsigned char* flags, double* gram_out, double* ws, void* stream);

/* The d x d solve of LinearFeatureBaseline.fit on the device (linear_feature_baseline.py:26-37): w_out [d = 2O+4]
 * float64 from gram (b200rl_lfb_gram layout, already all-reduced), regularisation reg_coeff escalated x10 up to 5 times
 * while the Cholesky solve fails; info_out [3] = (final reg, attempts used, ok flag).  Keeps the baseline fit free of
 * host round trips. */
int b200rl_lfb_solve(int obs_dim, const double* gram, double reg_coeff, double* w_out, double* info_out, void* stream);

/* Surrogate loss and KL(old||new) (npo.py:72-82, vpg.py:91-99, diagonal_gaussian.py:14-34,58-69):
 * out[0] = scale * sum(-w*adv) (w = likelihood ratio for TRPO, logp for VPG), out[1] = scale * sum(kl),
 * out[2] = max(kl).  old_log_std [A] (state-independent ParamLayer, lasagne_layers.py:9-30).
 * Common to the update passes: `flags` ([B] or NULL) -- samples carrying B200RL_FLAG_MASKED are skipped; `count` (device
 * pointer or NULL) -- the sums are additionally divided by *count, the all-reduced number of valid samples
 * (sums_out[2] of b200rl_process_samples): pass scale = 1 and count = &sums[2] for the mean over the valid samples of
 * all ranks without reading the count back to the host.
 * Arithmetic of the three update passes (loss_kl, grad, fvp): float32 per sample, float32 sums inside one 128-sample
 * tile, float64 above.  (32,32) nets: every pass runs its dense layers on the wgmma tensor cores with the three-pass
 * TF32 split (float32-grade, 4e-7 of the output scale); (64,64) nets: grad and fvp (with h_cache) likewise, loss_kl on
 * the FP32 pipe in the rollout's summation order (ratio exactly 1 at theta_old).  While b200rl_peer_fuse_updates(1) is in
 * effect the outputs are reduced over all ranks of the bound peer communicator inside the pass. */
int b200rl_loss_kl(int loss_kind, const float* params_f32, int obs_dim, int h1, int h2, int act_dim, float min_std,
                   long long B, const float* obs, const float* act, const float* adv, const float* old_mean,
                   const float* old_log_std, const unsigned char* flags, double scale, const double* count, double* out,
                   double* ws, void* stream);

/* Flat gradient of the surrogate (theano.grad in conjugate_gradient_optimizer.py:184-186 /
 * first_order_optimizer.py:62-64): g_out [P] float64 = scale * sum over samples.  loss_out (3 doubles or NULL)
 * receives the b200rl_loss_kl triple of the same pass (loss, sum kl, max kl) at no extra cost.  h_cache_out
 * ([h1+h2][B] float32 planes, or NULL) receives the hidden activations tanh(.) of both layers: theta is fixed during the
 * CG solve, so the (cg_iters+1) Fisher-vector products that follow can read them back (256 B/sample of HBM traffic,
 * ~1 % of the roofline) instead of recomputing two dense layers and 64 tanh per sample. */
int b200rl_grad(int loss_kind, const float* params_f32, int obs_dim, int h1, int h2, int act_dim, float min_std,
                long long B, const float* obs, const float* act, const float* adv, const float* old_mean,
                const float* old_log_std, const unsigned char* flags, double scale, const double* count, double* g_out,
                double* loss_out, float* h_cache_out, double* ws, void* stream);

/* Gradient of the penalised objective of PPO's L-BFGS step (penalty_lbfgs_optimizer.py:52-63 over the surrogate and
 * mean KL of npo.py:72-82): g_out [P] float64 = scale * sum over valid samples of grad(surrogate_s + penalty * kl_s),
 * kl_s = KL(old || new) of sample s, with the min_std mask of b200rl_grad on the log_std slot.  loss_out (3 doubles or
 * NULL) receives the UNPENALISED triple (loss, sum kl, max kl) of the same pass, bit-identical to b200rl_grad's; the
 * caller forms loss + penalty * mean kl in float64.  loss_kind: B200RL_LOSS_TRPO or B200RL_LOSS_VPG.  penalty >= 0 is applied in
 * float32; penalty 0 runs b200rl_grad's pass (identical outputs).  Arguments otherwise as b200rl_grad (no activation
 * cache).  Tensor-core kernels only: B200RL_EUNSUPPORTED in a B200RL_AB_TILE32 build. */
int b200rl_grad_penalized(int loss_kind, double penalty, const float* params_f32, int obs_dim, int h1, int h2,
                          int act_dim, float min_std, long long B, const float* obs, const float* act, const float* adv,
                          const float* old_mean, const float* old_log_std, const unsigned char* flags, double scale,
                          const double* count, double* g_out, double* loss_out, double* ws, void* stream);

/* Fisher/Hessian-vector product of mean KL at theta_old (PerlmutterHvp, conjugate_gradient_optimizer.py:22-55):
 * Hx_out [P] = scale * sum_samples J^T M J x  (+ reg_coeff*x and the log_std block added once: pass
 * add_diag=1 on exactly one rank, or on all ranks with diag_scale = 1/world_size).  h_cache: activations written by
 * b200rl_grad at the SAME parameters, or NULL to recompute them.  tile_list (device int[n_list], or NULL = the whole
 * batch): indices of the 128-sample tiles to visit -- subsample_factor < 1 of conjugate_gradient_optimizer.py:235-245
 * at tile granularity (the caller draws the subset and passes count = the number of valid samples in it, see
 * b200rl_count_valid). */
int b200rl_fvp(const float* params_f32, int obs_dim, int h1, int h2, int act_dim, float min_std, long long B,
               const float* obs, const unsigned char* flags, const double* x, double scale, const double* count,
               double reg_coeff, double diag_scale, double* Hx_out, const float* h_cache, const int* tile_list,
               int n_list, double* ws, void* stream);
/* count_out[0] = number of unmasked samples inside the listed 128-sample tiles (tile_list NULL = whole batch). */
int b200rl_count_valid(long long B, const unsigned char* flags, const int* tile_list, int n_list, double* count_out,
                       double* ws, void* stream);

/* float64 "parity mode" of the three passes above on the float64 master parameters (mode 0 = loss/KL -> loss_out[3],
 * 1 = gradient -> vec_out[P] (+ loss_out[3] if non-NULL), 2 = Fisher-vector product of x -> vec_out[P]).  The reference's
 * default floatX is float64; with cg_iters = 10 the CG recursion amplifies float32 rounding of the Hessian-vector
 * product past any useful tolerance (DESIGN.md "Parity limit"), so this mode exists to compare the whole TRPO step
 * with the oracle at the reference's default settings.  ~10x slower than the float32 kernels.
 * loss_kind B200RL_LOSS_KL with mode 1 returns the gradient of mean KL(old || new) at params_f64: the two evaluations of
 * FiniteDifferenceHvp (conjugate_gradient_optimizer.py:58-115), whose 1e-8 relative perturbation needs float64. */
int b200rl_update_f64(int mode, int loss_kind, const double* params_f64, int obs_dim, int h1, int h2, int act_dim,
                      double min_std, long long B, const float* obs, const float* act, const float* adv,
                      const float* old_mean, const float* old_log_std, const unsigned char* flags, const double* x,
                      double scale, const double* count, double reg_coeff, double diag_scale, double* vec_out,
                      double* loss_out, double* ws, void* stream);

/* ---- CategoricalMLPPolicy (rllab/policies/categorical_mlp_policy.py, rllab/distributions/categorical.py).  Net: tanh
 * (h1, h2) trunk, softmax output over n actions; flat layout [W0 (O,h1), b0, W1 (h1,h2), b1, Wout (h2,n), bout], no log_std
 * (P = O*h1+h1 + h1*h2+h2 + h2*n+n).  Compiled for O = 4, hidden (32,32), n = 2 (CartPole-v0); any other shape returns
 * B200RL_EUNSUPPORTED.  Lane layout as above with A = n: act [n][T][N] holds the ONE-HOT action (the reference's
 * flattened action), the mean planes hold prob [n][T][N].  The update passes take `act` one-hot and `old_prob` [n][B], and
 * follow the conventions of b200rl_loss_kl / b200rl_grad / b200rl_fvp (flags, scale, count, fixed-order reductions,
 * peer fusion); probabilities are softmax(z) (max-shifted, ascending-k sum) after the rollout's forward in every pass, so
 * the likelihood ratio is exactly 1 and the KL exactly 0 at theta_old. ---- */
long long b200rl_categorical_num_params(int obs_dim, int h1, int h2, int n_actions);

/* CategoricalMLPPolicy.get_actions: obs [O][n] -> act_out [n] int32 action indices = weighted_sample(prob, u)
 * (#{k : cumsum_k(prob) < u}, clipped to n_actions-1; rllab/misc/special.py:10-19), prob_out [n_actions][n].  u [n] or
 * NULL (Philox stream 0 at (lane0 + i, row), the first word of the uniform map, as b200rl_fill_noise with K = 1). */
int b200rl_categorical_get_actions(const float* params_f32, int obs_dim, int h1, int h2, int n_actions,
                                   const float* obs, long long n, const float* u, unsigned int seed, unsigned int iter,
                                   int row, long long lane0, int* act_out, float* prob_out, void* stream);

/* Fused rollout of a discrete-action env kind with a categorical policy: b200rl_rollout's lane semantics (auto-reset,
 * FLAG_DONE / FLAG_END / FLAG_CUT, tstep), with the action drawn as in b200rl_categorical_get_actions from u [T][N]
 * (tests) or NULL = Philox stream 0 row t.  Writes obs, one-hot act [n][T][N], prob [n][T][N], rew, flags, tstep. */
int b200rl_rollout_categorical(int env_kind, const float* params_f32, int h1, int h2, int N, int T,
                               int max_path_length, const float* u, const float* reset_raw, unsigned int seed,
                               unsigned int iter, long long lane0, float* obs, float* act, float* prob, float* rew,
                               unsigned char* flags, unsigned short* tstep, void* stream);

/* (loss, sum KL, max KL) as b200rl_loss_kl: TRPO  -adv (p_new.x + 1e-8) / (p_old.x + 1e-8),  VPG  -adv log(p.x + 1e-8),
 * KL = sum_k p_old (log(p_old + 1e-8) - log(p_new + 1e-8)) (categorical.py). */
int b200rl_categorical_loss_kl(int loss_kind, const float* params_f32, int obs_dim, int h1, int h2, int n_actions,
                               long long B, const float* obs, const float* act, const float* adv,
                               const float* old_prob, const unsigned char* flags, double scale, const double* count,
                               double* out, double* ws, void* stream);

/* Gradient of the surrogate plus penalty * mean KL (penalty 0: b200rl_grad, > 0: b200rl_grad_penalized); loss_out (3 or
 * NULL) = the unpenalised triple of the same pass, h_cache_out ([h1+h2][B] or NULL) the hidden activations. */
int b200rl_categorical_grad(int loss_kind, double penalty, const float* params_f32, int obs_dim, int h1, int h2,
                            int n_actions, long long B, const float* obs, const float* act, const float* adv,
                            const float* old_prob, const unsigned char* flags, double scale, const double* count,
                            double* g_out, double* loss_out, float* h_cache_out, double* ws, void* stream);

/* Fisher-vector product J^T M J x (+ diag_scale * reg_coeff * x) at theta_old, M = Hessian of the per-sample KL in the
 * logits at theta_old with the 1e-8 kept (DESIGN.md section 5); arguments as b200rl_fvp. */
int b200rl_categorical_fvp(const float* params_f32, int obs_dim, int h1, int h2, int n_actions, long long B,
                           const float* obs, const unsigned char* flags, const double* x, double scale,
                           const double* count, double reg_coeff, double diag_scale, double* Hx_out,
                           const float* h_cache, const int* tile_list, int n_list, double* ws, void* stream);

/* float64 parity mode of the three passes above on the float64 master parameters, as b200rl_update_f64 (mode 0 loss/KL
 * -> loss_out[3], 1 gradient -> vec_out[P] (+ loss_out), 2 Fisher-vector product of x -> vec_out[P]); loss_kind
 * B200RL_LOSS_KL with mode 1 is the gradient of mean KL(old || new) (FiniteDifferenceHvp).  Mode 2 is the exact Hessian
 * of mean KL at theta_old, including the O(1e-8) term of the KL's first derivative in the logits that the float32 pass
 * leaves out (DESIGN.md section 5).  Weight gradients are summed with float64 atomics: reruns agree to rounding. */
int b200rl_categorical_update_f64(int mode, int loss_kind, const double* params_f64, int obs_dim, int h1, int h2,
                                  int n_actions, long long B, const float* obs, const float* act, const float* adv,
                                  const float* old_prob, const unsigned char* flags, const double* x, double scale,
                                  const double* count, double reg_coeff, double diag_scale, double* vec_out,
                                  double* loss_out, double* ws, void* stream);

/* out [2] float64 = (sum over valid samples of -sum_k p_k log(p_k + 1e-8), number of valid samples) of prob [n][B]
 * (categorical.py:entropy; the sampler's Entropy is out[0] / out[1] after the all-reduce). */
int b200rl_categorical_entropy(int n_actions, long long B, const float* prob, const unsigned char* flags, double* out,
                               double* ws, void* stream);

/* ---- GaussianGRUPolicy (rllab/policies/gaussian_gru_policy.py, rllab/core/network.py:104-270 GRULayer / GRUNetwork,
 * rllab/distributions/recurrent_diagonal_gaussian.py).  x_t = [obs_t, prev_action_t] (include_action != 0) or obs_t;
 * r = sigma(x W_xr + h W_hr + b_r), u = sigma(x W_xu + h W_hu + b_u), c = tanh(x W_xc + r * (h W_hc) + b_c),
 * h' = (1 - u) h + u c, mean = h' W_out + b_out, log_std a state-independent parameter (no min_std clamp).  h = 0 and
 * prev_action = 0 at a path start (tstep == 0); inside a path prev_action is the previous raw action act[t-1].  Flat
 * layout [W_xr (I x H), W_hr (H x H), b_r, W_xu, W_hu, b_u, W_xc, W_hc, b_c, W_out (H x A), b_out, log_std].  Compiled
 * for obs_dim 4, hidden 32, act_dim 1 (CartpoleEnv), either include_action; other shapes return B200RL_EUNSUPPORTED.
 * The update passes take the lane geometry (N lanes, T steps, B = N T samples, planes [.][T][N]) and tstep, from
 * which they rebuild each lane's inputs and hidden states. ---- */

/* Number of GRU policy parameters P (including log_std); <0 if the shape is not compiled in. */
long long b200rl_gru_num_params(int obs_dim, int hidden, int act_dim, int include_action);

/* One GRU step for n rows (GaussianGRUPolicy.get_action, vectorised): obs [O][n], prev_action [A][n] (NULL = 0), h_in
 * [H][n] (NULL = 0) -> act_out = mean + exp(log_std) eps, mean_out [A][n], h_out [H][n], log_std_out [A].  eps [A][n]
 * or NULL (Philox stream 0 at (lane0 + i, row), as b200rl_policy_get_actions). */
int b200rl_gru_get_actions(const float* params_f32, int obs_dim, int hidden, int act_dim, int include_action,
                           const float* obs, const float* prev_action, const float* h_in, long long n, const float* eps,
                           unsigned int seed, unsigned int iter, int row, long long lane0, float* act_out,
                           float* mean_out, float* h_out, float* log_std_out, void* stream);

/* Fused rollout with the GRU policy: b200rl_rollout's lane semantics and planes (obs, raw act, mean, rew, flags, tstep,
 * log_std_out), with h and prev_action carried per lane and reset at every path start. */
int b200rl_rollout_gru(int env_kind, const float* params_f32, int hidden, int include_action, int N, int T,
                       int max_path_length, const float* eps, const float* reset_raw, unsigned int seed,
                       unsigned int iter, long long lane0, float* obs, float* act, float* mean, float* rew,
                       unsigned char* flags, unsigned short* tstep, float* log_std_out, void* stream);

/* (loss, sum KL, max KL) as b200rl_loss_kl over the lane batch (npo.py:67-82 with valids = not FLAG_MASKED);
 * h_cache_out ([H][T][N] or NULL) receives h_t. */
int b200rl_gru_loss_kl(int loss_kind, const float* params_f32, int obs_dim, int hidden, int act_dim,
                       int include_action, int N, int T, const float* obs, const float* act,
                       const unsigned short* tstep, const float* adv, const float* old_mean, const float* old_log_std,
                       const unsigned char* flags, double scale, const double* count, double* out, float* h_cache_out,
                       double* ws, void* stream);

/* Backpropagation-through-time gradient of the surrogate plus penalty * mean KL (penalty 0: b200rl_grad, > 0:
 * b200rl_grad_penalized); loss_out (3 or NULL) the unpenalised triple.  h_cache [H][T][N] is required: the forward sweep
 * writes h_t there and the backward sweep reads it (a later b200rl_gru_fvp may reuse it with h_valid = 1). */
int b200rl_gru_grad(int loss_kind, double penalty, const float* params_f32, int obs_dim, int hidden, int act_dim,
                    int include_action, int N, int T, const float* obs, const float* act, const unsigned short* tstep,
                    const float* adv, const float* old_mean, const float* old_log_std, const unsigned char* flags,
                    double scale, const double* count, double* g_out, double* loss_out, float* h_cache, double* ws,
                    void* stream);

/* Fisher-vector product J^T M J x (+ diag_scale * reg_coeff * x, and the log_std block) at theta_old, as b200rl_fvp:
 * a forward tangent sweep carries J x through h and writes M J x per sample into the workspace, then the gradient
 * pass's backward sweep runs on those deltas.  h_cache [H][T][N] is required; h_valid != 0: it already holds h_t at
 * these parameters (b200rl_gru_grad wrote it), else it is rewritten. */
int b200rl_gru_fvp(const float* params_f32, int obs_dim, int hidden, int act_dim, int include_action, int N, int T,
                   const float* obs, const float* act, const unsigned short* tstep, const unsigned char* flags,
                   const double* x, double scale, const double* count, double reg_coeff, double diag_scale,
                   double* Hx_out, float* h_cache, int h_valid, double* ws, void* stream);

/* float64 parity mode of the passes above on the float64 master parameters, as b200rl_update_f64 (mode 0 loss/KL, 1
 * gradient, 2 Fisher-vector product; loss_kind B200RL_LOSS_KL with mode 1 = gradient of mean KL for
 * FiniteDifferenceHvp).  h64 [H + A][T][N] float64 scratch (hidden states, and M J x in mode 2).  Weight gradients are
 * summed with float64 atomics: reruns agree to rounding. */
int b200rl_gru_update_f64(int mode, int loss_kind, const double* params_f64, int obs_dim, int hidden, int act_dim,
                          int include_action, int N, int T, const float* obs, const float* act,
                          const unsigned short* tstep, const float* adv, const float* old_mean,
                          const float* old_log_std, const unsigned char* flags, const double* x, double scale,
                          const double* count, double reg_coeff, double diag_scale, double* vec_out, double* loss_out,
                          double* h64, double* ws, void* stream);

/* ---- CategoricalGRUPolicy (rllab/policies/categorical_gru_policy.py, rllab/core/network.py GRUNetwork with a softmax
 * output, rllab/distributions/recurrent_categorical.py).  The GaussianGRUPolicy cell above with x_t = [obs_t, one-hot
 * prev_action_t] (include_action != 0) or obs_t, logits z = h' W_out + b_out and prob = softmax(z); no log_std.  Flat
 * layout [W_xr, W_hr, b_r, W_xu, W_hu, b_u, W_xc, W_hc, b_c, W_out (H x n), b_out (n)].  h = 0 and prev_action = 0 at a
 * path start; inside a path prev_action is the previous one-hot action act[t-1].  Compiled for obs_dim 4, hidden 32,
 * n_actions 2 (CartPole-v0), either include_action; other shapes return B200RL_EUNSUPPORTED.  The entry points mirror
 * the b200rl_gru_* ones with the categorical conventions of b200rl_categorical_*: act [n][T][N] one-hot, old_prob
 * [n][T][N] in place of old_mean / old_log_std, the 1e-8 of categorical.py in the ratio and the KL, and a Fisher-vector
 * product J^T M J x with M the full n x n logit block at theta_old. ---- */
long long b200rl_categorical_gru_num_params(int obs_dim, int hidden, int n_actions, int include_action);

/* One GRU step for n rows (CategoricalGRUPolicy.get_action, vectorised): obs [O][n], prev_action [n_actions][n] one-hot
 * (NULL = 0), h_in [H][n] (NULL = 0) -> act_out [n] int32 = weighted_sample(prob, u), prob_out [n_actions][n], h_out
 * [H][n].  u [n] or NULL (Philox stream 0 at (lane0 + i, row), as b200rl_categorical_get_actions). */
int b200rl_categorical_gru_get_actions(const float* params_f32, int obs_dim, int hidden, int n_actions,
                                       int include_action, const float* obs, const float* prev_action,
                                       const float* h_in, long long n, const float* u, unsigned int seed,
                                       unsigned int iter, int row, long long lane0, int* act_out, float* prob_out,
                                       float* h_out, void* stream);

/* Fused rollout with the categorical GRU policy: b200rl_rollout_categorical's planes (obs, one-hot act, prob, rew, flags,
 * tstep) and action draw (u [T][N] or NULL = Philox stream 0 row t), with h and prev_action carried per lane and reset at
 * every path start. */
int b200rl_rollout_categorical_gru(int env_kind, const float* params_f32, int hidden, int include_action, int N, int T,
                                   int max_path_length, const float* u, const float* reset_raw, unsigned int seed,
                                   unsigned int iter, long long lane0, float* obs, float* act, float* prob, float* rew,
                                   unsigned char* flags, unsigned short* tstep, void* stream);

/* (loss, sum KL, max KL) as b200rl_gru_loss_kl with the losses of b200rl_categorical_loss_kl. */
int b200rl_categorical_gru_loss_kl(int loss_kind, const float* params_f32, int obs_dim, int hidden, int n_actions,
                                   int include_action, int N, int T, const float* obs, const float* act,
                                   const unsigned short* tstep, const float* adv, const float* old_prob,
                                   const unsigned char* flags, double scale, const double* count, double* out,
                                   float* h_cache_out, double* ws, void* stream);

/* Backpropagation-through-time gradient of the surrogate plus penalty * mean KL, as b200rl_gru_grad. */
int b200rl_categorical_gru_grad(int loss_kind, double penalty, const float* params_f32, int obs_dim, int hidden,
                                int n_actions, int include_action, int N, int T, const float* obs, const float* act,
                                const unsigned short* tstep, const float* adv, const float* old_prob,
                                const unsigned char* flags, double scale, const double* count, double* g_out,
                                double* loss_out, float* h_cache, double* ws, void* stream);

/* Fisher-vector product J^T M J x (+ diag_scale * reg_coeff * x) at theta_old, as b200rl_gru_fvp: the forward tangent
 * sweep writes M(p_old) J x per sample into plane [n_actions][T][N] (float32 scratch of the caller, so any batch that
 * fits in memory runs), then the backward sweep reads it (M as in b200rl_categorical_fvp, the O(1e-8) first-derivative
 * term left out). */
int b200rl_categorical_gru_fvp(const float* params_f32, int obs_dim, int hidden, int n_actions, int include_action,
                               int N, int T, const float* obs, const float* act, const unsigned short* tstep,
                               const unsigned char* flags, const double* x, double scale, const double* count,
                               double reg_coeff, double diag_scale, double* Hx_out, float* h_cache, int h_valid,
                               float* plane, double* ws, void* stream);

/* float64 parity mode, as b200rl_gru_update_f64 (mode 0 loss/KL, 1 gradient, B200RL_LOSS_KL with mode 1 the gradient
 * of mean KL for FiniteDifferenceHvp, 2 Fisher-vector product).  h64 [H + n][T][N] float64 scratch.  Mode 2 is the
 * Gauss-Newton product J^T M J x of the float32 pass in float64: unlike b200rl_categorical_update_f64 it leaves out the
 * O(1e-8) first-derivative term as well (DESIGN.md section 5). */
int b200rl_categorical_gru_update_f64(int mode, int loss_kind, const double* params_f64, int obs_dim, int hidden,
                                      int n_actions, int include_action, int N, int T, const float* obs,
                                      const float* act, const unsigned short* tstep, const float* adv,
                                      const float* old_prob, const unsigned char* flags, const double* x, double scale,
                                      const double* count, double reg_coeff, double diag_scale, double* vec_out,
                                      double* loss_out, double* h64, double* ws, void* stream);

/* ---- GaussianMLPRegressor, the value function of GaussianMLPBaseline (rllab/regressors/gaussian_mlp_regressor.py,
 * rllab/baselines/gaussian_mlp_baseline.py).  Net: MLP(obs_dim -> h1 -> h2 -> 1), ReLU hidden units, no output
 * nonlinearity, one state-independent log_std (rllab/core/network.py:36-81, lasagne_layers.py ParamLayer); the flat
 * parameter layout is the policy's with act_dim = 1.  Compiled for obs_dim in {2, 3, 4, 6, 13, 20}, hidden (32,32).
 * stats [2*obs_dim+2] float64 = [x_mean (O), x_std (O), y_mean, y_std], the regressor's normalisation constants. ---- */

/* Number of regressor parameters P (including log_std) for (O, h1, h2); <0 if the shape is not compiled in. */
long long b200rl_vf_num_params(int obs_dim, int h1, int h2);

/* Normalisation constants of GaussianMLPRegressor.fit (gaussian_mlp_regressor.py:197-208): column means and population
 * standard deviations (+1e-8) of obs [O][B] and y [B] over the samples not carrying B200RL_FLAG_MASKED (flags may be
 * NULL), in float64 and in two passes.  acc [2O+3] float64.  stage 0: acc[0..O+1] = (sum x_o, sum y, count); stage 1:
 * acc[O+2..2O+2] = sum (x_o - mean_o)^2, sum (y - mean_y)^2 around the means of acc[0..O+1]; stage 2: stats_out from
 * acc; stage 3: all three.  Across GPUs: all-reduce acc[0..O+1] after stage 0 and acc[O+2..] after stage 1. */
int b200rl_vf_norm_stats(int obs_dim, long long B, const float* obs, const float* y, const unsigned char* flags,
                         int stage, double* acc, double* stats_out, double* ws, void* stream);

/* Regressor mean on obs [O][B] (f_predict / the mean half of f_pdists, gaussian_mlp_regressor.py:168-169,225-231):
 * out [B] float32 = mu((x - x_mean) / x_std), times y_std plus y_mean if denormalize != 0.  Every sample is written. */
int b200rl_vf_forward(const float* params_f32, int obs_dim, int h1, int h2, long long B, const float* obs,
                      const double* stats, int denormalize, float* out, void* stream);

/* One evaluation of the regressor objective (f_opt / f_loss / f_penalized_loss of penalty_lbfgs_optimizer.py:50-77 and
 * lbfgs_optimizer.py:34-48 on the loss and mean-KL expressions of gaussian_mlp_regressor.py:150-166):
 * loss_out [3] = scale * (sum NLL, sum KL(old || new), max KL) over the valid samples (divided by *count when count is
 * not NULL), with NLL and KL of the Gaussian N(mu(nx), exp(log_std)) in normalised space against ny = (y - y_mean) /
 * y_std.  mu_old [B] float32: the normalised mean at theta_old (b200rl_vf_forward with denormalize = 0), old_log_std its
 * log_std; mu_old == NULL: no trust region (KL = 0).  g_out [P] float64 (or NULL = forward only): gradient of
 * scale * sum (NLL + penalty * KL); with learn_std == 0 the log_std slot is 0 (not a trainable parameter).
 * Arithmetic as b200rl_grad: float32 per sample and inside a 128-sample tile, float64 above; deterministic.  Reduced over
 * the ranks of the peer communicator inside the pass while b200rl_peer_fuse_updates(1) is in effect. */
int b200rl_vf_loss_grad(const float* params_f32, int obs_dim, int h1, int h2, long long B, const float* obs,
                        const float* y, const unsigned char* flags, const double* stats, const float* mu_old,
                        float old_log_std, double penalty, int learn_std, double scale, const double* count,
                        double* g_out, double* loss_out, double* ws, void* stream);

/* Workspace size (float64 entries) sufficient for every reduction above on the current device. */
long long b200rl_ws_doubles(void);

/* ---- P-vector kernels (float64, single block; krylov.cg rllab/misc/krylov.py:7-39 and the step/line-search
 * arithmetic of conjugate_gradient_optimizer.py:258-293; lasagne.updates.adam for VPG) ---- */

/* cg_state [4] float64: 0 rdotr, 1 frozen flag (rdotr < tol seen), 2 last p.z, 3 iterations done.
 * p_f32 != 0 keeps the search direction p exactly representable in float32, the precision the float32 Fisher-vector
 * kernel reads it in, so that z = A p belongs to the very p of the recurrences (krylov.cg run with floatX = float32
 * stores p in float32 as well). */
int b200rl_cg_init(long long P, const double* g, double* x, double* r, double* p, double* cg_state, int p_f32,
                   void* stream);
int b200rl_cg_step(long long P, const double* z, double* x, double* r, double* p, double* cg_state,
                   double residual_tol, int p_f32, void* stream);
/* step_out [P] = beta * x with beta = sqrt(2*delta/(x.Hx + 1e-8)) (NaN -> 1); info_out[0] = beta */
int b200rl_trpo_step_size(long long P, const double* x, const double* Hx, double max_constraint_val,
                          double* step_out, double* info_out, void* stream);
/* theta_out = theta_prev - ratio * step (float64 master) and its float32 shadow */
int b200rl_axpy_params(long long P, const double* theta_prev, const double* step, double ratio, double* theta_out,
                       float* theta_f32_out, void* stream);
/* lasagne.updates.adam: t is the 1-based step index AFTER increment (first_order_optimizer.py:21-22,62-65) */
int b200rl_adam_step(long long P, double* theta, float* theta_f32, const double* g, double* m, double* v,
                     long long t, double lr, double b1, double b2, double eps, void* stream);
int b200rl_f64_to_f32(long long n, const double* src, float* dst, void* stream);
/* Local half of the one-collective "mixed all-reduce" of rllab_b200/parallel.py: gathered [world][n] (all-gather of every
 * rank's vector) -> out[i] = sum over ranks for i < n_sum, max over ranks for i >= n_sum, in rank order. */
int b200rl_reduce_ranks(const double* gathered, int world, long long n, long long n_sum, double* out, void* stream);

/* ---- peer-memory collectives over NVLink / NVSwitch (SURVEY.md 8e; the reference's update is single-process, it has
 * no counterpart).  One process per GPU.  Every rank creates an exchange window in its own HBM, the IPC handles are
 * swapped by the host (torch.distributed / any rendezvous), every rank maps all peers' windows and binds the table.
 * A collective is ONE kernel per rank: push the vector into every window, signal, wait for all peers, fold the `world`
 * copies in rank order (bit-identical results on all ranks).  See rllab_b200/csrc/peer.cuh. */
#define B200RL_PEER_MAX_RANKS 16
#define B200RL_IPC_HANDLE_BYTES 64
long long b200rl_peer_window_bytes(int world, long long n_cap);
/* window of `world` x 2 slots of n_cap float64 (+ flags), zeroed; handle_out [B200RL_IPC_HANDLE_BYTES] */
int b200rl_peer_window_create(int world, long long n_cap, void** window_out, unsigned char* handle_out);
int b200rl_peer_window_open(const unsigned char* handle, void** window_out);    /* map a peer's window */
int b200rl_peer_window_close(void* window);                                      /* unmap a peer's window */
int b200rl_peer_window_destroy(void* window);                                    /* free the own window */
/* windows [world]: device base pointers indexed by rank (entry `rank` = own window); NULL / world <= 1 unbinds */
int b200rl_peer_bind(void* const* windows, int rank, int world, long long n_cap);
/* in place: t[i] = sum over ranks (i < n_sum) | max over ranks (i >= n_sum); n <= n_cap */
int b200rl_peer_allreduce_mixed(double* t, long long n, long long n_sum, void* stream);
/* enable != 0: until switched off again, b200rl_loss_kl / b200rl_grad / b200rl_fvp / b200rl_update_f64 deliver results
 * reduced over ALL ranks -- the exchange is fused into the finalize kernel of the pass (one launch: fold the per-block
 * partials, push into the peers' windows, fold over ranks).  Every rank must issue the same sequence of calls. */
int b200rl_peer_fuse_updates(int enable);
/* Number of collectives of this rank that gave up waiting (30 s) for a peer; their results were poisoned with NaN.
 * Synchronising device->host read: call it at the end of a job, not inside the iteration. */
int b200rl_peer_timeouts(unsigned int* count_out_host);

/* ---- Cross-entropy method (rllab/algos/cem.py): a population of policies, one parameter row per member. ---- */

/* Parameter rows of CEM._worker_rollout_policy (cem.py:30-36, `np.random.standard_normal(K) * sample_std + cur_mean`):
 * theta_out [n][P] float64, row r = member m_r = members[r] (device int64 list) or member0 + r (members NULL):
 * theta[r][k] = cur_mean[k] + sample_std[k] * eps(seed, iter, m_r, k), sample_std[k] = sqrt(cur_std[k]^2 + extra_var)
 * (cem.py:117-118 with extra_var = extra_std^2 * max(1 - itr / extra_decay_time, 0)).  eps is Philox stream 2 (lane = m,
 * row 0, chunk k / 4) through the normal map of b200rl_fill_noise; every float64 operation is explicitly rounded, so the
 * same arithmetic in NumPy on the same eps gives the same bits.  Rows are a pure function of (seed, iter, m, cur_mean,
 * cur_std, extra_var): a rank can regenerate any member's row. */
int b200rl_population_sample(long long P, const double* cur_mean, const double* cur_std, double extra_var,
                             unsigned int seed, unsigned int iter, const long long* members, long long member0, int n,
                             double* theta_out, void* stream);

/* n_evals episodes of each of M policies (cem.py:37-57 over rollout, rllab/sampler/utils.py:6-43): member m's policy is
 * row m of theta [M][P] float64 (rounded to float32 when staged).  Every episode starts from reset and runs to done or
 * max_path_length (no auto-reset, nothing per step written); episode (m, e) uses lane lane0 + m*n_evals + e for its
 * action and reset noise and is bit-identical to the first path of lane e of b200rl_rollout(theta_m as float32,
 * N = n_evals, lane0 = lane0 + m*n_evals, same seed / iter).  Outputs [M][n_evals]: ret_out = discounted return
 * (discount_cumsum(rewards, discount)[0], float64 accumulated in the kernel), undisc_out = sum of rewards, len_out = episode
 * length; obs_first / obs_last [M][n_evals][O] (both NULL or both set) = the episode's first and last observation.
 * member_out [M][3] = (fitness mean(ret) - std(ret, ddof)/sqrt(n_evals), the same statistic of undisc, mean over action
 * dims of the member's action std exp(max(log_std, log(min_std)))), ddof = 1 if n_evals > 1 else 0 (cem.py:15-27).
 * ws: workspace of b200rl_ws_doubles() entries (its first word is the persistent grid's work counter). */
int b200rl_population_rollout(int env_kind, int h1, int h2, float min_std, const double* theta, int M, int n_evals,
                              int max_path_length, double discount, unsigned int seed, unsigned int iter,
                              long long lane0, double* ret_out, double* undisc_out, int* len_out, float* obs_first,
                              float* obs_last, double* member_out, double* ws, void* stream);

/* Elite indices of CEM.train (cem.py:138, `(-fs).argsort()[:n_best]`): idx_out [k] int64 = the indices of the k largest of
 * f [M] float64 in descending order, ties to the lower index, NaN last; deterministic, no host sort.  k <= M. */
int b200rl_population_topk(const double* f, int M, int k, long long* idx_out, double* ws, void* stream);

/* cur_mean / cur_std of CEM.train (cem.py:140-141): mean_out, std_out [P] = column mean and population std (ddof 0) of
 * rows [k][P] float64, summed over the rows in row order with explicitly rounded operations (NumPy's axis-0 reduction). */
int b200rl_rows_mean_std(long long P, int k, const double* rows, double* mean_out, double* std_out, void* stream);

/* ---- Relative entropy policy search (rllab/algos/reps.py): the dual g(eta, v) over the lane batch. ----
 * Sample (t, n) has the Bellman error delta = rew + (phi(t+1, n) - phi(t, n)) . v with the LinearFeatureBaseline feature
 * map phi = [clip(o, +-10), o^2, al, al^2, al^3, 1], al = tstep / 100 (reps.py:207-211), and phi(t+1, n) = 0 when (t, n)
 * carries B200RL_FLAG_END (the per-path feat_diff of reps.py:227-238, including a path cut by the end of the buffer).
 * v [2*obs_dim+4] float64.  masked != 0: samples carrying B200RL_FLAG_MASKED are left out of the maximum and every sum.
 * float64 arithmetic, two-stage fixed-order reductions (bit-identical reruns).  obs_dim in {2, 3, 4, 6, 13, 20}, else
 * B200RL_EUNSUPPORTED.  Across GPUs: all-reduce out_max (max) before b200rl_reps_dual_sums, and `out` (sum) after it. */

/* out_max[0] = M = max delta over this GPU's valid samples (the max(delta_v / eta) shift of reps.py:107,169-172). */
int b200rl_reps_delta_max(int obs_dim, int N, int T, const float* obs, const float* rew, const unsigned char* flags,
                          const unsigned short* tstep, int masked, const double* v, double* out_max, double* ws,
                          void* stream);

/* The sums behind the dual and its gradient (reps.py:164-187), with e = exp((delta - M) / eta) and M = *M (device):
 * out [2*obs_dim+6] float64 = [sum e, sum e (delta - M), sum e feat_diff (2*obs_dim+4 entries)] over the valid samples.
 * The caller forms g = eta eps + eta log(sum e / count) + M (+ L2 term) and its gradient from them.  w_out ([T][N] float32
 * or NULL) receives e per sample (0 on masked samples): the weights of the policy loss of reps.py:110-112. */
int b200rl_reps_dual_sums(int obs_dim, int N, int T, const float* obs, const float* rew, const unsigned char* flags,
                          const unsigned short* tstep, int masked, const double* v, double eta, const double* M,
                          double* out, float* w_out, double* ws, void* stream);

/* (T,N)-planar lane layout <-> the reference's sample-major (B, dim) float64 wire format
 * (samples_data["observations"] etc., rllab/sampler/base.py:74-104): dst[(t*N+n)*dim + k] = src[k][t][n]. */
int b200rl_planes_to_rows_f64(int dim, long long B, const float* src, double* dst, void* stream);

/* ---- DDPG (rllab/algos/ddpg.py) with DeterministicMLPPolicy and ContinuousMLPQFunction. ----
 * Env kinds: the classic-control Box kinds (point, cartpole, pendulum, cartpole_swingup, double_pendulum); planar and
 * discrete kinds return B200RL_EUNSUPPORTED.  Both nets are (32, 32) with ReLU hidden units.
 *   policy (deterministic_mlp_policy.py): [h0.W (O,32), h0.b, h1.W (32,32), h1.b, output.W (32,A), output.b], tanh out;
 *   qf (continuous_mlp_q_function.py, action_merge_layer = -2): [h1.W (O,32), h1.b, h2.W (32+A,32) (hidden rows, then
 *   action rows), h2.b, output.W (32,1), output.b], linear out.
 * A run's network state `nets` is [4][P] float64 with P = P_policy + P_qf: theta, Adam m, Adam v, target, each laid out
 * [policy | qf].  Adam is lasagne.updates.adam (beta1 0.9, beta2 0.999, epsilon 1e-8) with one step count for both
 * nets.  Minibatch size 32.
 *
 * Philox draws of run r at step itr (itr_lo = itr & 0x0FFFFFFF, itr_hi = itr >> 28):
 *   counter (r, itr_lo | stream << 28, sub, 0), key (seed, itr_hi)
 *   stream 1 (the reset stream): sub = chunk; a path's reset at step itr (the first reset at itr = 0)
 *   stream B200RL_DDPG_STREAM_EXPLORE: sub = chunk c holds the N(0,1) draws of action entries 4c..4c+3 (Box-Muller on
 *     word pairs, u = (w + 0.5) * 2^-32, float64: rad = sqrt(-2 log u0), n0 = rad cos(2 pi u1), n1 = rad sin(2 pi u1))
 *   stream B200RL_DDPG_STREAM_INDEX: sub = (update << 16) | (candidate >> 2), word candidate & 3; candidate j of update
 *     `update` maps to index = (bottom + ((uint64)w * size >> 32)) % replay_pool_size and is rejected when
 *     index == size - 1 (SimpleReplayPool.random_batch); the first 32 accepted candidates form the minibatch. */
#define B200RL_DDPG_BATCH 32
#define B200RL_DDPG_STREAM_EXPLORE 3
#define B200RL_DDPG_STREAM_INDEX 4
#define B200RL_ES_OU 0       /* rllab/exploration_strategies/ou_strategy.py */
#define B200RL_ES_GAUSSIAN 1 /* rllab/exploration_strategies/gaussian_strategy.py */
/* per-run statistics, float64, summed over the updates of every launch since the caller last cleared them */
#define B200RL_DDPG_NSTAT 9  /* n_updates, qf_loss, policy_surr, q, |q|, y, |y|, |q - y|, n_es_returns */

typedef struct {
  int n_updates_per_sample, max_path_length, min_pool_size, replay_pool_size;
  int include_horizon_terminal_transitions, es_kind;
  double discount, scale_reward, soft_target_tau;
  double qf_weight_decay, qf_learning_rate, policy_weight_decay, policy_learning_rate;
  double ou_mu, ou_theta, ou_sigma;                   /* OUStrategy */
  double gs_max_sigma, gs_min_sigma, gs_decay_period; /* GaussianStrategy */
} b200rl_ddpg_hparams;

/* The train() loop's state of one run between launches.  terminal: 0 = inside a path, 1 = the last step ended a path
 * (the next step resets and records path_return as an Es return), 2 = a fresh run (the next step resets, no return). */
typedef struct {
  float env_state[8];
  float obs[8];
  double ou_state[4];
  double path_return;
  long long itr, adam_t;
  int path_length, terminal, top, bottom, size, pad_;
} b200rl_ddpg_state;

typedef struct {
  int env_kind, f64;      /* f64: nets, backward passes and Adam in float64 (parity mode); the env is float32 always */
  int n_runs, n_steps;    /* one CTA per run; n_steps of the train() loop per launch */
  int es_cap;             /* capacity of each run's es_returns row */
  unsigned int seed;
  b200rl_ddpg_hparams hp;
  b200rl_ddpg_state* state;   /* [n_runs] */
  double* nets;               /* [n_runs][4][P] */
  float* pool_obs;            /* [n_runs][replay_pool_size][O] */
  float* pool_act;            /* [n_runs][replay_pool_size][A] */
  float* pool_rew;            /* [n_runs][replay_pool_size], reward * scale_reward */
  unsigned char* pool_term;   /* [n_runs][replay_pool_size] */
  double* stats;              /* [n_runs][B200RL_DDPG_NSTAT], accumulated */
  double* es_returns;         /* [n_runs][es_cap]: returns of the finished exploration paths, at stats[8] */
  void* stream;
} b200rl_ddpg_train_args;

/* P of the policy (which = 0) or the Q function (which = 1); negative when (obs_dim, act_dim) is not compiled in. */
long long b200rl_ddpg_num_params(int obs_dim, int act_dim, int which);

/* DeterministicMLPPolicy.get_actions: obs [O][n], act_out [A][n], policy parameters float32. */
int b200rl_deterministic_get_actions(const float* params_f32, int obs_dim, int act_dim, const float* obs, long long n,
                                     float* act_out, void* stream);

/* ContinuousMLPQFunction.get_qval: obs [O][n], act [A][n], q_out [n], Q parameters float32. */
int b200rl_qf_get_qval(const float* params_f32, int obs_dim, int act_dim, const float* obs, const float* act,
                       long long n, float* q_out, void* stream);

/* Noise-free lane rollout of the deterministic policy (the paths DDPG.evaluate samples), layouts of b200rl_rollout;
 * act receives the policy's output. */
int b200rl_rollout_deterministic(int env_kind, const float* params_f32, int N, int T, int max_path_length,
                                 const float* reset_raw, unsigned int seed, unsigned int iter, long long lane0, float* obs,
                                 float* act, float* rew, unsigned char* flags, unsigned short* tstep, void* stream);

/* One DDPG.do_training on the minibatch idx [32] (int) of one run's pool (layouts of b200rl_ddpg_train_args, pool of
 * pool_size rows): updates nets [4][P] in place with Adam step adam_t (>= 1) and writes grad_out [P] (the two loss
 * gradients with their weight decay, [policy | qf]), qval_out [32] and y_out [32] (float64) and
 * loss_out [2] = (qf_loss, policy_surr), both before their update.  Runs the fused loop's update code. */
int b200rl_ddpg_update(int env_kind, int f64, const b200rl_ddpg_hparams* hp, const float* pool_obs,
                       const float* pool_act, const float* pool_rew, const unsigned char* pool_term, int pool_size,
                       const int* idx, double* nets, long long adam_t, double* grad_out, double* qval_out,
                       double* y_out, double* loss_out, void* stream);

/* n_steps of DDPG.train()'s loop for n_runs independent runs in one launch; see b200rl_ddpg_train_args. */
int b200rl_ddpg_train(const b200rl_ddpg_train_args* args);

#ifdef __cplusplus
}
#endif
#endif /* B200RL_H_ */
