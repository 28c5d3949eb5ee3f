/*
 * rl4rs_b200.h -- C-ABI of the H100-native RL4RS hot path (librl4rs_b200.so).
 *
 * The reference has no FFI: its "operator API" for this path is the Python protocol
 * RecEnvBase / RecSimBase / RecState (rl4rs/env/base.py:26-57,111-175,178-273).  Each entry
 * point below names the reference interface it replaces (file:line under /root/reference).
 * The Python mirror of those classes (rl4rs_b200/env/) binds this library through ctypes
 * (rl4rs_b200/_capi.py); INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions: plain pointers and sizes only (no torch types); return 0 on success, a negative
 * r4_status otherwise, r4_last_error() gives the message; nothing throws across the ABI.
 * "dev" pointers are device memory owned by the CALLER (allocated by torch on the Python side);
 * the library only borrows them for the work it enqueues on `stream` (a cudaStream_t passed as
 * void*; NULL = legacy default stream).  Every call is asynchronous on that stream.  One r4_env
 * per device, not thread-safe (the reference is single-threaded, base.py:119-130); distinct
 * handles are independent.
 */
#ifndef RL4RS_B200_H
#define RL4RS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct r4_env r4_env;

typedef enum {
  R4_OK = 0,
  R4_ERR_ARG = -1,      /* bad argument / unsupported configuration */
  R4_ERR_STATE = -2,    /* call out of order (e.g. step before reset, step past max_steps) */
  R4_ERR_CUDA = -3,     /* CUDA runtime error (message holds cudaGetErrorString) */
  R4_ERR_NOMEM = -4
} r4_status;

/* config['...'] flags read by the reference via config.get (slate.py:22,92,98,153,245,250,299) */
enum {
  R4_FLAG_RLLIB_MASK = 1,     /* support_rllib_mask */
  R4_FLAG_D3RL_MASK = 2,      /* support_d3rl_mask */
  R4_FLAG_CONTI = 4,          /* support_conti_env */
  R4_FLAG_ONEHOT = 8,         /* support_onehot_action (action_emb = eye(action_size)) */
  R4_FLAG_RAWSTATE = 16,      /* rawstate_as_obs: no simulator forward for observations */
  R4_FLAG_INFO_FETCH = 32     /* simulator_info_fetch: expose per-item click probabilities */
};

enum { R4_ENV_SLATE = 0, R4_ENV_SEQSLATE = 1 };   /* rl4rs/__init__.py:10-18 */
/* config['algo'] (slate.py:239-242): which rl4rs/nets/<algo>.py graph the simulator is.
 *   DIEN  nets/dien.py:8-45   (sequence GRU/attention/AUGRU + dense tower + category attention; tensor-bound)
 *   DNN   nets/dnn.py:8-45    (mean-pooled category embeddings + dense tower + FC 256 + simulator_obs; gather-bound:
 *                              the sequence branch of that graph does not reach the output and is not evaluated)
 *   WIDEDEEP  nets/widedeep.py:8-45 (mean-pooled sequence embeddings -> Dense 256 | dense tower | flattened category
 *                              embeddings; 'simulator_obs' IS that 3072-wide concat, so obs buffers are f32 [B,3072])
 *   LSTM  nets/lstm.py:8-45   (Keras GRU -- hard sigmoid, reset_after False -- over each behaviour sequence and over the 21
 *                              category embeddings | dense tower | flattened category embeddings -> simulator_obs 256) */
enum { R4_SIM_DIEN = 0, R4_SIM_DNN = 1, R4_SIM_WIDEDEEP = 2, R4_SIM_LSTM = 3 };
/* width of the observation a simulator produces (256, or 3072 for widedeep) */
int r4_obs_dim(int simulator);

/* The config dict of the reference scripts (simulator_eval.py:9-12, modelfree_train.py:32-37). */
typedef struct {
  int32_t env_kind;             /* R4_ENV_SLATE | R4_ENV_SEQSLATE */
  int32_t flags;                /* R4_FLAG_* */
  int32_t batch_size;
  int32_t max_steps;            /* 9 (Slate) / 27 or 36 (SeqSlate) */
  int32_t page_items;           /* 9 */
  int32_t action_size;          /* 284 */
  int32_t action_emb_size;      /* 32 (ignored with R4_FLAG_ONEHOT) */
  int32_t maxlen;               /* 64 */
  int32_t seq_num;              /* 2 */
  int32_t dense_feature_num;    /* 432 */
  int32_t category_feature_num; /* 21 */
  int32_t category_hash_size;   /* 100000 */
  int32_t emb_size;             /* 128 */
  int32_t hidden_units;         /* 128 */
  int32_t max_rows_per_pass;    /* 0 = default; bound on simulator rows per launch group */
  int32_t simulator;            /* R4_SIM_DIEN | R4_SIM_DNN | R4_SIM_WIDEDEEP | R4_SIM_LSTM (ABI version >= 2) */
} r4_config;

/* Per-call output buffers (device, caller-owned).  NULL = not wanted.
 * Replaces the return values of RecSimBase._step / sample (base.py:157-175) and
 * SlateRecEnv.obs_fn (slate.py:244-279). */
typedef struct {
  float*   obs;          /* f32 [B,256]   simulator_obs layer (dien.py:35; [B,3072] for widedeep); NULL with RAWSTATE */
  uint8_t* action_mask;  /* u8  [B,A]     action_mask & location_mask & special_mask (slate.py:93-97) */
  double*  reward;       /* f64 [B]       slate.py:281-308 / seqslate.py:136-160 */
  uint8_t* done;         /* u8  [B]       base.py:165-168 */
  int32_t* chosen;       /* i32 [B]       item ids actually placed (kNN result in conti mode) */
  int32_t* cat;          /* i32 [B,21]    category_feature of the new state (datautil.py:59-65) */
  float*   dense;        /* f32 [B,432]   dense_feature (datautil.py:52-58) */
  int32_t* seq;          /* i32 [B,2,64]  sequence_feature (datautil.py:43-47) */
  float*   click_p;      /* f32 [B,9]     probs[:,1] of the reward pass (slate.py:298-301); written
                                          only on steps that compute a reward */
  int32_t* masked_actions; /* i32 [B,9|max_steps] d3rl 'masked_actions' (slate.py:98-104, seqslate.py:18-23) */
} r4_out;

/* ---- lifetime ---------------------------------------------------------------------------- */
/* SlateRecEnv.__init__/RecSimBase.__init__ (slate.py:223-237, base.py:114-131) */
int r4_create(const r4_config* cfg, int device, r4_env** out);
void r4_destroy(r4_env* env);
const char* r4_last_error(const r4_env* env);   /* env may be NULL: error of the last failed r4_create */

/* ---- static data ------------------------------------------------------------------------- */
/* SlateState.get_iteminfo_from_file / get_mask_from_file (slate.py:28-65).  HOST pointers,
 * n = action_size rows, row 0 = the implicit padding item.  special[i] != 0 marks the ids whose
 * special column == 2.  action_emb is f64 [n, emb_dim] (slate.py:47-52; eye(n) with ONEHOT). */
int r4_load_items(r4_env* env, const double* item_vec, int vec_dim, const double* price,
                  const uint8_t* special, const double* action_emb, int emb_dim, int n);

/* tf.train.Saver.restore (base.py:148-151): one named f32 tensor of the W-table (SURVEY.md 8a);
 * `data` may be a host or a device pointer.  r4_finalize_weights derives the fused layouts. */
int r4_load_weight(r4_env* env, const char* name, const float* data, const int64_t* shape, int rank);
int r4_finalize_weights(r4_env* env, void* stream);

/* RecDataBase (base.py:60-108): the parsed log, structure-of-arrays, DEVICE pointers that must
 * stay valid until the next r4_load_log / r4_destroy.  user_seq is pre-padded/truncated to maxlen
 * (datautil.py:43-46).  n_slots = 9 (dataset A) or 36 (b3 trajectories). */
int r4_load_log(r4_env* env, const int32_t* user_cat /*[N,10]*/, const float* user_dense /*[N,32]*/,
                const int32_t* user_seq /*[N,maxlen]*/, const int32_t* logged_items /*[N,n_slots]*/,
                const uint8_t* feedback /*[N,n_slots]*/, int64_t n_rows, int n_slots);

/* ---- episode ----------------------------------------------------------------------------- */
/* RecEnvBase.reset -> RecSimBase.sample (base.py:265-269,172-175): row_idx i32[B] (device) are
 * the log rows RecDataBase.sample chose (base.py:92-100). */
int r4_reset(r4_env* env, const int32_t* row_idx, const r4_out* out, void* stream);

/* RecEnvBase.step -> RecSimBase._step (base.py:256-263,157-170) -> SlateState.act
 * (slate.py:193-214 / seqslate.py:92-126).  action: i32[B] item ids, or with R4_FLAG_CONTI
 * f32[B,emb] (action_is_f64 = 0) / f64[B,emb] (action_is_f64 = 1) embeddings resolved by
 * get_nearest_neighbor_with_mask (slate.py:186-191). */
int r4_step(r4_env* env, const void* action, int action_is_f64, const r4_out* out, void* stream);

/* SlateState.offline_action / offline_reward (slate.py:149-174, seqslate.py:71-86).
 * items: i32[B]; emb (conti mode, may be NULL): f64[B,emb_dim]; reward: f64[B]. */
int r4_offline_action(r4_env* env, int32_t* items, double* emb, void* stream);
int r4_offline_reward(r4_env* env, double* reward, void* stream);

/* SlateState.get_violation (slate.py:133-147 / seqslate.py:52-69): i32[B] of 0/1. */
int r4_violation(r4_env* env, int32_t* out, void* stream);

/* The raw feature rows of the CURRENT state -- what RecState.state hands to obs_fn (slate.py:90-106, built by
 * slate.py:67-83,203-213 and padded by FeatureUtil.feature_extraction, datautil.py:34-69) -- without a simulator
 * pass: cat i32[B,21], dense f32[B,432], seq i32[B,2,64] (any may be NULL).  For custom obs_fn plug-ins. */
int r4_features(r4_env* env, int32_t* cat, float* dense, int32_t* seq, void* stream);

/* SlateState.get_nearest_neighbor (static, unmasked; slate.py:180-184; tutorial.ipynb:251-254) */
int r4_nearest_neighbor(r4_env* env, const void* action, int action_is_f64, int n, int32_t* out,
                        void* stream);

/* ---- introspection ----------------------------------------------------------------------- */
int r4_cur_steps(const r4_env* env);                 /* SlateState.cur_steps */
const int32_t* r4_prev_actions(const r4_env* env);   /* device i32[B,max_steps] (SlateState.prev_actions) */
int r4_copy_prev_actions(r4_env* env, int32_t* out /*dev i32[B,max_steps]*/, void* stream);
/* kernel launches issued by this handle since creation (bench.py's gpu_launches) */
int64_t r4_launch_count(const r4_env* env);
/* Per-kernel timing with CUDA events on the launching stream (bench.py's roofline leg).
 * mode 0 = off, 1 = the dominant kernel only (k_recur<256>, the AUGRU recurrence), 2 = every kernel.
 * r4_profile resets the counters; r4_profile_read synchronises the recorded events and returns, for
 * slot = 0,1,2,... the kernel name, summed device milliseconds, launches and algorithmic work
 * (FLOPs for the GEMM-shaped kernels, rows otherwise); it returns 1 past the last slot. */
int r4_profile(r4_env* env, int mode);
int r4_profile_read(r4_env* env, int slot, const char** name, double* ms, int64_t* launches, double* work);
/* ABI version of the build */
int r4_abi_version(void);
/* Wave-count rule between two AUGRU kernel shapes (2 = one recurrence per CTA pair, 3 = two per pair) for `ctas` =
 * 2 x ceil(rows / 128) tile-sequences on a device with `sms` multiprocessors; 0 for bad arguments.  Pure host arithmetic.
 * This build has ONE AUGRU kernel (k_augru_tc, wgmma): the rule and the "augru_*" / "scores_impl" options below are kept
 * for ABI compatibility and do not change which kernel runs.  No reference counterpart. */
int r4_augru_kernel_for(int ctas, int sms);
/* Process-wide kernel-choice overrides for parity tests and A/B timing (no reference counterpart):
 *   "augru_kernel"     0 = by r4_augru_kernel_for (default), 2 = always the pair kernel, 3 = always the ping-pong pair kernel
 *                      (two recurrences per pair)
 *   "augru_pair_impl"  hand-over / weight-ring variant of the pair kernels, <RELAY, TMAP>: 1 = <0,0> (default: direct
 *                      release.cta arrive, per-CTA bulk-copy ring), 2 = <0,1> (tensor-map ring), 3 = <1,0> (relayed
 *                      release.cluster hand-over), 4 = <1,1>
 *   "augru_cost_pair" / "augru_cost_pp"  the per-wave costs r4_augru_kernel_for compares (positive ints)
 *   "augru_cluster"    CTAs per cluster of the pair kernel: 2 (one pair), 4 or 8 (2 / 4 pairs share one multicast weight stream)
 *   "pay_obs_reuse"    1 (default): r4_step takes the observation of a PAYING step (the last step of a slate / page) from that
 *                      step's reward pass -- the state the step leaves (rl4rs/env/slate.py:203-213, seqslate.py:104-122) is the
 *                      last of the page's complete states (slate.py:117-131, seqslate.py:27-50), so the reference runs the same
 *                      feature row through the simulator twice; 0: launch the separate observation pass as well
 *   "scores_impl"      DIN attention scores (nets/utils.py:121-122): 2 (default) = k_scores_tc2, both attention layers on the
 *                      tensor pipe with the second GEMM's A operand in tensor memory; 1 = k_scores_tc (second layer as FMAs)
 *   "scores_shared_pct" share of an even CTA split given to a sequence whose cached rows are shared by all feature rows
 *                      (Slate's constant second sequence), 10..100 per cent
 * The environment variables R4_AUGRU_PAIR / R4_AUGRU_PP / R4_AUGRU_PAIR_IMPL / R4_AUGRU_RULE / R4_NO_PAY_OBS_REUSE / R4_SCORES_IMPL give the initial
 * values.  Returns 0, or R4_ERR_ARG for an unknown key / out-of-range value. */
int r4_set_option(const char* key, int value);

/* ---- policy + learner (K12): MyMaskActionsModel (rllib_mask_model.py:41-62) and the RLlib PPO / A2C losses ----
 * Stateless: every pointer is caller-owned DEVICE memory.  Flat parameter layout:
 * w1[256,64] b1[64] w2[64,A] b2[A] wv[64] bv[1]  (r4_policy_num_params(A) floats). */
int r4_policy_num_params(int action_size);
/* forward + SoftQ(T=1) sampling (explore != 0) or argmax (modelfree_train.py:398-402,412-414); obs f32[n,256],
 * mask u8[n,A] -> action i32[n], logp f32[n], value f32[n], logits f32[n,A] (masked logits; may be NULL). */
int r4_policy_act(const float* params, const float* obs, const uint8_t* mask, int n, int action_size, int explore,
                  uint64_t seed, uint64_t counter, int32_t* action, float* logp, float* value, float* logits,
                  void* stream);
/* gradient of the RLlib loss over samples idx[0..n) (NULL = 0..n-1) of a rollout:
 * mode 0 PPO surrogate (mean; modelfree_train.py:179-217), mode 1 A2C (sums; :248-304).
 * scratch: f32[G * (num_params + 5)], G = min(ceil(n/4), 148) CTAs; flat_grad f32[num_params] receives the
 * deterministic sum; stats_accum f32[5] += {policy_loss, vf_loss, kl, entropy, total} * stat_scale. */
int r4_policy_grad(int mode, const float* params, const float* obs, const uint8_t* mask, const int64_t* action,
                   const float* old_logp, const float* old_logits, const float* old_value, const float* adv,
                   const float* target, const int64_t* idx, int n, int action_size, float clip, float vf_clip,
                   float vf_coeff, float kl_coeff, float ent_coeff, float inv_n, float* scratch, int G,
                   float* flat_grad, float* stats_accum, float stat_scale, void* stream);
/* Generalised advantage estimation over complete episodes (RLlib postprocessing compute_advantages, bootstrap value 0):
 * reward / value / adv / target are f32 [T, B] device arrays; target = adv + value; gamma_lambda = the product gamma * lambda
 * (rounded once by the caller, as the reference's float arithmetic does).  One launch instead of a host loop. */
int r4_gae(const float* reward, const float* value, int T, int B, float gamma, float gamma_lambda, float* adv, float* target, void* stream);
/* Adam (torch.optim.Adam semantics) with optional global-norm clipping (clip <= 0 off; norm_scratch f32[1]).
 * grad_scale multiplies the gradient first (1/world after a SUM all-reduce). step is 1-based. */
int r4_adam_step(float* params, const float* grad, float* m, float* v, int n, int step, float lr, float beta1,
                 float beta2, float eps, float grad_scale, float clip, float* norm_scratch, void* stream);

/* One PPO SGD epoch on a single GPU (num_sgd_iter = 1 of modelfree_train.py:179-217): for every full minibatch
 * perm[s .. s+mb) of the rollout, r4_policy_grad (mode 0, mean over mb) followed by r4_adam_step, with no host round
 * trip between the steps.  step0 = Adam steps already taken; returns the number of steps done (>= 0) or a negative
 * r4_status.  Multi-GPU learners call r4_policy_grad / all-reduce / r4_adam_step per step instead. */
int r4_ppo_epoch(float* params, const float* obs, const uint8_t* mask, const int64_t* action, const float* old_logp,
                 const float* old_logits, const float* old_value, const float* adv, const float* target,
                 const int64_t* perm, int n, int mb, int action_size, float clip, float vf_clip, float vf_coeff,
                 float kl_coeff, float ent_coeff, float* scratch, float* flat_grad, float* stats_accum, float* m,
                 float* v, int step0, float lr, float beta1, float beta2, float eps, float grad_clip,
                 float* norm_scratch, void* stream);

/* ---- data-parallel learner: gradient exchange over NVLink peer memory (SURVEY.md 8e; no reference counterpart:
 * the reference's multi-worker path is Ray's object store, modelfree_train.py:181,403-405) ----------------------
 * One communicator per rank (= process = GPU).  r4_comm_create allocates this rank's inbox + flags on the CURRENT
 * device; r4_comm_handle exports it (64 bytes = cudaIpcMemHandle_t) for the caller to all-gather by any means
 * (torch.distributed here); r4_comm_open maps every peer's allocation (handles in rank order, world x 64 bytes).
 * After that the SGD steps of an epoch need no host-side collective: r4_ppo_epoch_dist enqueues, per minibatch,
 * the gradient kernel and ONE kernel that reduces the local partials, pushes them into every rank's inbox, waits
 * for the peers' flags, sums in rank order and applies Adam (replicas stay bit-identical).  Every rank must call
 * it with the same n, mb and hyper-parameters.  mb = minibatch size PER RANK; the loss is the mean over
 * mb x world samples (RLlib: sgd_minibatch_size is the total over devices). */
typedef struct r4_comm r4_comm;
int r4_comm_create(int rank, int world, int n_params, r4_comm** out);
int r4_comm_handle(r4_comm* comm, void* handle_out_64);
int r4_comm_open(r4_comm* comm, const void* handles, int n_handles);
void r4_comm_destroy(r4_comm* comm);
int r4_ppo_epoch_dist(r4_comm* comm, float* params, const float* obs, const uint8_t* mask, const int64_t* action,
                      const float* old_logp, const float* old_logits, const float* old_value, const float* adv,
                      const float* target, const int64_t* perm, int n, int mb, int action_size, float clip,
                      float vf_clip, float vf_coeff, float kl_coeff, float ent_coeff, float* scratch, float* flat_grad,
                      float* stats_accum, float* m, float* v, int step0, float lr, float beta1, float beta2, float eps,
                      void* stream);
/* The exchange alone: partial gradients of ONE r4_policy_grad-style launch (scratch, G as there; the caller ran the
 * gradient kernel through r4_policy_grad_partial) -> flat_grad = sum over ranks (A2C: global-norm clipping and Adam
 * follow through r4_adam_step). */
int r4_policy_grad_partial(int mode, const float* params, const float* obs, const uint8_t* mask, const int64_t* action,
                           const float* old_logp, const float* old_logits, const float* old_value, const float* adv,
                           const float* target, const int64_t* idx, int n, int action_size, float clip, float vf_clip,
                           float vf_coeff, float kl_coeff, float ent_coeff, float inv_n, float* scratch, int G,
                           void* stream);
int r4_grad_exchange(r4_comm* comm, const float* scratch, int G, int action_size, float* flat_grad, float* stats_accum,
                     float stat_scale, void* stream);
/* r4_grad_exchange for a flat gradient of any length (the communicator's n_params): partial = f32 [G][n_params] followed by
 * the statistics f32 [G][5]; flat_grad = the sum over the ranks, stats_accum += this rank's statistics * stat_scale. */
int r4_grad_exchange_n(r4_comm* comm, const float* partial, int G, int n_params, float* flat_grad, float* stats_accum,
                       float stat_scale, void* stream);

/* ---- Gaussian policy + learner of the continuous-action env (PPO_conti / A2C_conti, modelfree_train.py:46-48,218-247,
 * 270-290): RLlib's default FullyConnectedNetwork (fcnet_hiddens [256,256], tanh, vf_share_layers off) over obs f32[n,256],
 * a DiagGaussian over action_dim = D (even, 2..64) dimensions.  Flat parameter layout (r4_gauss_num_params(D) floats):
 * fc_1 w[256,256] b[256] | fc_2 w[256,256] b[256] | fc_out w[256,2D] b[2D] (mean | log_std) |
 * fc_value_1 w[256,256] b[256] | fc_value_2 w[256,256] b[256] | value_out w[256] b[1].  Stateless, caller-owned DEVICE memory. */
int r4_gauss_num_params(int action_dim);
/* floats of the scratch that r4_gauss_grad / r4_gauss_ppo_epoch* need (any n: samples are processed in chunks); -1 for a
 * bad action_dim */
int64_t r4_gauss_scratch_size(int action_dim);
/* forward + StochasticSampling (explore != 0: a = mean + exp(log_std) * N(0,1), counter-based noise keyed by seed, counter +
 * row and dimension) or the mean (RLlib explore=False; modelfree_train.py:412-414) -> action f32[n,D] (unclipped: what the
 * sample batch stores and logp is taken on), env_action f32[n,D] = clip(action, -1, 1) (clip_actions), logp f32[n], value
 * f32[n], dist_inputs f32[n,2D] (mean | log_std; may be NULL). */
int r4_gauss_act(const float* params, const float* obs, int n, int action_dim, int explore, uint64_t seed, uint64_t counter,
                 float* action, float* env_action, float* logp, float* value, float* dist_inputs, void* stream);
/* Gradient of the RLlib loss over samples idx[0..n) (NULL = 0..n-1) of a rollout, as r4_policy_grad but deterministic without
 * per-CTA partials (one CTA owns each tile of every weight gradient): mode 0 PPO surrogate over the DiagGaussian (mean; needs
 * old_logp, old_dist = the stored dist inputs f32[n,2D], old_value), mode 1 A2C (sums; old_* may be NULL).  flat_grad
 * f32[num_params] receives the gradient; stats_accum f32[5] (may be NULL) += {policy_loss, vf_loss, kl, entropy, total} *
 * stat_scale.  scratch: r4_gauss_scratch_size(D) floats. */
int r4_gauss_grad(int mode, const float* params, const float* obs, const float* action, const float* old_logp,
                  const float* old_dist, const float* old_value, const float* adv, const float* target, const int64_t* idx,
                  int n, int action_dim, float clip, float vf_clip, float vf_coeff, float kl_coeff, float ent_coeff,
                  float inv_n, float* scratch, float* flat_grad, float* stats_accum, float stat_scale, void* stream);
/* One PPO SGD epoch of the Gaussian policy on a single GPU, as r4_ppo_epoch: per full minibatch perm[s .. s+mb),
 * r4_gauss_grad (mode 0, mean over mb) then r4_adam_step (grad_clip <= 0: off).  Returns the steps done or a negative
 * r4_status. */
int r4_gauss_ppo_epoch(float* params, const float* obs, const float* action, const float* old_logp, const float* old_dist,
                       const float* old_value, const float* adv, const float* target, const int64_t* perm, int n, int mb,
                       int action_dim, float clip, float vf_clip, float vf_coeff, float kl_coeff, float ent_coeff,
                       float* scratch, float* flat_grad, float* stats_accum, float* m, float* v, int step0, float lr,
                       float beta1, float beta2, float eps, float grad_clip, float* norm_scratch, void* stream);
/* The data-parallel epoch of the Gaussian policy, as r4_ppo_epoch_dist (mb = minibatch PER RANK, loss = mean over
 * mb x world samples): per minibatch the gradient launches and ONE exchange + Adam kernel over peer memory.  The
 * communicator must have been created with r4_gauss_num_params(action_dim). */
int r4_gauss_ppo_epoch_dist(r4_comm* comm, float* params, const float* obs, const float* action, const float* old_logp,
                            const float* old_dist, const float* old_value, const float* adv, const float* target,
                            const int64_t* perm, int n, int mb, int action_dim, float clip, float vf_clip, float vf_coeff,
                            float kl_coeff, float ent_coeff, float* scratch, float* flat_grad, float* stats_accum, float* m,
                            float* v, int step0, float lr, float beta1, float beta2, float eps, void* stream);

/* ---- DDPG / TD3 on the continuous-action env (modelfree_train.py:46-48,79-105; modelfree_trainer.py:25-28; RLlib 1.5
 * ddpg / td3 defaults, INTEGRATION.md section 3): a deterministic actor obs(256) -> 400 relu -> 300 relu -> D, squashed
 * to Box(-1, 1) as tanh, and a critic concat(obs, a) -> 400 relu -> 300 relu -> 1 (TD3: plus a twin critic), action_dim
 * = D in 2..32.  Flat parameter layout (r4_ddpg_num_params(D, twin) floats):
 * actor  w1[256,400] b1[400] w2[400,300] b2[300] w3[300,D] b3[D] |
 * critic w1[256+D,400] b1[400] w2[400,300] b2[300] w3[300] b3[1] | twin critic as the critic (twin != 0 only).
 * The target parameters have the same layout.  Stateless: every pointer is caller-owned DEVICE memory. */
int r4_ddpg_num_params(int action_dim, int twin);
/* floats of the scratch r4_ddpg_grad / r4_ddpg_train_step need for batches of up to n samples; -1 for bad arguments */
int64_t r4_ddpg_scratch_size(int action_dim, int twin, int n);
/* The actor on obs f32[n,256] -> action f32[n,D], the env action and what the replay stores.  mode 0: the actor output
 * (DDPG's StochasticSampling over a deterministic distribution, and explore=False).  mode 1: OrnsteinUhlenbeckNoise with ONE
 * state f32[D] shared by every row: x' = x + theta (-x) + sigma N(0, I), a = clip(actor + noise_scale x', -1, 1), where the
 * caller passes noise_scale = scale * ou_base_scale * (high - low); ou_out receives x' (ou_out != ou_in: alternate two
 * buffers).  mode 2: the random phase, a = U(-1, 1) per row and dimension.  The draws are counter-based: splitmix64 keyed by
 * seed and ((counter + row) << 6) + dim (row 0 for the OU state), so the same seed and counter reproduce the actions. */
int r4_ddpg_act(const float* params, const float* obs, int n, int action_dim, int mode, uint64_t seed, uint64_t counter,
                const float* ou_in, float* ou_out, float ou_theta, float ou_sigma, float noise_scale, float* action,
                void* stream);
/* Replay (RLlib ReplayBuffer / PrioritizedReplayBuffer): a ring of `capacity` transitions in caller-owned arrays obs
 * f32[C,256], action f32[C,D], reward f32[C], new_obs f32[C,256], done u8[C] and, for prioritized replay, prio f32[C] (the
 * stored p^alpha) with max_prio f32[1] (the running maximum of |td| + eps, initially 1).
 * r4_replay_store: the [T,B] rollout rows r = t*B + b (obs f32[T*B,256], action f32[T*B,D], reward f32[T*B], done u8[T*B])
 * go to slot (pos + r) % capacity, pos = transitions stored before; new_obs = the obs of row r + B, or final_obs f32[B,256]
 * (what the last step returned) on the last step.  New items get max_prio^alpha (prio may be NULL: uniform replay). */
int r4_replay_store(float* r_obs, float* r_action, float* r_reward, float* r_new_obs, uint8_t* r_done, float* r_prio,
                    const float* max_prio, int capacity, int action_dim, int64_t pos, float alpha, const float* obs,
                    const float* final_obs, const float* action, const float* reward, const uint8_t* done, int T, int B,
                    void* stream);
/* n indices over the first `size` slots from the caller's uniforms u f32[n] in [0, 1): prio == NULL uniform, idx =
 * floor(u size), weight 1; else proportional with replacement, idx = the first i whose prefix sum of prio exceeds u * total
 * (float64 sums in a fixed order), weight = (p_i N)^-beta / (p_min N)^-beta with p = prio / total, N = size. */
int r4_replay_sample(const float* prio, int size, int n, float beta, const float* u, int64_t* idx, float* weights, void* stream);
/* prio[idx[i]] = (|td[i]| + eps)^alpha, the later position winning for a repeated index (RLlib's sequential loop), and
 * max_prio = max(max_prio, |td[i]| + eps). */
int r4_replay_update_priorities(float* prio, float* max_prio, const int64_t* idx, const float* td, int n, float alpha,
                                float eps, void* stream);
/* Gradient of the DDPG / TD3 losses over the replay rows idx[0..n) (weights f32[n] may be NULL = 1):
 * critic loss sum_i w_i (td1_i^2 + td2_i^2) / 2 * inv_n, td_k = Q_k(s, a) - (r + gamma (1 - done) min_k Q'_k(s', a')),
 * a' = clip(pi'(s') + clip(target_noise smooth_noise, -noise_clip, noise_clip), -1, 1) (smooth_noise f32[n,D] N(0,1)
 * draws, NULL: a' = pi'(s')); actor loss -sum_i Q1(s_i, pi(s_i)) * inv_n, applied to the actor weights only.  No l2 terms
 * (r4_ddpg_apply adds them).  grad f32[num_params] receives the gradient (deterministic: one writer per element), td f32[n]
 * (may be NULL) td1, stats f32[3] (may be NULL) {critic loss, actor loss, mean Q1(s, pi(s))}.  2 launches. */
int r4_ddpg_grad(const float* params, const float* target, int action_dim, int twin, const float* r_obs, const float* r_action,
                 const float* r_reward, const float* r_new_obs, const uint8_t* r_done, const int64_t* idx, const float* weights,
                 const float* smooth_noise, int n, float gamma, float target_noise, float noise_clip, float inv_n,
                 float* scratch, float* grad, float* td, float* stats, void* stream);
/* The optimiser step of both networks in one launch: g = grad * grad_scale + l2_reg * w on the kernels (not the biases);
 * torch.optim.Adam (betas 0.9 / 0.999, eps 1e-8) with one moment pair m, v f32[num_params] split by region: the actor with
 * actor_lr at 1-based actor_step (0: the actor is left unchanged, TD3's delayed steps), the critic(s) with critic_lr at
 * critic_step; then the soft target update target = tau params + (1 - tau) target over the whole buffer. */
int r4_ddpg_apply(float* params, float* target, const float* grad, float* m, float* v, int action_dim, int twin, int actor_step,
                  int critic_step, float actor_lr, float critic_lr, float l2_reg, float tau, float grad_scale, void* stream);
/* One SGD step with no host round trip: r4_replay_sample (n indices from u), r4_ddpg_grad, over peer memory the sum over the
 * ranks (comm != NULL; loss = mean over n x world samples; comm created with r4_ddpg_num_params), r4_ddpg_apply and, with
 * prio != NULL, r4_replay_update_priorities from td1.  stats (may be NULL) as r4_ddpg_grad.  5 launches. */
int r4_ddpg_train_step(r4_comm* comm, float* params, float* target, float* m, float* v, int action_dim, int twin,
                       const float* r_obs, const float* r_action, const float* r_reward, const float* r_new_obs,
                       const uint8_t* r_done, float* r_prio, float* max_prio, int size, int n, const float* u,
                       const float* smooth_noise, float beta, float alpha, float prio_eps, float gamma, float target_noise,
                       float noise_clip, int actor_step, int critic_step, float actor_lr, float critic_lr, float l2_reg,
                       float tau, float* scratch, float* stats, void* stream);

/* ---- RAINBOW on the discrete env (modelfree_train.py:50-51,146-178; RLlib 1.5 DQN defaults with num_atoms 8, v_min 0,
 * v_max 1000, n_step 3, noisy off, INTEGRATION.md section 3): the plain obs(256) -> 256 tanh -> 256 tanh trunk, an
 * advantage stream -> 128 relu -> A x atoms and a state-score stream -> 128 relu -> atoms, combined as
 * logits[a][k] = score[k] + adv[a][k] - mean_a adv[a][k]; Q(s, a) = sum_k z_k softmax(logits[a])_k with
 * z_k = v_min + k (v_max - v_min) / (atoms - 1).  A = num_actions in 2..512, atoms in 2..32, A x atoms <= 4096.
 * Flat parameter layout (r4_rainbow_num_params(A, atoms) floats; 491 496 at A = 284, atoms = 8):
 * trunk     w1[256,256] b1[256] w2[256,256] b2[256] |
 * advantage aw1[256,128] ab1[128] aw2[128,A*atoms] ab2[A*atoms] |
 * score     sw1[256,128] sb1[128] sw2[128,atoms] sb2[atoms].
 * The target parameters have the same layout.  Stateless: every pointer is caller-owned DEVICE memory. */
int r4_rainbow_num_params(int num_actions, int num_atoms);
/* floats of the scratch r4_rainbow_grad / r4_rainbow_train_step need for batches of up to n samples; -1 for bad arguments */
int64_t r4_rainbow_scratch_size(int num_actions, int num_atoms, int n);
/* The network on obs f32[n,256] -> action i32[n] and, when q != NULL, Q f32[n,A].  explore 0: the first argmax of Q.
 * explore 1: SoftQ (temperature 1), a ~ softmax(Q) by inverse CDF over one uniform per row, the top 24 bits of splitmix64
 * keyed by seed and (counter + row) << 6, so the same seed and counter reproduce the actions. */
int r4_rainbow_act(const float* params, const float* obs, int n, int num_actions, int num_atoms, float v_min, float v_max,
                   int explore, uint64_t seed, uint64_t counter, int32_t* action, float* q, void* stream);
/* The replay store of r4_replay_store with integer actions (action ring i32[C], rollout action i32[T*B]) and RLlib's
 * n-step fold per episode: row t keeps sum_{j < n_step, t + j < T} gamma^j reward[t + j] (the original rewards, added in j
 * order), and the new_obs and done of row min(t + n_step - 1, T - 1).  n_step = 1 stores the rows as they are. */
int r4_replay_store_nstep(float* r_obs, int32_t* r_action, float* r_reward, float* r_new_obs, uint8_t* r_done, float* r_prio,
                          const float* max_prio, int capacity, int64_t pos, float alpha, int n_step, float gamma,
                          const float* obs, const float* final_obs, const int32_t* action, const float* reward,
                          const uint8_t* done, int T, int B, void* stream);
/* Gradient of the distributional loss over the replay rows idx[0..n) (weights f32[n] may be NULL = 1): a* = argmax of the
 * online Q(s', .), p' = the target net's distribution at (s', a*), m = its projection of clip(r + gamma_n (1 - done) z,
 * v_min, v_max) onto the support (RLlib's QLoss, gamma_n = gamma^n_step), td = -sum_k m_k log p(s, a)_k, loss =
 * sum_i w_i td_i * inv_n.  grad f32[num_params] receives the gradient (deterministic: one writer per element), td f32[n]
 * (may be NULL) the td errors, stats f32[3] (may be NULL) {loss, mean td, mean Q(s, a)}, each sum times inv_n.  2 launches. */
int r4_rainbow_grad(const float* params, const float* target, int num_actions, int num_atoms, float v_min, float v_max,
                    const float* r_obs, const int32_t* r_action, const float* r_reward, const float* r_new_obs,
                    const uint8_t* r_done, const int64_t* idx, const float* weights, int n, float gamma_n, float inv_n,
                    float* scratch, float* grad, float* td, float* stats, void* stream);
/* The optimiser step in one launch: each of the 12 tensors' gradient scaled by grad_clip / ||g|| where its norm exceeds
 * grad_clip (per tensor, RLlib's minimize_and_clip; grad_clip <= 0: off), torch.optim.Adam (betas 0.9 / 0.999, eps
 * adam_eps) at the 1-based step, then target = params when copy_target != 0 (the hard target update). */
int r4_rainbow_apply(float* params, float* target, const float* grad, float* m, float* v, int num_actions, int num_atoms,
                     int step, float lr, float adam_eps, float grad_clip, int copy_target, void* stream);
/* One SGD step with no host round trip: r4_replay_sample (n indices from u), r4_rainbow_grad, over peer memory the sum over
 * the ranks (comm != NULL; loss = mean over n x world samples; comm created with r4_rainbow_num_params), r4_rainbow_apply
 * and, with prio != NULL, r4_replay_update_priorities from td.  stats (may be NULL) as r4_rainbow_grad.  5 launches. */
int r4_rainbow_train_step(r4_comm* comm, float* params, float* target, float* m, float* v, int num_actions, int num_atoms,
                          float v_min, float v_max, const float* r_obs, const int32_t* r_action, const float* r_reward,
                          const float* r_new_obs, const uint8_t* r_done, float* r_prio, float* max_prio, int size, int n,
                          const float* u, float beta, float alpha, float prio_eps, float gamma_n, int step, float lr,
                          float adam_eps, float grad_clip, int copy_target, float* scratch, float* stats, void* stream);

/* ---- the simulator alone (nets/dien.py:8-45), for parity tests and kernel benchmarks ------- */
/* seq i32[R,2,64], dense f32[R,432], cat i32[R,21] (device) -> obs f32[R,256], probs f32[R,2]
 * (either may be NULL).  Runs the uncached path: GRU-1 is recomputed for every row. */
int r4_dien_forward(r4_env* env, const int32_t* seq, const float* dense, const int32_t* cat,
                    int n_rows, float* obs, float* probs, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RL4RS_B200_H */
