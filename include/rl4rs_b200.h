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
  float*   click_p;      /* f32 [B,R]     probs[:,1] of the reward pass (slate.py:298-301), R = 9 (SeqSlate) or
                                          max_steps (Slate) rows per env; written only on steps that compute a reward */
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
 * items: i32[B]; emb (conti mode, may be NULL): f64[B,emb_dim]; reward: f64[B].
 * An env longer than its log rows (n_slots of r4_load_log) has no logged slot to give where the reference raises:
 * r4_offline_action returns R4_ERR_STATE at cur_steps >= n_slots while cur_steps < max_steps (the record split's
 * IndexError, slate.py:156), r4_offline_reward at a SeqSlate page end cur_steps > n_slots (the (B, 9) x (B, 0)
 * broadcast, seqslate.py:77-85).  At cur_steps == max_steps offline_action is item 0, and the Slate offline_reward after
 * the last step sums every logged slot, whatever max_steps is. */
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
/* -1 for an action_size outside 2..512 */
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
/* -1 for a bad action_dim */
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

/* ---- IMPALA (modelfree_train.py:345-390; RLlib 1.5 vtrace_torch_policy.py) over either policy ----------------------------
 * A rollout is B complete episodes of T steps (1..81), time-major: element [t * B + b] of every f32 [T, B] buffer; done at
 * T - 1 only.  Stateless, caller-owned DEVICE memory. */
/* The forward at stored actions (no sampling): obs f32[n,256], mask u8[n,A], action i64[n] -> logp f32[n] of the action
 * under params, value f32[n].  Equal, bit for bit, to what r4_policy_act wrote for its own sample on the same params. */
int r4_policy_eval(const float* params, const float* obs, const uint8_t* mask, const int64_t* action, int n, int action_size,
                   float* logp, float* value, void* stream);
/* The same for the Gaussian policy: action f32[n,D] (the unclipped sample r4_gauss_act stored). */
int r4_gauss_eval(const float* params, const float* obs, const float* action, int n, int action_dim, float* logp, float* value,
                  void* stream);
/* V-trace (vtrace.from_importance_weights), one thread per episode: rho = exp(target_logp - behaviour_logp), c = min(1, rho),
 * vs_t - V_t = min(rho_bar, rho_t) (r_t + g_t V_{t+1} - V_t) + g_t c_t (vs_{t+1} - V_{t+1}),
 * pg_adv_t = min(rho_pg_bar, rho_t) (r_t + g_t vs_{t+1} - V_t), g_t = gamma (0 at t = T - 1).  drop_last != 0 (RLlib 1.5): steps
 * 0..T-2 with the bootstrap V(s_{T-1}) = value[T-1], and vs[T-1] = value[T-1], pg_adv[T-1] = 0; drop_last = 0: every step,
 * bootstrap 0.  T 2..81 with drop_last, gamma in [0, 1], thresholds > 0.  Deterministic. */
int r4_vtrace(const float* behaviour_logp, const float* target_logp, const float* value, const float* reward, int T, int B,
              float gamma, float rho_bar, float rho_pg_bar, int drop_last, float* vs, float* pg_adv, void* stream);
/* One IMPALA learner step of the mask policy, with no host round trip: r4_policy_eval over all T * B rows (-> logp, value),
 * r4_vtrace (behaviour_logp = the logp r4_policy_act stored; -> vs, pg_adv), the A2C-mode gradient of r4_policy_grad with
 * adv = pg_adv and target = vs over the kept rows (the first T - 1 time steps with drop_last, else all), the exchange over
 * peer memory (comm; NULL = one GPU: the loss is summed over the global batch), the global-norm clip (grad_clip <= 0: off;
 * norm_scratch f32[1]; the norm is summed in a fixed order) and Adam (step is 1-based).  logits = the stored masked logits
 * (the KL statistic).  scratch: f32[G * (num_params + 5)], G = min(ceil(kept rows / 4), the device's SM count).
 * stats_accum f32[5] += the sums {policy_loss, vf_loss, kl, entropy, total}. */
int r4_impala_step(r4_comm* comm, float* params, const float* obs, const uint8_t* mask, const int64_t* action,
                   const float* behaviour_logp, const float* logits, const float* reward, int T, int B, int action_size,
                   float gamma, float rho_bar, float rho_pg_bar, int drop_last, float vf_coeff, float ent_coeff, float* logp,
                   float* value, float* vs, float* pg_adv, float* scratch, float* flat_grad, float* stats_accum, float* m,
                   float* v, int step, float lr, float beta1, float beta2, float eps, float grad_clip, float* norm_scratch,
                   void* stream);
/* r4_impala_step for the Gaussian policy over r4_gauss_eval and r4_gauss_grad (mode 1); scratch: r4_gauss_scratch_size(D)
 * floats; kl is reported as 0. */
int r4_gauss_impala_step(r4_comm* comm, float* params, const float* obs, const float* action, const float* behaviour_logp,
                         const float* reward, int T, int B, int action_dim, float gamma, float rho_bar, float rho_pg_bar,
                         int drop_last, float vf_coeff, float ent_coeff, float* logp, float* value, float* vs, float* pg_adv,
                         float* scratch, float* flat_grad, float* stats_accum, float* m, float* v, int step, float lr,
                         float beta1, float beta2, float eps, float grad_clip, float* norm_scratch, void* stream);

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

/* ---- batch RL on the logged dataset (batchrl_trainer.py:34-90; d3rlpy 0.91 DiscreteBC / DiscreteBCQ / DiscreteCQL as the
 * reference configures them, INTEGRATION.md section 3).  algo 0 BC, 1 BCQ, 2 CQL; obs_dim K in 11..4096 (the d3rl
 * observation: simulator obs | 9 prev actions | cur_steps), A = action_size in 2..512, with the shared planes within
 * 226 KB (every K at A = 284; K <= 2998 at A = 512).  Flat parameter layout:
 * masked net  w1[K,256] b1[256] emb[A,32] w2[576,A] b2[A] w3[A,A] b3[A]   (the custom encoder with_q + d3rlpy's head)
 * plain net   w1[K,256] b1[256] w2[256,256] b2[256] w3[256,A] b3[A]      (d3rlpy's default encoder + head)
 * BC: masked (imitator); BCQ: masked (Q) | masked (imitator); CQL: plain.  The target holds the Q part only
 * (r4_batchrl_target_size floats: 0 for BC).  Stateless: every pointer is caller-owned DEVICE memory. */
typedef struct {
  const float* obs;            /* f32[N, K] */
  const int32_t* action;       /* i32[N] */
  const float* reward;         /* f32[N] */
  const uint8_t* terminal;     /* u8[N] */
  const int64_t* transitions;  /* i64[T] from r4_batchrl_transitions */
  const uint8_t* location_mask;/* u8[3, A]: 1 where the page layer allows the item */
  const uint8_t* special;      /* u8[A]: 1 for the special items */
} r4_batchrl_data;
typedef struct {
  float gamma;                 /* discount */
  float beta;                  /* the imitator's penalty beta * mean(z^2) (BC 0 in the script, BCQ 0.5) */
  float alpha;                 /* CQL's conservative weight */
  float log_flex;              /* log(action_flexibility) of BCQ (log 0.3) */
  float reward_mean, reward_den;   /* CQL's reward scaler r' = (r - mean) / den (0, 1: off) */
} r4_batchrl_hyper;
int r4_batchrl_num_params(int algo, int obs_dim, int action_size);
int r4_batchrl_target_size(int algo, int obs_dim, int action_size);
/* floats of the scratch r4_batchrl_grad / r4_batchrl_epoch need for minibatches of up to n samples; -1 for bad arguments */
int64_t r4_batchrl_scratch_size(int algo, int obs_dim, int action_size, int n);
/* index i64[N] receives, in order, every entry i with terminal[i] == 0 that lies before the last terminal entry (the first
 * entry of each transition (obs[i], action[i], reward[i + 1], obs[i + 1], terminal[i + 1]) of d3rlpy's episodes, split at
 * the terminals); count i64[1] (device) receives how many.  1 launch. */
int r4_batchrl_transitions(const uint8_t* terminal, int64_t N, int64_t* index, int64_t* count, void* stream);
/* The gradient of the algorithm's loss (the minibatch mean) over the transitions data->transitions[idx[0..n)] -> grad
 * f32[num_params] (deterministic: one writer per element) and stats f32[3] (may be NULL): {loss, td or nll term, Q(s, a)
 * or the imitator's mean z^2}, each a minibatch mean.  3 launches. */
int r4_batchrl_grad(int algo, int obs_dim, int action_size, const float* params, const float* target,
                    const r4_batchrl_data* data, const r4_batchrl_hyper* hp, const int64_t* idx, int n, float* scratch,
                    float* grad, float* stats, void* stream);
/* torch.optim.Adam (betas 0.9 / 0.999, no clipping) at the 1-based step, then target = the Q part of params when
 * copy_target != 0.  1 launch. */
int r4_batchrl_apply(int algo, int obs_dim, int action_size, float* params, float* target, const float* grad, float* m,
                     float* v, int step, float lr, float adam_eps, int copy_target, void* stream);
/* One epoch of d3rlpy's RoundIterator with no host round trip: minibatch k is perm[k mb .. (k + 1) mb) for k < n_perm / mb
 * (the last partial minibatch dropped); each runs r4_batchrl_grad and r4_batchrl_apply at step step0 + k + 1, copying the
 * target after the steps whose 0-based index is a multiple of target_interval (target_interval <= 0: never).  stats
 * (may be NULL) receives f32[steps, 3].  Chained by programmatic dependent launch.  Returns the number of steps, or an
 * r4_status. */
int r4_batchrl_epoch(int algo, int obs_dim, int action_size, float* params, float* target, float* m, float* v,
                     const r4_batchrl_data* data, const r4_batchrl_hyper* hp, const int64_t* perm, int64_t n_perm, int mb,
                     int step0, float lr, float adam_eps, int target_interval, float* scratch, float* stats, void* stream);
/* kernels launched so far by the r4_batchrl_* entry points in this process (for launch-count measurements) */
int64_t r4_batchrl_launch_count(void);
/* The act rule on n observations (obs_f64 != 0: f64[n, K], as the env's 'torch' output; else f32[n, K]) -> action
 * i32[n].  mode 0: rl4rs policy_model.predict_with_mask (action_probs = BC's log-probs or softmax(Q), -2^15 where the
 * location layer cur_steps % 9 / 3, the 9 prev actions or, when one of them is special, the special items rule an item
 * out, the first argmax); mode 1: d3rlpy's predict (BC argmax log-prob, BCQ the imitator-filtered argmax of Q, CQL argmax Q).
 * probs f32[n, A] (may be NULL) receives action_probs, values f32[n, A] (may be NULL) the raw output (BC logits, else Q).
 * Only data->location_mask and data->special are read.  1 launch. */
int r4_batchrl_act(int algo, int obs_dim, int action_size, const float* params, const void* obs, int obs_f64, int n,
                   const r4_batchrl_data* data, int mode, float log_flex, int32_t* action, float* probs, float* values,
                   void* stream);

/* ---- continuous-action CQL on the logged dataset (batchrl_trainer.py:61-73, 91-107 'CQL-conti'; d3rlpy 0.91 CQL as the
 * script configures it, INTEGRATION.md section 3).  obs_dim K in 1..4096, action_dim D in 1..512, minibatch n in 1..4096,
 * n_action_samples S in 1..64.  Flat parameter layout (H = 256):
 * actor     w1[K,H] b1[H] w2[H,H] b2[H] w3[H,2D] b3[2D]   (output [mu | logstd], logstd clamped to [-20, 2], tanh squash)
 * critic k  w1[K+D,H] b1[H] w2[H,H] b2[H] w3[H,1] b3[1]   (k = 0, 1; input [obs | action])
 * then log_temp, log_alpha.  The target (r4_cqlc_target_size floats) is [critic 0 | critic 1].  The noise of a step is
 * counter-based, keyed by (seed, step, stream, row, sample, dim) (csrc/r4_cqlconti.cuh); every pointer is caller-owned
 * DEVICE memory.  The kernels count in r4_batchrl_launch_count. */
typedef struct {
  const float* obs;            /* f32[N, K] */
  const float* action;         /* f32[N, D] */
  const float* reward;         /* f32[N] */
  const uint8_t* terminal;     /* u8[N] */
  const int64_t* transitions;  /* i64[T] from r4_batchrl_transitions */
} r4_cqlc_data;
typedef struct {
  float gamma, tau;            /* discount, soft target update rate */
  float lr_actor, lr_critic, lr_temp, lr_alpha, adam_eps;   /* torch.optim.Adam per group, betas 0.9 / 0.999 */
  float alpha_threshold, conservative_weight;
  float reward_mean, reward_den;   /* the reward scaler r' = (r - mean) / den (0, 1: off) */
  int n_action_samples;        /* S */
  uint64_t seed;               /* the noise seed */
} r4_cqlc_hyper;
int r4_cqlc_num_params(int obs_dim, int action_dim);
int r4_cqlc_target_size(int obs_dim, int action_dim);
/* floats of the scratch r4_cqlc_grad / r4_cqlc_epoch need for minibatches of up to n; -1 for bad arguments */
int64_t r4_cqlc_scratch_size(int obs_dim, int action_dim, int n_action_samples, int n);
/* floats of the scratch r4_cqlc_act needs for n rows; -1 for bad arguments */
int64_t r4_cqlc_act_scratch_size(int obs_dim, int action_dim, int n);
/* The gradients of the four losses of one step (temperature, alpha, critic, actor) at the given parameters, with the noise
 * of step `step` (>= 1), over the transitions data->transitions[idx[0..n)] -> grad f32[num_params] (each group's part from
 * its own loss; deterministic) and stats f32[5] (may be NULL): {critic loss, actor loss, temperature loss, alpha loss,
 * mean Q_0(s, a)}.  Nothing is updated.  54 launches. */
int r4_cqlc_grad(int obs_dim, int action_dim, const float* params, const float* target, const r4_cqlc_data* data,
                 const r4_cqlc_hyper* hp, const int64_t* idx, int n, int step, float* scratch, float* grad, float* stats,
                 void* stream);
/* One epoch of d3rlpy's RoundIterator with no host round trip: minibatch k is perm[k mb .. (k + 1) mb) for k < n_perm / mb;
 * each is one SGD step at step step0 + k + 1: temperature, alpha, critic and actor updates in that order (each phase sees
 * the parameters the earlier ones left), Adam per group, the soft target update after the critic's Adam.  stats (may be
 * NULL) receives f32[steps, 5].  56 launches per step.  Returns the number of steps, or an r4_status. */
int r4_cqlc_epoch(int obs_dim, int action_dim, float* params, float* target, float* m, float* v, const r4_cqlc_data* data,
                  const r4_cqlc_hyper* hp, const int64_t* perm, int64_t n_perm, int mb, int step0, float* scratch,
                  float* stats, void* stream);
/* predict on n observations (n <= 2^20; obs_f64 != 0: f64[n, K], as the env's 'torch' output; else f32[n, K]): action f32[n, D]
 * (may be NULL) = tanh(mu); q f32[n] (may be NULL) = the mean of the two critics at (obs, action_in) (action_in f32[n, D],
 * or NULL for the predicted action).  At least one of action, q.  5 launches (12 with q). */
int r4_cqlc_act(int obs_dim, int action_dim, const float* params, const void* obs, int obs_f64, int n,
                const float* action_in, float* action, float* q, float* scratch, void* stream);

/* ---- continuous-action BCQ on the logged dataset (batchrl_trainer.py:61-73, 91-107 'BCQ-conti'; d3rlpy 0.91 BCQ as the
 * script configures it, INTEGRATION.md section 3).  obs_dim K in 1..4096, action_dim D in 1..512, latent_size L in 1..512,
 * minibatch n in 1..4096, n_action_samples S in 1..256 (n S <= 2^20 for r4_bcqc_act).  Flat parameter layout (H = 256;
 * each net w1[in,H] b1[H] w2[H,H] b2[H] w3[H,out] b3[out]): actor (K+D -> D; pi = clamp(a + flex tanh(f), -1, 1)) |
 * critic 0 (K+D -> 1) | critic 1 | VAE encoder (K+D -> [mu | logstd] 2L, logstd clamped to [-20, 2]) | VAE decoder
 * (K+L -> D, tanh).  The target (r4_bcqc_target_size floats) is [actor | critic 0 | critic 1], the first floats of the
 * layout.  The data is r4_cqlc_data; the kernels count in r4_batchrl_launch_count. */
typedef struct {
  float gamma, tau;            /* discount, soft target update rate */
  float lr_actor, lr_critic, lr_imitator, adam_eps;   /* torch.optim.Adam per group, betas 0.9 / 0.999 */
  float lam;                   /* the target's mix lam min_k + (1 - lam) max_k */
  float beta;                  /* the VAE's KL weight */
  float action_flexibility;    /* the actor's residual scale */
  float reward_mean, reward_den;   /* the reward scaler r' = (r - mean) / den (0, 1: off) */
  int n_action_samples;        /* S */
  int latent_size;             /* L */
  uint64_t seed;               /* the noise seed */
} r4_bcqc_hyper;
int r4_bcqc_num_params(int obs_dim, int action_dim, int latent_size);
int r4_bcqc_target_size(int obs_dim, int action_dim, int latent_size);
/* floats of the scratch r4_bcqc_grad / r4_bcqc_epoch need for minibatches of up to n; -1 for bad arguments */
int64_t r4_bcqc_scratch_size(int obs_dim, int action_dim, int latent_size, int n_action_samples, int n);
/* floats of the scratch r4_bcqc_act needs for n rows; -1 for bad arguments */
int64_t r4_bcqc_act_scratch_size(int obs_dim, int action_dim, int latent_size, int n_action_samples, int n);
/* The gradients of the three losses of one step (imitator, critic, actor) at the given parameters, with the noise of step
 * `step` (>= 1), over data->transitions[idx[0..n)] -> grad f32[num_params] (each group's part from its own loss) and stats
 * f32[5] (may be NULL): {imitator loss, critic loss, actor loss, mean Q_0(s, a), VAE reconstruction mse}.  Nothing is
 * updated.  66 launches. */
int r4_bcqc_grad(int obs_dim, int action_dim, const float* params, const float* target, const r4_cqlc_data* data,
                 const r4_bcqc_hyper* hp, const int64_t* idx, int n, int step, float* scratch, float* grad, float* stats,
                 void* stream);
/* One epoch of d3rlpy's RoundIterator with no host round trip (as r4_cqlc_epoch): each minibatch is one SGD step at step
 * step0 + k + 1: imitator, critic and actor updates in that order, Adam per group, the soft target update of the critics
 * after their Adam and of the actor after its Adam.  stats (may be NULL) receives f32[steps, 5].  69 launches per step.
 * Returns the number of steps, or an r4_status. */
int r4_bcqc_epoch(int obs_dim, int action_dim, float* params, float* target, float* m, float* v, const r4_cqlc_data* data,
                  const r4_bcqc_hyper* hp, const int64_t* perm, int64_t n_perm, int mb, int step0, float* scratch,
                  float* stats, void* stream);
/* predict on n observations (obs_f64 != 0: f64[n, K], else f32[n, K]): action f32[n, D] (may be NULL) = the candidate with
 * the largest Q_0 among S decoded, perturbed actions (latent draws keyed by (hp->seed, counter)); q f32[n] (may be NULL)
 * = the mean of the two critics at (obs, action_in), or at the predicted action when action_in is NULL.  Needs action, or
 * q with action_in.  13 launches for the action, 8 for q. */
int r4_bcqc_act(int obs_dim, int action_dim, const float* params, const void* obs, int obs_f64, int n,
                const r4_bcqc_hyper* hp, uint64_t counter, const float* action_in, float* action, float* q, float* scratch,
                void* stream);

/* ---- the simulator alone (nets/dien.py:8-45), for parity tests and kernel benchmarks ------- */
/* seq i32[R,2,64], dense f32[R,432], cat i32[R,21] (device) -> obs f32[R,256], probs f32[R,2]
 * (either may be NULL).  Runs the uncached path: GRU-1 is recomputed for every row. */
int r4_dien_forward(r4_env* env, const int32_t* seq, const float* dense, const int32_t* cat,
                    int n_rows, float* obs, float* probs, void* stream);

/* ---- training the DIEN simulator (nets/dien.py:8-45 in training mode, supervised_train.py <train> <test> <model> dien 0) on
 * item samples: sample i of the per-record store is (record i / 9, exposed item i % 9) (data_preprocess.py:91-131,
 * INTEGRATION.md section 8).  emb_size 128, hidden_units 128, maxlen 64, 432 dense and 21 category features, seq_num 2;
 * hash_size H = category_hash_size in 1..4000000.  Flat parameter layout (tf_checkpoint.dien_layer_plan order, row-major):
 *   emb_cat[H,128] dense_w1[432,128] dense_b1[128] dense_w2[128,128] dense_b2[128] emb_seq[H,128]
 *   then for sequence i = 0, 1: gru_wg[256,256] gru_bg[256] gru_wc[256,128] gru_bc[128] att_w1[512,64] att_b1[64]
 *     att_w2[64,16] att_b2[16] att_k[16,1] att_b[1] augru_wg[384,512] augru_bg[512] augru_wc[384,256] augru_bc[256]
 *   obs_w[3456,256] obs_b[256] rew_w[256,2] rew_b[2]
 * Stateless: every pointer is caller-owned DEVICE memory.  Every id must lie in [0, H) (checked where the store is built). */
typedef struct {
  const int32_t* user_cat;     /* i32[N, 10] portrait ids */
  const float* user_dense;     /* f32[N, 32] portrait dense features */
  const int32_t* sequence_id;  /* i32[N] */
  const int32_t* items;        /* i32[N, 9] exposed items */
  const uint8_t* feedback;     /* u8[N, 9] labels */
  const float* item_feature;   /* f32[N, 360] the record's item features (9 x 40) */
  const int32_t* seq;          /* i32[N, 2, 64] user_seqfeature | the earlier pages' items, pre-padded / pre-truncated */
} r4_simtrain_data;
/* floats of the flat parameters (27 413 956 at H = 100000); -1 for H out of range */
int64_t r4_simtrain_num_params(int hash_size);
/* BYTES of the scratch r4_simtrain_grad / _step / _eval need for n samples (n in 1..4096); -1 out of range */
int64_t r4_simtrain_scratch_size(int n);
/* The gradient of the loss (Keras binary_crossentropy of the softmax output on one_hot(label, 2), p clipped to
 * [1e-7, 1 - 1e-7], mean over both columns and the n samples idx[0..n)) -> grad f32[num_params].  The embedding tables of
 * grad must be zero on entry (r4_simtrain_apply leaves them so); only the rows the samples touch are written.  Dropout on
 * the two dense-tower outputs: keep_in (may be NULL) u8[n, 256] (layer-major, 1 = kept), else a unit is kept when the
 * counter-based draw of (seed, counter, sample, unit) is >= drop_rate; kept units are scaled by 1 / (1 - drop_rate).
 * keep_out (may be NULL) receives the bits used.  stats (may be NULL) f32[2] = {mean loss, mean binary accuracy};
 * acc (may be NULL) f64[405] accumulates {loss sum, accuracy sum, samples, positives[201], negatives[201]}, where bin b counts
 * the probabilities above exactly b of Keras's 200 AUC thresholds (both one-hot columns).  Deterministic. */
int r4_simtrain_grad(int hash_size, const float* params, const r4_simtrain_data* data, const int64_t* idx, int n, uint64_t seed,
                     uint64_t counter, float drop_rate, const uint8_t* keep_in, uint8_t* keep_out, void* scratch, float* grad,
                     float* stats, double* acc, void* stream);
/* Keras Adam over every parameter at the 1-based step: m += (g - m)(1 - beta1), v += (g^2 - v)(1 - beta2),
 * p -= lr sqrt(1 - beta2^step) / (1 - beta1^step) m / (sqrt(v) + eps).  Clears the embedding rows of grad.  1 launch. */
int r4_simtrain_apply(int hash_size, float* params, float* grad, float* m, float* v, int step, float lr, float beta1, float beta2,
                      float eps, void* stream);
/* r4_simtrain_grad (keep bits drawn) then r4_simtrain_apply, with no host round trip. */
int r4_simtrain_step(int hash_size, float* params, float* grad, float* m, float* v, const r4_simtrain_data* data,
                     const int64_t* idx, int n, uint64_t seed, uint64_t counter, float drop_rate, int step, float lr, float beta1,
                     float beta2, float eps, void* scratch, float* stats, double* acc, void* stream);
/* The forward without dropout -> probs f32[n, 2] (may be NULL); acc (may be NULL) accumulates as in r4_simtrain_grad. */
int r4_simtrain_eval(int hash_size, const float* params, const r4_simtrain_data* data, const int64_t* idx, int n, void* scratch,
                     float* probs, double* acc, void* stream);
/* ---- the slate-label heads on the same backbone (nets/dien_slate.py, nets/dien_slate_multiclass.py; supervised_train.py
 * <train> <test> <model> dien_slate[_multiclass] 1).  head selects simulator_reward's width C and the loss:
 *   R4_SIMHEAD_ITEM (C = 2): the r4_simtrain_* entry points above.
 *   R4_SIMHEAD_SLATE (C = 9): sigmoid output against the page's 9 clicks; binary cross-entropy from the logits (no clip),
 *     mean over the 9 columns and the n samples.  acc f64[408] = the 405 of the item head (accuracy: binary accuracy at
 *     0.5 per column; histograms over all 9 columns) then {TP, FP, FN} at p > 0.5.
 *   R4_SIMHEAD_SLATE_MULTICLASS (C = 22): softmax output against the class sum_j y_j [1,2,4,1,2,4,1,2,4]_j; categorical
 *     cross-entropy from the logits, mean over the n samples.  acc f64[3] = {loss sum, hits (first argmax == class), samples}.
 * For the slate heads idx holds RECORD indices: sample s is record idx[s] (data_preprocess.py tfrecord_slate): cat = portrait
 * ids + [sequence_id] + the 9 items + the pad id 0, dense = portrait dense + item features + 40 zeros.  The flat layout is the
 * item head's with rew_w [256, C], rew_b [C]; scratch_size depends on the head.  Each entry point has the signature of its
 * r4_simtrain_* namesake with head first; probs is f32[n, C].  Bad head, hash_size or n: -1 or R4_ERR_ARG, nothing written.
 * Each r4_simtrain_head_* is r4_simtrain_net_* below with net R4_SIM_DIEN, and each r4_simtrain_* is r4_simtrain_head_*
 * with head R4_SIMHEAD_ITEM: one implementation, one argument check and the same results, launches and scratch layout. */
enum { R4_SIMHEAD_ITEM = 0, R4_SIMHEAD_SLATE = 1, R4_SIMHEAD_SLATE_MULTICLASS = 2 };
int64_t r4_simtrain_head_num_params(int head, int hash_size);
int64_t r4_simtrain_head_scratch_size(int head, int n);
int r4_simtrain_head_grad(int head, int hash_size, const float* params, const r4_simtrain_data* data, const int64_t* idx, int n,
                          uint64_t seed, uint64_t counter, float drop_rate, const uint8_t* keep_in, uint8_t* keep_out,
                          void* scratch, float* grad, float* stats, double* acc, void* stream);
int r4_simtrain_head_apply(int head, int hash_size, float* params, float* grad, float* m, float* v, int step, float lr,
                           float beta1, float beta2, float eps, void* stream);
int r4_simtrain_head_step(int head, int hash_size, float* params, float* grad, float* m, float* v, const r4_simtrain_data* data,
                          const int64_t* idx, int n, uint64_t seed, uint64_t counter, float drop_rate, int step, float lr,
                          float beta1, float beta2, float eps, void* scratch, float* stats, double* acc, void* stream);
int r4_simtrain_head_eval(int head, int hash_size, const float* params, const r4_simtrain_data* data, const int64_t* idx, int n,
                          void* scratch, float* probs, double* acc, void* stream);
/* ---- the other backbones and adversarial_slate (nets/dnn*.py, widedeep*.py, lstm*.py, adversarial_slate.py).  net is
 * an R4_SIM_* value or R4_SIMNET_ADVERSARIAL_SLATE; nets 0..3 take heads 0..2, net 4 only R4_SIMHEAD_ADVERSARIAL.  Each entry
 * point takes the arguments of its r4_simtrain_head_* namesake after net; net R4_SIM_DIEN is the DIEN net above.  A bad
 * pair, hash_size, n, drop_rate or step, or a NULL pointer: -1 or R4_ERR_ARG ("bad argument"), nothing written.  The samples, keep bits, dropout, heads, acc layouts and Adam are
 * the DIEN heads' (R4_SIMHEAD_ADVERSARIAL: the R4_SIMHEAD_SLATE acc layout, f64[408]).  The flat layouts, with H =
 * hash_size, E = U = 128 and C the head's width (2, 9, 22; adversarial 9), in tf_checkpoint.*_layer_plan order:
 *   dnn       emb_cat[H,E] dense_w1[432,128] dense_b1 dense_w2[128,128] dense_b2 fc_w[256,256] fc_b obs_w[256,256] obs_b
 *             rew_w[256,C] rew_b[C]                                  (dnn.py's second Embedding feeds nothing: not held)
 *   widedeep  emb_cat dense_w1 dense_b1 dense_w2 dense_b2 emb_seq[H,E] fc_w[256,256] fc_b rew_w[3072,C] rew_b[C]
 *   lstm      emb_cat cgru_k[128,384] cgru_rk[128,384] cgru_b[384] dense_w1 dense_b1 dense_w2 dense_b2 emb_seq
 *             sgru0_k sgru0_rk sgru0_b sgru1_k sgru1_rk sgru1_b obs_w[3200,256] obs_b rew_w[256,C] rew_b[C]
 *   adversarial_slate  emb_cat dense_w1 dense_b1 dense_w2 dense_b2 emb_seq w[512,9] b[9]
 * The lstm GRUs are Keras-v1 GRUs (hard sigmoid, reset_after = False, gates [z | r | h]; its slope is taken as 0.2 at both
 * kinks).  adversarial_slate's loss per record: 0.1 mean_j BCE(y_j, sigmoid(z_j)) + sum_j softmax(sigmoid(z))_j (1 - y_j).
 * Launches per step (grad + apply; the radix sort counted once): dnn 18, widedeep 17, lstm 34, adversarial_slate 14; eval:
 * dnn 7, widedeep 6, lstm 12, adversarial_slate 5. */
enum { R4_SIMNET_ADVERSARIAL_SLATE = 4 };
enum { R4_SIMHEAD_ADVERSARIAL = 3 };
int64_t r4_simtrain_net_num_params(int net, int head, int hash_size);
int64_t r4_simtrain_net_scratch_size(int net, int head, int n);
int r4_simtrain_net_grad(int net, int head, int hash_size, const float* params, const r4_simtrain_data* data, const int64_t* idx,
                         int n, uint64_t seed, uint64_t counter, float drop_rate, const uint8_t* keep_in, uint8_t* keep_out,
                         void* scratch, float* grad, float* stats, double* acc, void* stream);
int r4_simtrain_net_apply(int net, int head, int hash_size, float* params, float* grad, float* m, float* v, int step, float lr,
                          float beta1, float beta2, float eps, void* stream);
int r4_simtrain_net_step(int net, int head, int hash_size, float* params, float* grad, float* m, float* v,
                         const r4_simtrain_data* data, const int64_t* idx, int n, uint64_t seed, uint64_t counter, float drop_rate,
                         int step, float lr, float beta1, float beta2, float eps, void* scratch, float* stats, double* acc,
                         void* stream);
int r4_simtrain_net_eval(int net, int head, int hash_size, const float* params, const r4_simtrain_data* data, const int64_t* idx,
                         int n, void* scratch, float* probs, double* acc, void* stream);
/* kernels launched so far by the r4_simtrain_* entry points in this process (the radix sort counted once) */
int64_t r4_simtrain_launch_count(void);
/* ---- Exact-K (nets/exact_k/model.py, script/exact_k_train.py): the pointer-network slate generator and its reward
 * critic.  Every pointer is device memory; the work runs on stream.  fp32 row-major; one writer per output element, so
 * results are deterministic.
 *
 * Generator (R4_EXACTK_GENERATOR), hidden_units 64 (D = 128), 4 heads, 2 blocks, one glimpse, one LSTM layer, res_length 9.
 * Flat parameters, in this order (kernels [in, out]):
 *   u_w[256,64] u_b[64] emb[500,64]
 *   per block 0, 1: qkv_w[128,384] (Q | K | V columns) qkv_b[384] ln1_beta[128] ln1_gamma[128] ff1_w[128,256] ff1_b[256]
 *                   ff2_w[256,128] ff2_b[128] ln2_beta[128] ln2_gamma[128]
 *   lstm_w[256,512] (rows: input | h; columns: gates i | j | f | o) lstm_b[512] c0[128] x0[128] (first input) h0[128]
 *   intra: W_b[128,128] v_dec[128] W_bef[128,128] bias_dec[128]
 *   glimpse_0, then attention (the pointer), each: W_q[128,128] W_dec[128,128] v[128] bias[128] W_ref[128,128]
 * Critic (R4_EXACTK_CRITIC): w1[256,128] b1 w2[128,128] b2 w3[128,128] b3 w4[128,1] b4[1]; relu on the three hidden layers.
 *
 * user: f32[n, 256]; n in 1..4096; seq_length T in 9..500 (the candidates are the item ids 0..T-1).  masks: u8[4, T], rows
 * the location masks of positions 0-2, 3-5 and 6-8 and the special items; the point mask of position t is its location
 * mask, minus the items already chosen, minus every special item once one is chosen (position 0: its location mask).
 * Masked logits are -2^32 + 1.  dropout (the rate, in [0, 1)) is live on the encoder input and both blocks' attention
 * probabilities; keep draws and the SAMPLE draws are U[0, 1) = (top 24 bits of a splitmix64 hash of (seed, call, stream,
 * element)) / 2^24 (see r4_exactk.cuh: draw24), kept when U >= dropout.  SAMPLE picks the first candidate whose running
 * sum of exp(logit / temperature - max) reaches (U + 2^-25) times their total. */
enum { R4_EXACTK_GENERATOR = 0, R4_EXACTK_CRITIC = 1 };
enum { R4_EXACTK_SAMPLE = 0, R4_EXACTK_GREEDY = 1, R4_EXACTK_TRAIN = 2 };
/* parameter count of net; -1 for another net */
int64_t r4_exactk_num_params(int net);
/* BYTES of scratch the generator (net 0) or the critic (net 1, seq_length ignored) needs for n rows; -1 out of range */
int64_t r4_exactk_scratch_size(int net, int n, int seq_length);
/* The encoder and the nine decode steps: path i32[n, 9] (TRAIN: the teacher path on entry) and logits f32[n, 9, T] (may be
 * NULL).  122 launches. */
int r4_exactk_decode(const float* params, const float* user, int n, int seq_length, const uint8_t* masks, int mode,
                     float temperature, uint64_t seed, uint64_t call, float dropout, int32_t* path, float* logits, void* scratch,
                     void* stream);
/* The teacher-forced forward on target i32[n, 9] and the gradient of mean_b(sum_t CE(logits[b, t], target[b, t]) reward[b])
 * into grad f32[num_params] (overwritten); loss f32[1] (may be NULL).  349 launches (348 without loss).
 * Targets (and the TRAIN path of r4_exactk_decode) are candidate indices in [0, T); an entry outside is clamped into it.
 * After r4_exactk_decode or r4_exactk_grad the scratch begins with the encoder's activations, f32 planes in this order,
 * each starting at a multiple of 64 floats: relu(user W_u + b_u) [n,64], X0 [n,T,128], then per block 0, 1: the key /
 * query mask [n,T], relu(X W_qkv + b_qkv) [n,T,384], softmax [n,4,T,T], dropped probabilities [n,4,T,T], attention output
 * [n,T,128], Y1 [n,T,128], its normalised input [n,T,128], 1 / std [n,T], relu(Y1 W_1 + b_1) [n,T,256], Y2 [n,T,128], its
 * normalised input [n,T,128], 1 / std [n,T]. */
int r4_exactk_grad(const float* params, const float* user, int n, int seq_length, const uint8_t* masks, const int32_t* target,
                   const float* reward, uint64_t seed, uint64_t call, float dropout, float* grad, float* loss, void* scratch,
                   void* stream);
/* The critic: pred f32[n] (may be NULL); with target f32[n], also loss = sum_b (target - pred)^2 (f32[1], may be NULL) and
 * its gradient into grad (overwritten).  5 launches without target, 27 with. */
int r4_exactk_critic(const float* params, const float* user, int n, const float* target, float* pred, float* grad, float* loss,
                     void* scratch, void* stream);
/* TF1 AdamOptimizer step `step` (1-based) of net: m, v, params updated in place.  1 launch. */
int r4_exactk_adam(int net, float* params, float* grad, float* m, float* v, int step, float lr, float beta1, float beta2,
                   float eps, void* stream);
/* kernels launched so far by the r4_exactk_* entry points in this process */
int64_t r4_exactk_launch_count(void);
/* ---- The MDP checker's seq2seq transformer (keras-transformer 0.40's get_model, rl4rs_b200/mdpchecker) ----
 * Every call is asynchronous on `stream`; pointers other than cfg are DEVICE memory; results are deterministic.
 * Config: src_tokens / tgt_tokens in 4..65536 (equal when use_same_embed), embed_dim E a multiple of 32 up to 512,
 * head_num dividing E, hidden_dim F a multiple of 32 up to 1024, encoder_num / decoder_num in 1..6.
 * Flat parameters, in this order (kernels [in, out]):
 *   the encoder token table [src_tokens, E], then the decoder's [tgt_tokens, E] unless use_same_embed
 *   per encoder block: self-attention Wq[E,E] bq[E] Wk bk Wv bv Wo bo, its LayerNorm gamma[E] beta[E],
 *                      FeedForward W1[E,F] b1[F] W2[F,E] b2[E], its LayerNorm gamma beta
 *   per decoder block: self-attention (as above), LayerNorm, query attention (as above), LayerNorm, FeedForward, LayerNorm
 *   the output bias [tgt_tokens]
 * Tokens are int32; 0 is PAD (masked as a key, and out of the loss as a decoder input); tokens outside the table are
 * clamped into it.  Sequence lengths are 1..64.  Dropout (rate in [0, 1)) follows each sub-layer before its residual add;
 * its keep draws are Exact-K's (r4_exactk.cuh: draw24) on the key (seed, call * 32 + sub-layer, 0, row * E + column), the
 * sub-layers numbered encoder blocks first (2 each), then decoder blocks (3 each). */
typedef struct {
  int32_t src_tokens, tgt_tokens, embed_dim, head_num, hidden_dim, encoder_num, decoder_num, use_same_embed;
} r4_s2s_config;
enum { R4_S2S_TRAIN = 0, R4_S2S_PREDICT = 1, R4_S2S_SEARCH = 2, R4_S2S_STEP = 3 };
/* parameter count; -1 for a config out of range */
int64_t r4_s2s_num_params(const r4_s2s_config* cfg);
/* BYTES of scratch for one call of `mode` over n source rows of length src_len: TRAIN (r4_s2s_grad, and r4_s2s_epoch at
 * n = its batch), PREDICT (r4_s2s_predict, r4_s2s_score: tgt_len decoder positions of `beam` paths per row),
 * SEARCH (r4_s2s_beam_search: tgt_len = target_len, k = candidates), STEP (r4_s2s_decode_step: k = its k); -1 out of
 * range.  Grid limits: n * beam * head_num <= 65535. */
int64_t r4_s2s_scratch_size(const r4_s2s_config* cfg, int mode, int n, int src_len, int tgt_len, int beam, int k);
/* The loss sum(mask ce) / sum(mask) of keras 2.2.5's sparse categorical cross-entropy (probabilities clipped to
 * [1e-7, 1 - 1e-7]) on enc i32[n, src_len], dec / target i32[n, tgt_len], and its gradient into grad f32[num_params]
 * (overwritten); loss f32[1] may be NULL. */
int r4_s2s_grad(const r4_s2s_config* cfg, const float* params, const int32_t* enc, const int32_t* dec, const int32_t* target,
                int n, int src_len, int tgt_len, uint64_t seed, uint64_t call, float dropout, float* grad, float* loss,
                void* scratch, void* stream);
/* After r4_s2s_grad over (n, src_len, tgt_len), its scratch holds each FeedForward's relu(x W1 + b1), f32[n * len,
 * hidden_dim], encoder blocks first, then decoder blocks: their BYTE offsets into offsets[encoder_num + decoder_num].
 * Returns the count, or -1 out of range. */
int r4_s2s_relu_offsets(const r4_s2s_config* cfg, int n, int src_len, int tgt_len, int64_t* offsets);
/* keras 2.2.5 Adam step `step` (1-based) over every parameter: m, v, params updated in place.  1 launch. */
int r4_s2s_apply(const r4_s2s_config* cfg, float* params, const float* grad, float* m, float* v, int step, float lr,
                 float beta1, float beta2, float eps, void* stream);
/* One epoch: for each minibatch k of `batch` rows of perm i64[n_perm] (the last one partial), gather its rows of the
 * N-row arrays enc / dec / target, r4_s2s_grad with call = call0 + k, and Adam step step0 + k + 1; losses f32[steps]. */
int r4_s2s_epoch(const r4_s2s_config* cfg, float* params, float* grad, float* m, float* v, const int32_t* enc,
                 const int32_t* dec, const int32_t* target, int64_t N, int src_len, int tgt_len, const int64_t* perm,
                 int64_t n_perm, int batch, int step0, uint64_t seed, uint64_t call0, float dropout, float lr, float beta1,
                 float beta2, float eps, float* losses, void* scratch, void* stream);
/* Softmax probabilities f32[n, tgt_len, tgt_tokens] of the decoder on enc i32[n, src_len] and dec i32[n, tgt_len]. */
int r4_s2s_predict(const r4_s2s_config* cfg, const float* params, const int32_t* enc, const int32_t* dec, int n, int src_len,
                   int tgt_len, float* probs, void* scratch, void* stream);
/* The k most probable next tokens after dec i32[n, tgt_len] (times the candidate mask of cand i32[n, n_cand] when cand is
 * not NULL), by probability descending, ties to the lower token: val f64[n, k], idx i32[n, k].  1 <= k < tgt_tokens. */
int r4_s2s_decode_step(const r4_s2s_config* cfg, const float* params, const int32_t* enc, int n, int src_len,
                       const int32_t* dec, int tgt_len, const int32_t* cand, int n_cand, int k, double* val, int32_t* idx,
                       void* scratch, void* stream);
/* rl4rs/mdpchecker/decoder.py's beam_search: paths i32[n, beam, target_len + 1] (START = 1 first) and their products of
 * probabilities f64[n, beam].  Step 1 takes the top beam; with n_cand > 0 the later steps keep only the n_cand best tokens
 * of step 1 (the reference's candidates); each later step takes the top beam of the beam^2 products, ties to the lower
 * (beam, token) flat index.  beam in 1..256, < tgt_tokens; n_cand < tgt_tokens, at most 8192; target_len 1..63. */
int r4_s2s_beam_search(const r4_s2s_config* cfg, const float* params, const int32_t* enc, int n, int src_len, int beam,
                       int target_len, int n_cand, int32_t* path, double* score, void* scratch, void* stream);
/* Experiment I's scores: prob f32[n, beam, target_len], entry i the probability the decoder gives path[., ., i + 1] after
 * the prefix path[., ., :i + 1] (one causal pass over each path). */
int r4_s2s_score(const r4_s2s_config* cfg, const float* params, const int32_t* enc, int n, int src_len, const int32_t* path,
                 int beam, int target_len, float* prob, void* scratch, void* stream);
/* kernels launched so far by the r4_s2s_* entry points in this process */
int64_t r4_s2s_launch_count(void);

/* ---- Off-policy evaluation (script/offline_evaluation.py's `ope` stage, rl4rs_b200/offline_evaluation.py) ----
 * Every call is asynchronous on `stream`; pointers are caller-owned DEVICE memory; results are deterministic.
 * The logged-policy (behaviour) net is nets/dnn.py's graph at 50 dense features and C classes (149 <= C <= 65536), with
 * flat parameters in this order (kernels [in, out]): emb_cat [H, 128], dense_w1 [50, 128], dense_b1 [128],
 * dense_w2 [128, 128], dense_b2 [128], fc_w [256, 256], fc_b [256], obs_w [256, 256], obs_b [256], rew_w [256, C],
 * rew_b [C].  1 <= H <= 2^24, 1 <= B <= 2^21. */
/* parameter count; -1 out of range */
int64_t r4_ope_num_params(int H, int C);
/* FLOATS of scratch for one r4_ope_behavior call over B rows; -1 out of range */
int64_t r4_ope_behavior_scratch_size(int B, int C);
/* The behaviour probabilities of page `page` (0 <= page < P) of B records: the page's category ids -- head i32[B, 11]
 * (user_protrait[:10], sequence_id), then items i32[B, P * K] at [page K, page K + K), post-padded with 0 to 21; ids
 * outside [0, H) are clamped into the table -- and its dense row, feat f32[B, P * 5K] at [page 5K, page 5K + 5K),
 * post-padded with 0 to 50 (1 <= K <= 10).  y = softmax of the net; out f32[B, C - 1] column c - 1 = y[c] divided by the
 * sum of its slice: y[1:40], y[40:148] or y[148:C] (sums in f64).  7 launches. */
int r4_ope_behavior(int B, int H, int C, int K, int P, int page, const float* params, const int32_t* head,
                    const int32_t* items, const float* feat, float* out, float* scratch, void* stream);
/* Step t (0 <= t < T) of an evaluation episode: column t of the [T, B] buffers.  1 launch.
 *   pol f32  the policy's probability of the offline action off i32[B]: probs f32[B, A] (logits 0) or the softmax of the
 *            logits f32[B, A] (logits 1; the sum in f64);
 *   beh f32  the behaviour probability of the offline action: block f32[B, C - 1] (r4_ope_behavior's page) at layer
 *            (>= 1) with behavior_model.action_probs' slice and clip (layer 1, 2, any other);
 *   val f32  values f32[B, A] at own i32[B] (per_action 1), or values f32[B] (per_action 0; own may be NULL);
 *   rew f64  reward f64[B];  offr f64  off_reward f64[B].
 * 2 <= A <= 65536, A <= C.  A device-side action outside [0, A) writes NaN into the columns that index with it. */
int r4_ope_step(int t, int T, int B, int A, int C, int layer, const float* probs, int logits, const int32_t* off,
                const float* block, const int32_t* own, const float* values, int per_action, const double* reward,
                const double* off_reward, float* pol, float* beh, float* val, double* rew, double* offr, void* stream);
/* kernels launched so far by the r4_ope_* entry points in this process */
int64_t r4_ope_launch_count(void);

/* kernels launched so far by every learner entry point in this process (r4_policy_*, r4_gae, r4_adam_step, r4_ppo_epoch*,
 * r4_grad_exchange*, r4_gauss_*, r4_vtrace, r4_impala_step, r4_ddpg_*, r4_replay_*, r4_rainbow_*, r4_batchrl_*,
 * r4_simtrain_*, r4_exactk_*, r4_s2s_*, r4_ope_*): the sum of the batch RL, simulator-trainer, Exact-K, seq2seq and OPE
 * counts above and the online learners'. */
int64_t r4_learner_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* RL4RS_B200_H */
