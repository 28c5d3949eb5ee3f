"""ctypes binding of librl4rs_b200.so (include/rl4rs_b200.h).  Thin: no compute here.

The library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).  There is NO CPU
fallback: if the shared object is missing or cannot be loaded the import of any env class fails
with the reason; if it loads but no CUDA device is present, creating an env fails.
"""
import ctypes as C
import os

import torch

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "librl4rs_b200.so")

FLAG_RLLIB_MASK, FLAG_D3RL_MASK, FLAG_CONTI, FLAG_ONEHOT, FLAG_RAWSTATE, FLAG_INFO_FETCH = 1, 2, 4, 8, 16, 32
ENV_SLATE, ENV_SEQSLATE = 0, 1
SIM_DIEN, SIM_DNN, SIM_WIDEDEEP, SIM_LSTM = 0, 1, 2, 3
SIMULATORS = {"dien": SIM_DIEN, "dnn": SIM_DNN, "widedeep": SIM_WIDEDEEP, "lstm": SIM_LSTM}


class R4Config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "env_kind", "flags", "batch_size", "max_steps", "page_items", "action_size", "action_emb_size",
        "maxlen", "seq_num", "dense_feature_num", "category_feature_num", "category_hash_size",
        "emb_size", "hidden_units", "max_rows_per_pass", "simulator")]


class R4Out(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "obs", "action_mask", "reward", "done", "chosen", "cat", "dense", "seq", "click_p",
        "masked_actions")]


class BatchRLData(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("obs", "action", "reward", "terminal", "transitions", "location_mask", "special")]


class SimTrainData(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("user_cat", "user_dense", "sequence_id", "items", "feedback", "item_feature", "seq")]


class BatchRLHyper(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("gamma", "beta", "alpha", "log_flex", "reward_mean", "reward_den")]


class CQLContiData(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("obs", "action", "reward", "terminal", "transitions")]


class CQLContiHyper(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("gamma", "tau", "lr_actor", "lr_critic", "lr_temp", "lr_alpha", "adam_eps",
                                         "alpha_threshold", "conservative_weight", "reward_mean", "reward_den")] + \
        [("n_action_samples", C.c_int), ("seed", C.c_uint64)]


class BCQContiHyper(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("gamma", "tau", "lr_actor", "lr_critic", "lr_imitator", "adam_eps", "lam", "beta",
                                         "action_flexibility", "reward_mean", "reward_den")] + \
        [("n_action_samples", C.c_int), ("latent_size", C.c_int), ("seed", C.c_uint64)]


EXPORTS = {
    # name: (restype, argtypes)
    "r4_create": (C.c_int, [C.POINTER(R4Config), C.c_int, C.POINTER(C.c_void_p)]),
    "r4_destroy": (None, [C.c_void_p]),
    "r4_last_error": (C.c_char_p, [C.c_void_p]),
    "r4_load_items": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "r4_load_weight": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int]),
    "r4_finalize_weights": (C.c_int, [C.c_void_p, C.c_void_p]),
    "r4_load_log": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int]),
    "r4_reset": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(R4Out), C.c_void_p]),
    "r4_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(R4Out), C.c_void_p]),
    "r4_offline_action": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r4_offline_reward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "r4_violation": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "r4_features": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r4_nearest_neighbor": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "r4_cur_steps": (C.c_int, [C.c_void_p]),
    "r4_prev_actions": (C.c_void_p, [C.c_void_p]),
    "r4_copy_prev_actions": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "r4_launch_count": (C.c_int64, [C.c_void_p]),
    "r4_profile": (C.c_int, [C.c_void_p, C.c_int]),
    "r4_profile_read": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_double),
                                  C.POINTER(C.c_int64), C.POINTER(C.c_double)]),
    "r4_abi_version": (C.c_int, []),
    "r4_obs_dim": (C.c_int, [C.c_int]),
    "r4_augru_kernel_for": (C.c_int, [C.c_int, C.c_int]),
    "r4_set_option": (C.c_int, [C.c_char_p, C.c_int]),
    "r4_policy_num_params": (C.c_int, [C.c_int]),
    "r4_policy_act": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_uint64,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r4_policy_grad": (C.c_int, [C.c_int] + [C.c_void_p] * 10 + [C.c_int, C.c_int] + [C.c_float] * 6 +
                       [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p]),
    "r4_ppo_epoch": (C.c_int, [C.c_void_p] * 10 + [C.c_int] * 3 + [C.c_float] * 5 + [C.c_void_p] * 5 + [C.c_int] +
                     [C.c_float] * 5 + [C.c_void_p, C.c_void_p]),
    "r4_gae": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r4_comm_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "r4_comm_handle": (C.c_int, [C.c_void_p, C.c_void_p]),
    "r4_comm_open": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    "r4_comm_destroy": (None, [C.c_void_p]),
    "r4_ppo_epoch_dist": (C.c_int, [C.c_void_p] * 11 + [C.c_int] * 3 + [C.c_float] * 5 + [C.c_void_p] * 5 + [C.c_int] +
                          [C.c_float] * 4 + [C.c_void_p]),
    "r4_policy_grad_partial": (C.c_int, [C.c_int] + [C.c_void_p] * 10 + [C.c_int, C.c_int] + [C.c_float] * 6 +
                               [C.c_void_p, C.c_int, C.c_void_p]),
    "r4_grad_exchange": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p]),
    "r4_grad_exchange_n": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p]),
    "r4_gauss_num_params": (C.c_int, [C.c_int]),
    "r4_gauss_scratch_size": (C.c_int64, [C.c_int]),
    "r4_gauss_act": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_uint64] + [C.c_void_p] * 6),
    "r4_gauss_grad": (C.c_int, [C.c_int] + [C.c_void_p] * 9 + [C.c_int, C.c_int] + [C.c_float] * 6 +
                      [C.c_void_p] * 3 + [C.c_float, C.c_void_p]),
    "r4_gauss_ppo_epoch": (C.c_int, [C.c_void_p] * 9 + [C.c_int] * 3 + [C.c_float] * 5 + [C.c_void_p] * 5 + [C.c_int] +
                           [C.c_float] * 5 + [C.c_void_p, C.c_void_p]),
    "r4_gauss_ppo_epoch_dist": (C.c_int, [C.c_void_p] * 10 + [C.c_int] * 3 + [C.c_float] * 5 + [C.c_void_p] * 5 + [C.c_int] +
                                [C.c_float] * 4 + [C.c_void_p]),
    "r4_policy_eval": (C.c_int, [C.c_void_p] * 4 + [C.c_int, C.c_int] + [C.c_void_p] * 3),
    "r4_gauss_eval": (C.c_int, [C.c_void_p] * 3 + [C.c_int, C.c_int] + [C.c_void_p] * 3),
    "r4_vtrace": (C.c_int, [C.c_void_p] * 4 + [C.c_int, C.c_int] + [C.c_float] * 3 + [C.c_int] + [C.c_void_p] * 3),
    "r4_impala_step": (C.c_int, [C.c_void_p] * 8 + [C.c_int] * 3 + [C.c_float] * 3 + [C.c_int] + [C.c_float] * 2 +
                       [C.c_void_p] * 9 + [C.c_int] + [C.c_float] * 5 + [C.c_void_p] * 2),
    "r4_gauss_impala_step": (C.c_int, [C.c_void_p] * 6 + [C.c_int] * 3 + [C.c_float] * 3 + [C.c_int] + [C.c_float] * 2 +
                             [C.c_void_p] * 9 + [C.c_int] + [C.c_float] * 5 + [C.c_void_p] * 2),
    "r4_ddpg_num_params": (C.c_int, [C.c_int, C.c_int]),
    "r4_ddpg_scratch_size": (C.c_int64, [C.c_int, C.c_int, C.c_int]),
    "r4_ddpg_act": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p] +
                    [C.c_float] * 3 + [C.c_void_p, C.c_void_p]),
    "r4_replay_store": (C.c_int, [C.c_void_p] * 7 + [C.c_int, C.c_int, C.c_int64, C.c_float] + [C.c_void_p] * 5 +
                        [C.c_int, C.c_int, C.c_void_p]),
    "r4_replay_sample": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r4_replay_update_priorities": (C.c_int, [C.c_void_p] * 4 + [C.c_int, C.c_float, C.c_float, C.c_void_p]),
    "r4_ddpg_grad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 8 + [C.c_int] + [C.c_float] * 4 +
                     [C.c_void_p] * 5),
    "r4_ddpg_apply": (C.c_int, [C.c_void_p] * 5 + [C.c_int] * 4 + [C.c_float] * 5 + [C.c_void_p]),
    "r4_ddpg_train_step": (C.c_int, [C.c_void_p] * 5 + [C.c_int, C.c_int] + [C.c_void_p] * 7 + [C.c_int, C.c_int] +
                           [C.c_void_p] * 2 + [C.c_float] * 6 + [C.c_int, C.c_int] + [C.c_float] * 4 + [C.c_void_p] * 3),
    "r4_rainbow_num_params": (C.c_int, [C.c_int, C.c_int]),
    "r4_rainbow_scratch_size": (C.c_int64, [C.c_int, C.c_int, C.c_int]),
    "r4_rainbow_act": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_uint64,
                                 C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r4_replay_store_nstep": (C.c_int, [C.c_void_p] * 7 + [C.c_int, C.c_int64, C.c_float, C.c_int, C.c_float] +
                              [C.c_void_p] * 5 + [C.c_int, C.c_int, C.c_void_p]),
    "r4_rainbow_grad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float] + [C.c_void_p] * 7 +
                        [C.c_int, C.c_float, C.c_float] + [C.c_void_p] * 5),
    "r4_rainbow_apply": (C.c_int, [C.c_void_p] * 5 + [C.c_int] * 3 + [C.c_float] * 3 + [C.c_int, C.c_void_p]),
    "r4_rainbow_train_step": (C.c_int, [C.c_void_p] * 5 + [C.c_int, C.c_int, C.c_float, C.c_float] + [C.c_void_p] * 7 +
                              [C.c_int, C.c_int, C.c_void_p] + [C.c_float] * 4 + [C.c_int, C.c_float, C.c_float, C.c_float,
                                                                                  C.c_int] + [C.c_void_p] * 3),
    "r4_padqn_num_params": (C.c_int, [C.c_int, C.c_int]),
    "r4_padqn_scratch_size": (C.c_int64, [C.c_int, C.c_int, C.c_int]),
    "r4_padqn_cache_size": (C.c_int64, [C.c_int]),
    "r4_padqn_refresh": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r4_padqn_act": (C.c_int, [C.c_void_p] * 4 + [C.c_int] * 4 + [C.c_uint64, C.c_uint64] + [C.c_void_p] * 4),
    "r4_padqn_store": (C.c_int, [C.c_void_p] * 8 + [C.c_int, C.c_int, C.c_int64, C.c_float] + [C.c_void_p] * 7 +
                       [C.c_int, C.c_int, C.c_void_p]),
    "r4_padqn_grad": (C.c_int, [C.c_void_p] * 5 + [C.c_int, C.c_int] + [C.c_void_p] * 8 + [C.c_int, C.c_float, C.c_float] +
                      [C.c_void_p] * 5),
    "r4_padqn_apply": (C.c_int, [C.c_void_p] * 6 + [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int] + [C.c_float] * 3 +
                       [C.c_int, C.c_void_p]),
    "r4_padqn_train_step": (C.c_int, [C.c_void_p] * 7 + [C.c_int, C.c_int] + [C.c_void_p] * 8 + [C.c_int, C.c_int, C.c_void_p] +
                            [C.c_float] * 4 + [C.c_int] + [C.c_float] * 3 + [C.c_int] + [C.c_void_p] * 3),
    "r4_batchrl_num_params": (C.c_int, [C.c_int] * 3),
    "r4_batchrl_target_size": (C.c_int, [C.c_int] * 3),
    "r4_batchrl_scratch_size": (C.c_int64, [C.c_int] * 4),
    "r4_batchrl_transitions": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r4_batchrl_grad": (C.c_int, [C.c_int] * 3 + [C.c_void_p, C.c_void_p, C.POINTER(BatchRLData), C.POINTER(BatchRLHyper),
                                                  C.c_void_p, C.c_int] + [C.c_void_p] * 4),
    "r4_batchrl_apply": (C.c_int, [C.c_int] * 3 + [C.c_void_p] * 5 + [C.c_int, C.c_float, C.c_float, C.c_int, C.c_void_p]),
    "r4_batchrl_epoch": (C.c_int, [C.c_int] * 3 + [C.c_void_p] * 4 + [C.POINTER(BatchRLData), C.POINTER(BatchRLHyper),
                                                                   C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_float,
                                                                   C.c_float, C.c_int] + [C.c_void_p] * 3),
    "r4_batchrl_launch_count": (C.c_int64, []),
    "r4_batchrl_act": (C.c_int, [C.c_int] * 3 + [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(BatchRLData), C.c_int,
                                                  C.c_float] + [C.c_void_p] * 4),
    "r4_cqlc_num_params": (C.c_int, [C.c_int] * 2),
    "r4_cqlc_target_size": (C.c_int, [C.c_int] * 2),
    "r4_cqlc_scratch_size": (C.c_int64, [C.c_int] * 4),
    "r4_cqlc_act_scratch_size": (C.c_int64, [C.c_int] * 3),
    "r4_cqlc_grad": (C.c_int, [C.c_int] * 2 + [C.c_void_p] * 2 + [C.POINTER(CQLContiData), C.POINTER(CQLContiHyper),
                                                                C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 4),
    "r4_cqlc_epoch": (C.c_int, [C.c_int] * 2 + [C.c_void_p] * 4 + [C.POINTER(CQLContiData), C.POINTER(CQLContiHyper),
                                                                 C.c_void_p, C.c_int64, C.c_int, C.c_int] + [C.c_void_p] * 3),
    "r4_cqlc_act": (C.c_int, [C.c_int] * 2 + [C.c_void_p] * 2 + [C.c_int, C.c_int] + [C.c_void_p] * 5),
    "r4_bcqc_num_params": (C.c_int, [C.c_int] * 3),
    "r4_bcqc_target_size": (C.c_int, [C.c_int] * 3),
    "r4_bcqc_scratch_size": (C.c_int64, [C.c_int] * 5),
    "r4_bcqc_act_scratch_size": (C.c_int64, [C.c_int] * 5),
    "r4_bcqc_grad": (C.c_int, [C.c_int] * 2 + [C.c_void_p] * 2 + [C.POINTER(CQLContiData), C.POINTER(BCQContiHyper),
                                                                C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 4),
    "r4_bcqc_epoch": (C.c_int, [C.c_int] * 2 + [C.c_void_p] * 4 + [C.POINTER(CQLContiData), C.POINTER(BCQContiHyper),
                                                                 C.c_void_p, C.c_int64, C.c_int, C.c_int] + [C.c_void_p] * 3),
    "r4_bcqc_act": (C.c_int, [C.c_int] * 2 + [C.c_void_p] * 2 + [C.c_int, C.c_int, C.POINTER(BCQContiHyper), C.c_uint64] +
                    [C.c_void_p] * 5),
    "r4_adam_step": (C.c_int,[C.c_void_p] * 4 + [C.c_int, C.c_int] + [C.c_float] * 6 + [C.c_void_p, C.c_void_p]),
    "r4_dien_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r4_simtrain_num_params": (C.c_int64, [C.c_int]),
    "r4_simtrain_scratch_size": (C.c_int64, [C.c_int]),
    "r4_simtrain_grad": (C.c_int, [C.c_int, C.c_void_p, C.POINTER(SimTrainData), C.c_void_p, C.c_int, C.c_uint64, C.c_uint64,
                                   C.c_float] + [C.c_void_p] * 7),
    "r4_simtrain_apply": (C.c_int, [C.c_int] + [C.c_void_p] * 4 + [C.c_int] + [C.c_float] * 4 + [C.c_void_p]),
    "r4_simtrain_step": (C.c_int, [C.c_int] + [C.c_void_p] * 4 + [C.POINTER(SimTrainData), C.c_void_p, C.c_int, C.c_uint64,
                                                                C.c_uint64, C.c_float, C.c_int] + [C.c_float] * 4 +
                         [C.c_void_p] * 4),
    "r4_simtrain_eval": (C.c_int, [C.c_int, C.c_void_p, C.POINTER(SimTrainData), C.c_void_p, C.c_int] + [C.c_void_p] * 4),
    "r4_simtrain_head_num_params": (C.c_int64, [C.c_int, C.c_int]),
    "r4_simtrain_head_scratch_size": (C.c_int64, [C.c_int, C.c_int]),
    "r4_simtrain_head_grad": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.POINTER(SimTrainData), C.c_void_p, C.c_int, C.c_uint64,
                                        C.c_uint64, C.c_float] + [C.c_void_p] * 7),
    "r4_simtrain_head_apply": (C.c_int, [C.c_int, C.c_int] + [C.c_void_p] * 4 + [C.c_int] + [C.c_float] * 4 + [C.c_void_p]),
    "r4_simtrain_head_step": (C.c_int, [C.c_int, C.c_int] + [C.c_void_p] * 4 + [C.POINTER(SimTrainData), C.c_void_p, C.c_int,
                                                                             C.c_uint64, C.c_uint64, C.c_float, C.c_int] +
                              [C.c_float] * 4 + [C.c_void_p] * 4),
    "r4_simtrain_head_eval": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.POINTER(SimTrainData), C.c_void_p, C.c_int] +
                              [C.c_void_p] * 4),
    "r4_simtrain_net_num_params": (C.c_int64, [C.c_int, C.c_int, C.c_int]),
    "r4_simtrain_net_scratch_size": (C.c_int64, [C.c_int, C.c_int, C.c_int]),
    "r4_simtrain_net_grad": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.POINTER(SimTrainData), C.c_void_p, C.c_int,
                                       C.c_uint64, C.c_uint64, C.c_float] + [C.c_void_p] * 7),
    "r4_simtrain_net_apply": (C.c_int, [C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 4 + [C.c_int] + [C.c_float] * 4 + [C.c_void_p]),
    "r4_simtrain_net_step": (C.c_int, [C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 4 + [C.POINTER(SimTrainData), C.c_void_p,
                                                                                        C.c_int, C.c_uint64, C.c_uint64, C.c_float,
                                                                                        C.c_int] +
                             [C.c_float] * 4 + [C.c_void_p] * 4),
    "r4_simtrain_net_eval": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.POINTER(SimTrainData), C.c_void_p, C.c_int] +
                             [C.c_void_p] * 4),
    "r4_simtrain_launch_count": (C.c_int64, []),
    "r4_learner_launch_count": (C.c_int64, []),
    "r4_exactk_num_params": (C.c_int64, [C.c_int]),
    "r4_exactk_scratch_size": (C.c_int64, [C.c_int, C.c_int, C.c_int]),
    "r4_exactk_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_uint64,
                                   C.c_uint64, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r4_exactk_grad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                 C.c_uint64, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "r4_exactk_critic": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 6),
    "r4_exactk_adam": (C.c_int, [C.c_int] + [C.c_void_p] * 4 + [C.c_int] + [C.c_float] * 4 + [C.c_void_p]),
    "r4_exactk_launch_count": (C.c_int64, []),
    "r4_s2s_num_params": (C.c_int64, [C.c_void_p]),
    "r4_s2s_scratch_size": (C.c_int64, [C.c_void_p] + [C.c_int] * 6),
    "r4_s2s_grad": (C.c_int, [C.c_void_p] * 5 + [C.c_int] * 3 + [C.c_uint64, C.c_uint64, C.c_float] + [C.c_void_p] * 4),
    "r4_s2s_relu_offsets": (C.c_int, [C.c_void_p] + [C.c_int] * 3 + [C.c_void_p]),
    "r4_s2s_apply": (C.c_int, [C.c_void_p] * 5 + [C.c_int] + [C.c_float] * 4 + [C.c_void_p]),
    "r4_s2s_epoch": (C.c_int, [C.c_void_p] * 8 + [C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_int,
                                                  C.c_uint64, C.c_uint64] + [C.c_float] * 5 + [C.c_void_p] * 3),
    "r4_s2s_predict": (C.c_int, [C.c_void_p] * 4 + [C.c_int] * 3 + [C.c_void_p] * 3),
    "r4_s2s_decode_step": (C.c_int, [C.c_void_p] * 3 + [C.c_int] * 2 + [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int] +
                           [C.c_void_p] * 4),
    "r4_s2s_beam_search": (C.c_int, [C.c_void_p] * 3 + [C.c_int] * 5 + [C.c_void_p] * 4),
    "r4_s2s_score": (C.c_int, [C.c_void_p] * 3 + [C.c_int] * 2 + [C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 3),
    "r4_s2s_launch_count": (C.c_int64, []),
    "r4_ope_num_params": (C.c_int64, [C.c_int, C.c_int]),
    "r4_ope_behavior_scratch_size": (C.c_int64, [C.c_int, C.c_int]),
    "r4_ope_behavior": (C.c_int, [C.c_int] * 6 + [C.c_void_p] * 7),
    "r4_ope_step": (C.c_int, [C.c_int] * 6 + [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int] +
                    [C.c_void_p] * 8),
    "r4_ope_launch_count": (C.c_int64, []),
}


class S2SConfig(C.Structure):
    """r4_s2s_config of include/rl4rs_b200.h."""
    _fields_ = [(k, C.c_int32) for k in ("src_tokens", "tgt_tokens", "embed_dim", "head_num", "hidden_dim", "encoder_num",
                                         "decoder_num", "use_same_embed")]


S2S_TRAIN, S2S_PREDICT, S2S_SEARCH, S2S_STEP = 0, 1, 2, 3

_lib = None


class R4Error(RuntimeError):
    pass


def load_library(path=None):
    """Load the shared object and declare every entry point of include/rl4rs_b200.h."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise R4Error("%s is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                      "(there is no CPU fallback)" % path)
    lib = C.CDLL(path)
    for name, (res, args) in EXPORTS.items():
        fn = getattr(lib, name)      # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def ptr(t, byte_offset=0):
    """The device (or host) address of tensor t plus byte_offset as a void* argument; NULL for None."""
    return C.c_void_p(t.data_ptr() + byte_offset) if t is not None else C.c_void_p(0)


def stream(device):
    """The current torch stream of device as the cudaStream_t argument every entry point ends with."""
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def check(lib, handle, rc, what):
    if rc != 0:
        msg = lib.r4_last_error(handle)
        raise R4Error("%s failed (%d): %s" % (what, rc, msg.decode() if msg else "?"))


def set_option(key, value):
    """r4_set_option: process-wide kernel-choice override (parity tests / A-B timing)."""
    lib = load_library()
    check(lib, None, lib.r4_set_option(key.encode(), int(value)), "r4_set_option(%s)" % key)
