"""Batch (offline) RL on the logged dataset: the ``train`` and ``eval`` stages of ``script/batchrl_train.py:109-128`` for
the three discrete algorithms of ``script/batchrl_trainer.py:get_model`` -- BC, BCQ and CQL -- over the dataset
``rl4rs_b200.dataset`` writes (Slate and SeqSlate).

The names are the reference's, so the script changes only its imports:
  get_model(config, algo)       -> a model with d3rlpy's AlgoBase surface the scripts call: fit, save_model, load_model,
                                   predict, predict_value
  build_with_dataset(model, ds) -> builds the networks for the dataset's observation width and fits CQL's reward scaler
  policy_model(model, config)   -> rl4rs/policy/policy_model.py: predict_with_mask, predict, action_probs, predict_q
  evaluate(config, policy)      -> batchrl_trainer.py:395-426 on the GPU env; returns the average reward
  load_dataset(path)            -> the writer's .npz (fit also takes the dict data_generate_* returns)

On a CUDA device the dataset is uploaded once and stays there; an epoch is one device permutation and one library call
(r4_batchrl_epoch: every minibatch's gradient and Adam step chained on the device, csrc/r4_batchrl.cuh), and acting is
r4_batchrl_act.  On the CPU the torch twin (policy.BatchRLNet) runs the same algorithm.  The d3rlpy 0.91 semantics
restated here are listed in INTEGRATION.md section 3 as not verified (d3rlpy is not in this
project's environment).

'BCQ-conti' (ContinuousBCQ) and 'CQL-conti' (ContinuousCQL) train on the continuous dataset (data_generate_rl4rs_a_conti /
_b_conti) for a config with support_conti_env: r4_bcqc_epoch / r4_cqlc_epoch on CUDA (csrc/r4_bcqconti.cuh,
csrc/r4_cqlconti.cuh), policy.BatchRLContiBCQNet / BatchRLContiNet on the CPU, r4_bcqc_act / r4_cqlc_act to act.

Both kinds share one front: DeviceDataset holds either kind of action, and BatchRLBase owns the set-up, the reward
scaler, fit and its epoch loops, and the checkpoints.  The discrete models (BatchRLModel) and the continuous ones
(ContinuousCQL, ContinuousBCQ) add their twin, hyper-parameters, entry-point calls, act and checkpoint keys.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _capi
from ._capi import ptr
from .policy import BatchRLContiBCQNet, BatchRLContiNet, BatchRLNet

ALGOS = {"BC": 0, "BCQ": 1, "CQL": 2}
NOT_BUILT = {
    "dynamics": "the ProbabilisticEnsembleDynamics model",
    "MOPO": "MOPO (needs the dynamics model)",
    "COMBO": "COMBO (needs the dynamics model)",
}
# the continuous learners exist for the continuous dataset only: the script sets support_conti_env for them
CONTI_ONLY = {"BCQ-conti": "continuous-action BCQ", "CQL-conti": "continuous-action CQL"}
# d3rlpy 0.91 defaults as batchrl_trainer.py:34-90 leaves or sets them (INTEGRATION.md section 3, not verified)
DEFAULTS = {
    "BC": {"batch_size": 256, "learning_rate": 1e-3, "eps": 1e-8, "beta": 0.0},
    "BCQ": {"batch_size": 256, "learning_rate": 6.25e-5, "eps": 1e-8, "gamma": 0.99, "beta": 0.5,
            "action_flexibility": 0.3, "target_update_interval": 8000},
    "CQL": {"batch_size": 256, "learning_rate": 6.25e-5, "eps": 1e-8, "gamma": 1.0, "alpha": 1.0,
            "target_update_interval": 8000, "reward_scaler": "standard"},
    # d3rlpy 0.91 BCQ (continuous) with batchrl_trainer.py:61-73's batch size (INTEGRATION.md section 3, not verified)
    "BCQ-conti": {"batch_size": 256, "actor_learning_rate": 1e-3, "critic_learning_rate": 1e-3,
                  "imitator_learning_rate": 1e-3, "eps": 1e-8, "gamma": 0.99, "tau": 0.005, "lam": 0.75,
                  "n_action_samples": 100, "action_flexibility": 0.05, "latent_size": 32, "beta": 0.5,
                  "update_actor_interval": 1, "rl_start_epoch": 0, "reward_scaler": None},
    # d3rlpy 0.91 CQL (continuous) with batchrl_trainer.py:61-73's batch size, gamma and reward scaler
    "CQL-conti": {"batch_size": 256, "actor_learning_rate": 1e-4, "critic_learning_rate": 3e-4,
                  "temp_learning_rate": 1e-4, "alpha_learning_rate": 1e-4, "eps": 1e-8, "gamma": 1.0, "tau": 0.005,
                  "initial_temperature": 1.0, "initial_alpha": 1.0, "alpha_threshold": 10.0, "conservative_weight": 5.0,
                  "n_action_samples": 10, "soft_q_backup": False, "reward_scaler": "standard"},
}


def get_model(config, algo, dynamics=None):
    """batchrl_trainer.get_model: 'BC', 'BCQ' or 'CQL' (alpha = config['CQL_alpha']), and 'CQL-conti' for a config with
    support_conti_env (the script sets it for the conti names).  CQL-conti ignores CQL_alpha, as d3rlpy 0.91's continuous
    CQL drops the unknown `alpha` argument: its initial alpha is 1.0 (INTEGRATION.md section 3).  The other names of the
    reference raise NotImplementedError; any other name fails its assert."""
    if algo in NOT_BUILT:
        raise NotImplementedError("%s: %s is not built in this project" % (algo, NOT_BUILT[algo]))
    if algo in CONTI_ONLY:
        if not config.get("support_conti_env", False):
            raise NotImplementedError("%s: %s is built for a support_conti_env config only (the continuous dataset of "
                                      "data_generate_rl4rs_a_conti / _b_conti)" % (algo, CONTI_ONLY[algo]))
        return {"BCQ-conti": ContinuousBCQ, "CQL-conti": ContinuousCQL}[algo](config)
    assert algo in ("BC", "BCQ", "CQL", "MOPO", "COMBO")
    cls = {"BC": DiscreteBC, "BCQ": DiscreteBCQ, "CQL": DiscreteCQL}[algo]
    extra = {"alpha": float(config["CQL_alpha"])} if algo == "CQL" and "CQL_alpha" in config else {}
    return cls(config, **extra)


def build_with_dataset(model, dataset):
    """batchrl_trainer.build_with_dataset: the networks for the dataset's observation width, then the reward scaler."""
    model.build_with_dataset(dataset)
    return model


def load_dataset(path):
    """The .npz rl4rs_b200.dataset writes -> a dict of its arrays."""
    with np.load(path) as z:
        return {k: z[k] for k in z.files}


def d3rlpy_eval(*args, **kwargs):
    raise NotImplementedError("d3rlpy_eval: the soft_opc / discrete_action_match scorers are not built in this project")


def ope_eval(*args, **kwargs):
    """Not here: the `ope` stage is rl4rs_b200.offline_evaluation.ope_eval (with its behavior_model), as the reference
    keeps it in script/offline_evaluation.py."""
    raise NotImplementedError("ope: the off-policy evaluation stage is not built in this project")


def _masks(config, A):
    """(location_mask [4, A], special_items) from the config (batchrl_train.py:32-40 puts them there), else from the
    catalog the env is built from, else from config['iteminfo_file'] (SlateState.get_mask_from_file)."""
    from .env.slate import SlateState
    if config.get("location_mask") is not None and config.get("special_items") is not None:
        return np.asarray(config["location_mask"]), [int(i) for i in config["special_items"]]
    if config.get("catalog") is not None:
        return SlateState._location_mask(A), [int(i) for i in config["catalog"].special_items]
    return SlateState.get_mask_from_file(config["iteminfo_file"], A)


def transitions_host(terminals):
    """The transition list of d3rlpy's episodes (split at the terminals): every entry i with terminals[i] == 0 before the last
    terminal entry.  The same rule as r4_batchrl_transitions, for the CPU path and the tests."""
    t = torch.as_tensor(np.asarray(terminals)).reshape(-1) != 0
    idx = torch.nonzero(t).reshape(-1)
    if idx.numel() == 0:
        return torch.zeros(0, dtype=torch.int64)
    last = int(idx[-1])
    return torch.nonzero(~t[:last]).reshape(-1).to(torch.int64)


class DeviceDataset(object):
    """The dataset where the learner runs: obs f32 [N, K], action i32 [N] (discrete: item ids) or f32 [N, D] (continuous:
    the logged items' embeddings, not clipped), reward f32 [N], terminal u8 [N] and the transition entries i64 [T].
    continuous: the kind the model needs; None takes the dataset's own (its discrete_action flag, else a single action
    column means discrete).  On CUDA it is uploaded once; a dataset that does not fit raises MemoryError."""

    def __init__(self, dataset, device, continuous=None):
        obs = np.asarray(dataset["observations"], dtype=np.float32)
        N = obs.shape[0]
        act = np.asarray(dataset["actions"])
        discrete = np.asarray(dataset.get("discrete_action", act.ndim < 2 or act.shape[1] == 1)).item()
        self.continuous = not discrete if continuous is None else bool(continuous)
        if self.continuous:
            act = np.asarray(act, dtype=np.float32)
            if discrete or act.ndim != 2 or act.shape[0] != N:
                raise ValueError("continuous batch RL needs the continuous dataset (actions f32 [N, D], discrete_action "
                                 "False): data_generate_rl4rs_a_conti / _b_conti")
        else:
            act = act.reshape(N)
            if np.any(act != np.round(act)) or act.min(initial=0) < 0:
                raise ValueError("batch RL here is discrete: the dataset's actions must be item ids")
            act = act.astype(np.int32)
        self.device, self.N, self.K = torch.device(device), N, obs.shape[1]
        self.D = act.shape[1] if self.continuous else None
        need = obs.nbytes + act.nbytes + N * (4 + 1 + 8)
        if self.device.type == "cuda":
            free = torch.cuda.mem_get_info(self.device)[0]
            if need > free:
                raise MemoryError("the dataset needs %d bytes on %s, %d are free" % (need, self.device, free))
        try:
            self.obs = torch.from_numpy(obs).to(self.device)
            self.action = torch.from_numpy(act).to(self.device)
            self.reward = torch.from_numpy(np.asarray(dataset["rewards"], dtype=np.float32).reshape(N)).to(self.device)
            self.terminal = torch.from_numpy((np.asarray(dataset["terminals"]).reshape(N) != 0).astype(np.uint8)).to(self.device)
            if self.device.type == "cuda":
                lib = _capi.load_library()
                index = torch.empty(N, dtype=torch.int64, device=self.device)
                count = torch.zeros(1, dtype=torch.int64, device=self.device)
                rc = lib.r4_batchrl_transitions(ptr(self.terminal), N, ptr(index), ptr(count), _capi.stream(self.device))
                _capi.check(lib, None, rc, "r4_batchrl_transitions")
                self.transitions = index[:int(count)]
            else:
                self.transitions = transitions_host(self.terminal)
        except torch.OutOfMemoryError as exc:
            raise MemoryError("the dataset needs %d bytes on %s: %s" % (need, self.device, exc)) from exc
        self.n = int(self.transitions.numel())

    def batch(self, pos):
        """(obs, action, reward, next_obs, terminal) of the transitions at positions pos of the transition list."""
        e = self.transitions[pos]
        return self.obs[e], self.action[e], self.reward[e + 1], self.obs[e + 1], self.terminal[e + 1]

    def c_data(self):
        """The r4_cqlc_data structure of a continuous dataset (r4_cqlc_* and r4_bcqc_*)."""
        return _capi.CQLContiData(self.obs.data_ptr(), self.action.data_ptr(), self.reward.data_ptr(),
                                  self.terminal.data_ptr(), self.transitions.data_ptr())


class BatchRLBase(object):
    """d3rlpy AlgoBase's surface the scripts use (fit, save_model, load_model, predict, predict_value), shared by the
    discrete and continuous learners.  A family supplies its twin net (_new_net), its kernels' shape checks
    (_scratch_size), its hyper-parameters (_hyper, _hyper_c), one epoch and one gradient through its entry points
    (_epoch_call, grad_kernels), one twin step (train_step_twin), act, STAT_NAMES and its checkpoint keys (CKPT_ACTION,
    _extra_state / _load_extra)."""

    algo = None
    continuous = False
    STAT_NAMES = ()
    PREFIX = None
    CKPT_ACTION = None              # (the checkpoint key of the action shape, the attribute holding it, its unit)

    def __init__(self, config, device=None, seed=0, use_kernels=None, **overrides):
        self.config = dict(config)
        self.hp = dict(DEFAULTS[self.algo], **overrides)
        self.batch_size = int(self.hp["batch_size"])
        if device is None:
            device = "cuda" if torch.cuda.is_available() and config.get("gpu", True) else "cpu"
        self.device = torch.device(device)
        self.use_kernels = (self.device.type == "cuda") if use_kernels is None else bool(use_kernels)
        self.seed = seed
        self.net = None
        self.reward_mean, self.reward_std = 0.0, 1.0
        self.reward_scaler = None
        self._data, self._data_src = None, None
        self.step = 0

    # ---- building ------------------------------------------------------------------------------------
    def create_impl(self, obs_dim):
        self.net = self._new_net(obs_dim)
        z = lambda: torch.zeros(self.net.n_params, dtype=torch.float32, device=self.device)
        self.m, self.v = z(), z()
        self.step = 0
        self._gen = torch.Generator(device=self.device).manual_seed(self.seed)
        if self.use_kernels:
            self.lib = _capi.load_library()
            n = self._scratch_size(obs_dim)
            self.grad = z()
            self.stats = torch.zeros(len(self.STAT_NAMES), dtype=torch.float32, device=self.device)
            self.scratch = torch.zeros(n, dtype=torch.float32, device=self.device)

    def build_with_dataset(self, dataset):
        obs = dataset["observations"]
        if self.net is None or self.net.K != obs.shape[1]:
            self.create_impl(obs.shape[1])
        if self.hp.get("reward_scaler") == "standard":
            self.fit_reward_scaler(dataset)

    def fit_reward_scaler(self, dataset):
        """d3rlpy StandardRewardScaler.fit: mean and (population) std of the transitions' rewards, rewards[i] over the
        transition entries i."""
        idx = transitions_host(dataset["terminals"]).numpy()
        r = np.asarray(dataset["rewards"], dtype=np.float64).reshape(-1)[idx]
        self.reward_mean, self.reward_std = float(r.mean()), float(r.std())
        self.reward_scaler = "standard"

    def _reward_norm(self):
        """The reward normalisation the losses apply, r -> (r - reward_mean) / reward_den (identity without a scaler)."""
        return {"reward_mean": self.reward_mean if self.reward_scaler else 0.0,
                "reward_den": (self.reward_std + 1e-3) if self.reward_scaler else 1.0}

    # ---- training ------------------------------------------------------------------------------------
    def _device_data(self, dataset):
        if self._data_src is not dataset:
            self._data = None                       # release the previous upload first
            self._data = DeviceDataset(dataset, self.device, self.continuous)
            self._data_src = dataset
        return self._data

    def fit(self, dataset, n_epochs=1, eval_episodes=None, show_progress=False, **kwargs):
        """d3rlpy fit with its RoundIterator: per epoch one permutation of the transitions (drawn on the device) and
        floor(n / batch_size) minibatches in order.  eval_episodes is accepted and not scored (no scorers are passed).
        A standard reward scaler is fitted here only when it has not been fitted yet (on the first dataset, or by
        build_with_dataset): a later fit on another dataset keeps those statistics; build_with_dataset refits them.
        Returns [(epoch, {STAT_NAMES: the epoch's means})]."""
        data = self._device_data(dataset)
        if self.continuous and data.D != self.D:
            raise ValueError("the dataset's actions have %d dims, the model %d" % (data.D, self.D))
        if self.net is None or self.net.K != data.K:
            self.build_with_dataset(dataset)
        elif self.hp.get("reward_scaler") == "standard" and self.reward_scaler is None:
            self.fit_reward_scaler(dataset)
        mb = self.batch_size
        if data.n < mb:
            raise ValueError("the dataset has %d transitions, fewer than one minibatch of %d" % (data.n, mb))
        out = []
        for epoch in range(1, int(n_epochs) + 1):
            perm = torch.randperm(data.n, generator=self._gen, device=self.device)
            st = self._epoch_kernels(data, perm) if self.use_kernels else self._epoch_twin(data, perm)
            out.append((epoch, dict(zip(self.STAT_NAMES, st))))
            if show_progress:
                print("epoch %d %s" % (epoch, out[-1][1]))
        return out

    def _epoch_twin(self, data, perm):
        mb, steps = self.batch_size, data.n // self.batch_size
        acc = torch.zeros(len(self.STAT_NAMES), dtype=torch.float64)
        for k in range(steps):
            acc += self.train_step_twin(data.batch(perm[k * mb:(k + 1) * mb])).double().cpu()
        return [float(v) for v in acc / max(steps, 1)]

    def _epoch_kernels(self, data, perm):
        steps, nst = data.n // self.batch_size, len(self.STAT_NAMES)
        stats = torch.zeros(steps * nst, dtype=torch.float32, device=self.device)
        rc = self._epoch_call(data, perm, stats)
        if rc < 0:
            self._check(rc, self.PREFIX + "_epoch")
        self.step += rc
        return [float(v) for v in stats.view(steps, nst).double().mean(0)]

    def _stream(self):
        return _capi.stream(self.device)

    def _check(self, rc, what):
        _capi.check(self.lib, None, rc, what)

    # ---- acting --------------------------------------------------------------------------------------
    def _obs(self, obs):
        """Observations (numpy or torch, f32 or f64 [n, K]) as a contiguous device tensor, f32 or f64."""
        x = torch.as_tensor(obs, device=self.device)
        if x.dtype not in (torch.float32, torch.float64):
            x = x.to(torch.float32)
        return x.reshape(-1, self.net.K).contiguous()

    # ---- checkpoints ---------------------------------------------------------------------------------
    def save_model(self, fname):
        """torch.save of every network (the flat vector), the target, the Adam moments, the step counter, the reward
        scaler and the family's own keys (_extra_state), so a loaded model predicts and continues fit as the saved one
        would."""
        key, attr, _ = self.CKPT_ACTION
        torch.save(dict({"algo": self.algo, "obs_dim": self.net.K, key: getattr(self, attr),
                         "params": self.net.flat.detach().cpu(), "target": self.net.target.cpu(), "m": self.m.cpu(),
                         "v": self.v.cpu(), "step": self.step, "reward_scaler": self.reward_scaler,
                         "reward_mean": self.reward_mean, "reward_std": self.reward_std}, **self._extra_state()), fname)

    def load_model(self, fname):
        ck = torch.load(fname, map_location="cpu")
        key, attr, unit = self.CKPT_ACTION
        if ck["algo"] != self.algo or ck.get(key) != getattr(self, attr):
            raise ValueError("%s holds a %s model for %d %s" % (fname, ck["algo"], ck.get(key, -1), unit))
        if self.net is None or self.net.K != ck["obs_dim"]:
            self.create_impl(ck["obs_dim"])
        with torch.no_grad():
            for dst, k in ((self.net.flat, "params"), (self.net.target, "target"), (self.m, "m"), (self.v, "v")):
                dst.copy_(ck[k].to(self.device))
        self.step = int(ck["step"])
        self.reward_scaler, self.reward_mean, self.reward_std = ck["reward_scaler"], ck["reward_mean"], ck["reward_std"]
        self._load_extra(ck)

    def _extra_state(self):
        return {}

    def _load_extra(self, ck):
        pass


class BatchRLModel(BatchRLBase):
    """The discrete learners over policy.BatchRLNet (CPU) or the r4_batchrl_* kernels (CUDA)."""

    STAT_NAMES = ("loss", "td", "q")
    PREFIX = "r4_batchrl"
    CKPT_ACTION = ("action_size", "A", "actions")

    def __init__(self, config, **kw):
        super(BatchRLModel, self).__init__(config, **kw)
        self.A = int(config.get("action_size", 284))
        if int(config.get("page_items", 9)) != 9:
            raise ValueError("the custom encoder reads 9 prev actions (page_items = 9)")
        self.location_mask, self.special_items = _masks(config, self.A)

    # ---- building ------------------------------------------------------------------------------------
    def _new_net(self, obs_dim):
        return BatchRLNet(self.algo, obs_dim, self.location_mask, self.special_items, self.A, self.device, self.seed)

    def _scratch_size(self, obs_dim):
        k = ALGOS[self.algo]
        assert self.lib.r4_batchrl_num_params(k, obs_dim, self.A) == self.net.n_params
        assert self.lib.r4_batchrl_target_size(k, obs_dim, self.A) == self.net.n_target
        n = self.lib.r4_batchrl_scratch_size(k, obs_dim, self.A, self.batch_size)
        if n < 0:
            raise ValueError("obs_dim %d / action_size %d is outside the kernels' range" % (obs_dim, self.A))
        return n

    @property
    def _tables(self):
        return BatchRLDataPtrs(self.net)

    def _hyper(self):
        hp = self.hp
        return dict({"gamma": float(hp.get("gamma", 0.0)), "beta": float(hp.get("beta", 0.0)),
                     "alpha": float(hp.get("alpha", 0.0)),
                     "log_flex": float(np.float32(math.log(hp.get("action_flexibility", 0.3))))}, **self._reward_norm())

    def _hyper_c(self):
        h = self._hyper()
        return _capi.BatchRLHyper(h["gamma"], h["beta"], h["alpha"], h["log_flex"], h["reward_mean"], h["reward_den"])

    # ---- training ------------------------------------------------------------------------------------
    def train_step_twin(self, batch, hp=None):
        """One SGD step of the twin: autograd gradient, the kernels' Adam, the hard target copy when due."""
        hp = hp or self._hyper()
        net = self.net
        if net.flat.grad is not None:
            net.flat.grad.zero_()
        loss, st = net.loss(*batch, hp)
        loss.backward()
        self.step += 1
        with torch.no_grad():
            adam_(net.flat.data, net.flat.grad, self.m, self.v, self.step, self.hp["learning_rate"], self.hp["eps"])
            if self._copy_due(self.step):
                net.target.copy_(net.flat.detach()[:net.n_target])
        self._last_stats = st
        return st

    def _copy_due(self, step):
        ti = int(self.hp.get("target_update_interval", 0))
        return self.net.n_target > 0 and ti > 0 and (step - 1) % ti == 0

    def _epoch_call(self, data, perm, stats):
        return self.lib.r4_batchrl_epoch(ALGOS[self.algo], self.net.K, self.A, ptr(self.net.flat), ptr(self.net.target),
                                         ptr(self.m), ptr(self.v), C.byref(self._tables.data(data)),
                                         C.byref(self._hyper_c()), ptr(perm), perm.numel(), self.batch_size, self.step,
                                         self.hp["learning_rate"], self.hp["eps"],
                                         int(self.hp.get("target_update_interval", 0)), ptr(self.scratch), ptr(stats),
                                         self._stream())

    def grad_kernels(self, data, pos):
        """r4_batchrl_grad over the transitions at positions pos (i64, device) -> self.grad, self.stats."""
        rc = self.lib.r4_batchrl_grad(ALGOS[self.algo], self.net.K, self.A, ptr(self.net.flat), ptr(self.net.target),
                                      C.byref(self._tables.data(data)), C.byref(self._hyper_c()), ptr(pos), pos.numel(),
                                      ptr(self.scratch), ptr(self.grad), ptr(self.stats), self._stream())
        self._check(rc, "r4_batchrl_grad")

    # ---- acting --------------------------------------------------------------------------------------
    def act(self, obs, mode=0, want_probs=False, want_values=False):
        """The act rule on observations (numpy or torch, f32 or f64 [n, K]) -> (action i32 [n], probs or None, values or
        None) as device tensors.  mode 0: predict_with_mask's rule; mode 1: d3rlpy's predict."""
        x = self._obs(obs)
        log_flex = self._hyper()["log_flex"]
        if not self.use_kernels:
            a, probs, raw = self.net.act(x, mode, log_flex)
            return a, probs if want_probs else None, raw if want_values else None
        n = x.shape[0]
        a = torch.empty(n, dtype=torch.int32, device=self.device)
        probs = torch.empty(n, self.A, dtype=torch.float32, device=self.device) if want_probs else None
        vals = torch.empty(n, self.A, dtype=torch.float32, device=self.device) if want_values else None
        rc = self.lib.r4_batchrl_act(ALGOS[self.algo], self.net.K, self.A, ptr(self.net.flat), ptr(x),
                                     int(x.dtype == torch.float64), n, C.byref(self._tables.tables()), mode, log_flex,
                                     ptr(a), ptr(probs), ptr(vals), self._stream())
        self._check(rc, "r4_batchrl_act")
        return a, probs, vals

    def predict(self, x):
        """d3rlpy predict: the greedy action of the algorithm (no location mask) -> int array [n]."""
        return self.act(x, 1)[0].long().cpu().numpy()

    def predict_value(self, x, action):
        """d3rlpy predict_value: Q(s, a) in the scaled reward units (BC: its logit of a)."""
        vals = self.act(x, 1, want_values=True)[2]
        a = torch.as_tensor(np.asarray(action), device=self.device).long().reshape(-1)
        return vals[torch.arange(vals.shape[0], device=self.device), a].cpu().numpy()


class DiscreteBC(BatchRLModel):
    algo = "BC"
    STAT_NAMES = ("loss", "nll", "penalty")


class DiscreteBCQ(BatchRLModel):
    algo = "BCQ"


class DiscreteCQL(BatchRLModel):
    algo = "CQL"


class ContinuousCQL(BatchRLBase):
    """d3rlpy 0.91 CQL (continuous actions) as batchrl_trainer.py:61-73 configures 'CQL-conti', over
    policy.BatchRLContiNet (CPU) or the r4_cqlc_* kernels (CUDA).  One SGD step updates the temperature, alpha, the
    critics and the actor in that order, each with its own Adam, then the critics' soft target.  The noise of step t is
    keyed by (seed, t) (policy.cqlc_draws), so the CPU and CUDA paths draw the same numbers.  Its checkpoint also holds
    the act counter and the epoch-permutation generator's state."""

    algo = "CQL-conti"
    continuous = True
    PREFIX = "r4_cqlc"
    STAT_NAMES = ("critic_loss", "actor_loss", "temp_loss", "alpha_loss", "q")
    CKPT_ACTION = ("action_dim", "D", "action dims")
    # (loss, learning-rate key, its stats slots), in update order; the soft target update follows SOFT_AFTER's update
    PHASES = (("temp", "temp_learning_rate", (2,)), ("alpha", "alpha_learning_rate", (3,)),
              ("critic", "critic_learning_rate", (0, 4)), ("actor", "actor_learning_rate", (1,)))
    SOFT_AFTER = "critic"

    def __init__(self, config, **kw):
        super(ContinuousCQL, self).__init__(config, **kw)
        if self.hp.get("soft_q_backup"):
            raise NotImplementedError("CQL-conti: soft_q_backup is not built (the script leaves it False)")
        onehot = config.get("support_onehot_action", False)
        self.D = int(config.get("action_size", 284)) if onehot else int(config.get("action_emb_size", 32))
        self.act_counter = 0

    # ---- building ------------------------------------------------------------------------------------
    def _new_net(self, obs_dim):
        hp = self.hp
        return BatchRLContiNet(obs_dim, self.D, self.device, self.seed, hp["initial_temperature"], hp["initial_alpha"])

    def _dims(self, K):
        """The leading shape arguments of the r4_*_num_params / _target_size / _scratch_size calls."""
        return (K, self.D)

    def _scratch_size(self, obs_dim):
        dims = self._dims(obs_dim)
        if getattr(self.lib, self.PREFIX + "_num_params")(*dims) != self.net.n_params:
            raise ValueError("obs_dim %d / action_dim %d is outside the kernels' range" % (obs_dim, self.D))
        assert getattr(self.lib, self.PREFIX + "_target_size")(*dims) == self.net.n_target
        n = getattr(self.lib, self.PREFIX + "_scratch_size")(*dims, int(self.hp["n_action_samples"]), self.batch_size)
        if n < 0:
            raise ValueError("batch_size %d / n_action_samples %d is outside the kernels' range"
                             % (self.batch_size, self.hp["n_action_samples"]))
        return n

    def build_with_dataset(self, dataset):
        act = np.asarray(dataset["actions"])
        if act.ndim != 2 or act.shape[1] != self.D:
            raise ValueError("the dataset's actions have shape %s, the model takes [N, %d] (action_emb_size, or "
                             "action_size with support_onehot_action)" % (act.shape, self.D))
        super(ContinuousCQL, self).build_with_dataset(dataset)

    def _hyper(self):
        hp = self.hp
        return dict({"gamma": float(hp["gamma"]), "tau": float(hp["tau"]), "alpha_threshold": float(hp["alpha_threshold"]),
                     "conservative_weight": float(hp["conservative_weight"])}, **self._reward_norm())

    def _hyper_c(self):
        h, hp = self._hyper(), self.hp
        return _capi.CQLContiHyper(h["gamma"], h["tau"], hp["actor_learning_rate"], hp["critic_learning_rate"],
                                   hp["temp_learning_rate"], hp["alpha_learning_rate"], hp["eps"], h["alpha_threshold"],
                                   h["conservative_weight"], h["reward_mean"], h["reward_den"], int(hp["n_action_samples"]),
                                   self.seed)

    # ---- training ------------------------------------------------------------------------------------
    def train_step_twin(self, batch):
        """One SGD step of the twin with the kernels' noise: the PHASES' updates in order (each loss at the parameters the
        earlier updates left), the soft target update after SOFT_AFTER's.  -> stats [5]."""
        net, hp, h = self.net, self.hp, self._hyper()
        self.step += 1
        noise = net.noise(self.seed, self.step, batch[0].shape[0], int(hp["n_action_samples"]))
        st = torch.zeros(5, dtype=torch.float32, device=self.device)
        for name, lr, slots in self.PHASES:
            losses, s = net.losses(batch, noise, h)
            g = torch.autograd.grad(losses[name], net.flat)[0]
            sl = net.group(name)
            for k in slots:
                st[k] = s[k]
            adam_(net.flat.data[sl], g[sl], self.m[sl], self.v[sl], self.step, hp[lr], hp["eps"])
            if name == self.SOFT_AFTER:
                net.soft_update(hp["tau"])
        self._last_stats = st
        return st

    def _epoch_call(self, data, perm, stats):
        return getattr(self.lib, self.PREFIX + "_epoch")(self.net.K, self.D, ptr(self.net.flat), ptr(self.net.target),
                                                          ptr(self.m), ptr(self.v), C.byref(data.c_data()),
                                                          C.byref(self._hyper_c()), ptr(perm), perm.numel(),
                                                          self.batch_size, self.step, ptr(self.scratch), ptr(stats),
                                                          self._stream())

    def grad_kernels(self, data, pos, step=None):
        """r4_cqlc_grad / r4_bcqc_grad over the transitions at positions pos (i64, device) with the noise of `step`
        (default: the next step) -> self.grad, self.stats."""
        rc = getattr(self.lib, self.PREFIX + "_grad")(self.net.K, self.D, ptr(self.net.flat), ptr(self.net.target), C.byref(data.c_data()),
                                   C.byref(self._hyper_c()), ptr(pos), pos.numel(), self.step + 1 if step is None else step,
                                   ptr(self.scratch), ptr(self.grad), ptr(self.stats), self._stream())
        self._check(rc, self.PREFIX + "_grad")

    # ---- acting --------------------------------------------------------------------------------------
    def _act_inputs(self, obs, action):
        x = self._obs(obs)
        a_in = None if action is None else torch.as_tensor(np.asarray(action) if not torch.is_tensor(action) else action,
                                                             device=self.device, dtype=torch.float32).reshape(-1, self.D)
        return x, None if a_in is None else a_in.contiguous()

    def act(self, obs, action=None, want_q=False):
        """tanh(mu) [n, D] and (want_q) the critics' mean at (obs, action or tanh mu) [n], as device tensors; obs numpy
        or torch, f32 or f64 [n, K]."""
        x, a_in = self._act_inputs(obs, action)
        if not self.use_kernels:
            with torch.no_grad():
                a = self.net.predict(x.to(torch.float32))
                q = self.net.predict_value(x.to(torch.float32), a if a_in is None else a_in) if want_q else None
            return a, q
        n = x.shape[0]
        a = torch.empty(n, self.D, dtype=torch.float32, device=self.device)
        q = torch.empty(n, dtype=torch.float32, device=self.device) if want_q else None
        scratch = torch.empty(self.lib.r4_cqlc_act_scratch_size(self.net.K, self.D, n), dtype=torch.float32,
                              device=self.device)
        rc = self.lib.r4_cqlc_act(self.net.K, self.D, ptr(self.net.flat), ptr(x), int(x.dtype == torch.float64), n,
                                  ptr(a_in), ptr(a), ptr(q), ptr(scratch), self._stream())
        self._check(rc, "r4_cqlc_act")
        return a, q

    def predict(self, x):
        """d3rlpy predict: tanh(mu) -> f32 numpy [n, D]."""
        return self.act(x)[0].cpu().numpy()

    def predict_value(self, x, action):
        """d3rlpy predict_value: the mean of the two critics' Q(s, a), in the scaled reward units -> numpy [n]."""
        return self.act(x, action, want_q=True)[1].cpu().numpy()

    # ---- checkpoints ---------------------------------------------------------------------------------
    def _extra_state(self):
        return {"act_counter": self.act_counter, "gen": self._gen.get_state()}

    def _load_extra(self, ck):
        self.act_counter = int(ck["act_counter"])
        self._gen.set_state(ck["gen"])


class ContinuousBCQ(ContinuousCQL):
    """d3rlpy 0.91 BCQ (continuous actions) as batchrl_trainer.py:61-73 configures 'BCQ-conti', over
    policy.BatchRLContiBCQNet (CPU) or the r4_bcqc_* kernels (CUDA).  One SGD step updates the VAE imitator, the critics
    and the actor in that order, each with its own Adam, then the soft update of the actor and critic targets.  predict is
    stochastic: each call draws its latents from (seed, the call counter)."""

    algo = "BCQ-conti"
    PREFIX = "r4_bcqc"
    STAT_NAMES = ("imitator_loss", "critic_loss", "actor_loss", "q", "reconstruction")
    PHASES = (("imitator", "imitator_learning_rate", (0, 4)), ("critic", "critic_learning_rate", (1, 3)),
              ("actor", "actor_learning_rate", (2,)))
    SOFT_AFTER = "actor"

    def __init__(self, config, **kw):
        super(ContinuousBCQ, self).__init__(config, **kw)
        if int(self.hp["update_actor_interval"]) != 1 or int(self.hp["rl_start_epoch"]) != 0:
            raise NotImplementedError("BCQ-conti: update_actor_interval != 1 and rl_start_epoch != 0 are not built (the "
                                      "script leaves them at 1 and 0)")

    def _new_net(self, obs_dim):
        return BatchRLContiBCQNet(obs_dim, self.D, self.device, self.seed, int(self.hp["latent_size"]))

    def _dims(self, K):
        return (K, self.D, int(self.hp["latent_size"]))

    def _hyper(self):
        hp = self.hp
        return {"gamma": float(hp["gamma"]), "tau": float(hp["tau"]), "lam": float(hp["lam"]), "beta": float(hp["beta"]),
                "action_flexibility": float(hp["action_flexibility"]),
                "reward_mean": self.reward_mean if self.reward_scaler else 0.0,
                "reward_den": (self.reward_std + 1e-3) if self.reward_scaler else 1.0}

    def _hyper_c(self):
        h, hp = self._hyper(), self.hp
        return _capi.BCQContiHyper(h["gamma"], h["tau"], hp["actor_learning_rate"], hp["critic_learning_rate"],
                                   hp["imitator_learning_rate"], hp["eps"], h["lam"], h["beta"], h["action_flexibility"],
                                   h["reward_mean"], h["reward_den"], int(hp["n_action_samples"]), int(hp["latent_size"]),
                                   self.seed)

    def act(self, obs, action=None, want_q=False):
        """The best of n_action_samples decoded, perturbed candidates by Q_0 [n, D] (when action is None) and (want_q)
        the critics' mean at (obs, action or that prediction) [n], as device tensors."""
        x, a_in = self._act_inputs(obs, action)
        n, S = x.shape[0], int(self.hp["n_action_samples"])
        a = None
        if a_in is None:
            self.act_counter += 1
        if not self.use_kernels:
            with torch.no_grad():
                x32 = x.to(torch.float32)
                if a_in is None:
                    z = self.net.predict_noise(self.seed, self.act_counter, n, S)
                    a = self.net.predict(x32, z, self._hyper())
                q = self.net.predict_value(x32, a if a_in is None else a_in) if want_q else None
            return a, q
        a = torch.empty(n, self.D, dtype=torch.float32, device=self.device) if a_in is None else None
        q = torch.empty(n, dtype=torch.float32, device=self.device) if want_q else None
        size = self.lib.r4_bcqc_act_scratch_size(self.net.K, self.D, int(self.hp["latent_size"]), S, n)
        if size < 0:
            raise ValueError("predict on %d rows x %d samples is outside the kernels' range" % (n, S))
        scratch = torch.empty(size, dtype=torch.float32, device=self.device)
        rc = self.lib.r4_bcqc_act(self.net.K, self.D, ptr(self.net.flat), ptr(x), int(x.dtype == torch.float64), n,
                                  C.byref(self._hyper_c()), self.act_counter, ptr(a_in), ptr(a), ptr(q), ptr(scratch),
                                  self._stream())
        self._check(rc, "r4_bcqc_act")
        return a, q


class BatchRLDataPtrs(object):
    """The r4_batchrl_data structure: the device dataset's planes and the net's masking tables."""

    def __init__(self, net):
        self.net = net

    def tables(self):
        from ._capi import BatchRLData
        d = BatchRLData()
        d.location_mask, d.special = self.net.location_mask.data_ptr(), self.net.special.data_ptr()
        return d

    def data(self, ds):
        d = self.tables()
        d.obs, d.action, d.reward = ds.obs.data_ptr(), ds.action.data_ptr(), ds.reward.data_ptr()
        d.terminal, d.transitions = ds.terminal.data_ptr(), ds.transitions.data_ptr()
        return d


@torch.no_grad()
def adam_(p, g, m, v, step, lr, eps, b1=0.9, b2=0.999):
    """torch.optim.Adam's update in the operation order of csrc/r4_ppo.cuh adam_update."""
    m.mul_(b1).add_((1 - b1) * g)
    v.mul_(b2).add_((1 - b2) * g * g)
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    p.sub_((lr / bc1) * (m / (v.sqrt() / math.sqrt(bc2) + eps)))


class policy_model(object):
    """rl4rs/policy/policy_model.py over a batch-RL model or a model-free trainer (trainer.get_rl_model's PPO / A2C /
    PG / IMPALA and RAINBOW: the RLlib branch of policy_model.py:37-38, 47-50, 62-69, 83-87, through compute_actions)."""

    def __init__(self, model, config={}):
        self.policy = model
        self.config = config
        self.page_items = int(config.get("page_items", 9))
        self.mask_size = self.page_items + 1
        self.location_mask = config.get("location_mask", None)
        self.special_items = config.get("special_items", None)

    @property
    def _rllib(self):
        return hasattr(self.policy, "compute_actions")

    @staticmethod
    def _rllib_obs(obs):
        """policy_model.py's dict(enumerate(obs)) for a list of rows; batched arrays, tensors and field dicts go as they
        are (compute_actions takes both forms)."""
        return dict(enumerate(obs)) if isinstance(obs, list) else obs

    def predict_with_mask(self, obs):
        """policy_model.py:17-36: action_probs, -2^15 where the location layer, the prev actions or the special-item rule
        exclude an item, the first argmax.  A device tensor in gives a device tensor out, else a numpy array.  Under
        support_conti_env it is predict (policy_model.py:18-19); a continuous model then returns device actions
        f32 [n, D] for a device tensor.  A trainer: predict (policy_model.py:37-38)."""
        if self._rllib:
            return self.predict(obs)
        if self.config.get("support_conti_env", False):
            if hasattr(obs, "is_cuda") and self.policy.continuous:
                return self.policy.act(obs)[0]
            return self.predict(obs)
        a = self.policy.act(obs, 0)[0]
        return a if hasattr(obs, "is_cuda") else a.long().cpu().numpy()

    def predict(self, obs):
        if self._rllib:
            a = self.policy.compute_actions(self._rllib_obs(obs), explore=False)
            return np.array(list(a.values())) if isinstance(a, dict) else np.asarray(a)
        return self.policy.predict(obs)

    def predict_q(self, obs, action):
        if self._rllib:
            _, _, infos = self.policy.compute_actions(self._rllib_obs(obs), explore=False, full_fetch=True)
            if "q_values" in infos:
                return infos["q_values"][range(len(action)), action]
            return infos["vf_preds"]
        q = self.policy.predict_value(obs, action)
        if self.policy.reward_scaler is not None:
            return q * (self.policy.reward_std + 1e-3) + self.policy.reward_mean
        return q

    def action_probs(self, obs):
        """BC: the imitator's log-probs; BCQ / CQL: softmax(Q); a trainer: softmax(action_dist_inputs)."""
        if self._rllib:
            from scipy.special import softmax
            _, _, infos = self.policy.compute_actions(self._rllib_obs(obs), explore=False, full_fetch=True)
            return softmax(infos["action_dist_inputs"], axis=1)
        return self.policy.act(obs, 0, want_probs=True)[1].cpu().numpy()

    def _ope_fetch(self, obs):
        """One act of the policy for offline_evaluation.ope_eval, as device tensors where the policy runs: (the env
        action, probs [n, A] or logits, whether they are logits, the own action or None, values [n, A] or [n], the host
        fix of the values or None).  The same numbers predict_with_mask, action_probs and predict_q give."""
        if self._rllib:
            a, infos = self.policy._fetch(obs)
            env_a = a if hasattr(obs, "is_cuda") or isinstance(obs, dict) and hasattr(next(iter(obs.values())), "is_cuda") \
                else a.long().cpu().numpy()
            if "q_values" in infos:
                return env_a, infos["action_dist_inputs"], True, a, infos["q_values"], None
            return env_a, infos["action_dist_inputs"], True, None, infos["vf_preds"], None
        a, probs, vals = self.policy.act(obs, 0, want_probs=True, want_values=True)
        env_a = a if hasattr(obs, "is_cuda") else a.long().cpu().numpy()
        fix = None
        if self.policy.reward_scaler is not None:
            std, mean = self.policy.reward_std, self.policy.reward_mean
            fix = lambda q: q * (std + 1e-3) + mean
        return env_a, probs, False, a, vals, fix


def make_eval_env(config, batch_size=2048):
    """The eval env of batchrl_trainer.evaluate: is_eval, the given batch, the d3rl mask and the 'torch' output format."""
    from . import gymshim as gym
    from .env.seqslate import SeqSlateRecEnv, SeqSlateState
    from .env.slate import SlateRecEnv, SlateState
    cfg = dict(config, is_eval=True, batch_size=batch_size, support_d3rl_mask=True, support_rllib_mask=False,
               output_format="torch")
    cfg.setdefault("cache_size", batch_size)
    name = cfg.get("env", "SlateRecEnv-v0")
    assert name in ("SlateRecEnv-v0", "SeqSlateRecEnv-v0")
    if name == "SeqSlateRecEnv-v0":
        return gym.make(name, recsim=SeqSlateRecEnv(cfg, state_cls=SeqSlateState))
    return gym.make(name, recsim=SlateRecEnv(cfg, state_cls=SlateState))


def evaluate(config, policy, batch_size=2048, episodes=4, env=None):
    """batchrl_trainer.evaluate (:395-426): `episodes` episodes of max_steps steps at `batch_size` with
    predict_with_mask; prints the reference's lines and returns the average episode reward."""
    env = env if env is not None else make_eval_env(config, batch_size)
    T = config["max_steps"]
    total, rmax, rmin, B = 0.0, -math.inf, math.inf, batch_size
    for i in range(episodes):
        obs = env.reset()
        print("test batch at ", i)
        ep = None
        for _ in range(T):
            action = policy.predict_with_mask(obs)
            obs, reward, done, info = env.step(action)
            r = torch.as_tensor(reward).to(torch.float64)
            ep = r if ep is None else ep + r
        total, B = total + float(ep.sum()), ep.numel()
        rmax, rmin = max(rmax, float(ep.max())), min(rmin, float(ep.min()))
    print("reward max min", rmax, rmin)
    avg = total / B / episodes
    print("avg reward", avg)
    return avg
