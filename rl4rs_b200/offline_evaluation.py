"""Off-policy evaluation: the `ope` stage of script/batchrl_train.py and script/modelfree_train.py, which build a
behaviour model from logged_policy.h5 and call script/offline_evaluation.py:ope_eval.  The scripts change only their
import:

  behavior_model(config, modelfile)   -> rl4rs/policy/behavior_model.py: action_probs(records, action, layer, page=0)
  ope_eval(config, eval_env, algo, sample_model=None)
                                      -> offline_evaluation.py:9-73: prints 'IS DR WIPS SeqDR' and the mean and std over
                                         epochs of the (value, half-width) pairs, and returns the [epoch, 4, 2] metrics

The behaviour net is nets/dnn.py's graph at 50 dense features (behavior_model.py:11-13 fixes its inputs) with as many
classes as its stored `simulator_reward` kernel has.  On CUDA it runs on the r4_ope_* kernels (csrc/r4_ope.cuh): the
records are parsed and uploaded once per reset, each page's forward runs once per episode and stays on the device, and
each step is one gather launch that writes the step's propensities, value and rewards into [T, B] device buffers, which
the host copies once per epoch.  With use_kernels=False, or without CUDA, a torch twin runs the same net, gather and loop.
The estimators are utils.offline_policy_metrics.  INTEGRATION.md "Off-policy evaluation" lists the reference quirks kept
here and what is not verified.
"""
import contextlib

import numpy as np
import torch

from . import _capi
from ._capi import ptr
from .batchrl import policy_model
from .utils import offline_policy_metrics as OPE
from .utils import tf_checkpoint
from .utils.datautil import FeatureUtil

E, NHEAD, NCAT, NDENSE, NITEMF = 128, 11, 21, 50, 5
DNN_CFG = {"dense_feature_num": NDENSE, "category_feature_num": NCAT, "emb_size": E, "hidden_units": 128}


def dnn_plan(H, C):
    """tf_checkpoint.dnn_layer_plan for the behaviour net: [(W-table name, Keras layer scope, shape)]."""
    return tf_checkpoint.dnn_layer_plan(dict(DNN_CFG, category_hash_size=H, class_num=C))


def _check_table(w, where):
    """A W-table of the behaviour net: every plan entry present at its shape (H and C from emb_cat and rew_w)."""
    if "emb_cat" not in w or "rew_w" not in w:
        raise KeyError("%s is not the dnn behaviour net: it has no emb_cat / rew_w (keys %s)" % (where, sorted(w)))
    H, C = int(np.shape(w["emb_cat"])[0]), int(np.shape(w["rew_w"])[-1])
    out = {}
    for name, _, shape in dnn_plan(H, C):
        if name not in w:
            raise KeyError("%s: %s is missing (the dnn behaviour net needs %s)" % (where, name, [n for n, _, _ in dnn_plan(H, C)]))
        if tuple(np.shape(w[name])) != tuple(shape):
            raise ValueError("%s: %s has shape %s, the dnn behaviour net needs %s" % (where, name, np.shape(w[name]), shape))
        out[name] = np.ascontiguousarray(w[name], dtype=np.float32)
    return out, H, C


def _h5_table(path):
    """Keras .h5 (model_weights/<layer>/<layer>/<var>:0) -> W-table, each plan entry taken from its layer scope by
    shape.  Needs h5py."""
    try:
        import h5py
    except ImportError as exc:
        raise ImportError("reading %s needs h5py; without it, convert the weights to an .npz keyed by the dnn W-table "
                          "names (%s) and pass that file" % (path, ", ".join(n for n, _, _ in dnn_plan(1, 149)))) from exc
    with h5py.File(path, "r") as f:
        root = f["model_weights"] if "model_weights" in f else f
        found = {}
        root.visititems(lambda name, obj: found.__setitem__(name, np.asarray(obj)) if isinstance(obj, h5py.Dataset) else None)
    scoped = {}
    for name, arr in found.items():
        scoped.setdefault(name.split("/")[0], []).append((name, arr))
    rew = [a for _, a in scoped.get("simulator_reward", []) if a.ndim == 2]
    emb = [a for _, a in scoped.get("embedding", []) if a.ndim == 2]
    if len(rew) != 1 or len(emb) != 1:
        raise KeyError("%s: no single simulator_reward kernel / embedding table (layers %s)" % (path, sorted(scoped)))
    H, C = emb[0].shape[0], rew[0].shape[1]
    w = {}
    for name, scope, shape in dnn_plan(H, C):
        hits = [a for _, a in scoped.get(scope, []) if tuple(a.shape) == tuple(shape)]
        if len(hits) != 1:
            raise KeyError("%s: cannot resolve %s (layer %r, shape %s): %d candidates" % (path, name, scope, shape, len(hits)))
        w[name] = hits[0]
    return w


def load_behavior_weights(modelfile, name_map=None):
    """(W-table, H, C) of the behaviour net from a TF1 Saver prefix, an .npz keyed by W-table names, or a Keras .h5.  A
    file of another graph fails the plan's resolution."""
    path = str(modelfile)
    if tf_checkpoint.is_saver_prefix(path):
        rd = tf_checkpoint.TensorBundleReader(path)
        shapes = {k: tuple(sh) for k, (dt, sh) in rd.variables().items()}
        rew = [sh for k, sh in shapes.items() if k.split("/")[0] == "simulator_reward" and len(sh) == 2]
        emb = [sh for k, sh in shapes.items() if k.split("/")[0] == "embedding" and len(sh) == 2]
        if len(rew) != 1 or len(emb) != 1:
            raise KeyError("%s: no single simulator_reward kernel / embedding table: not the dnn behaviour net" % path)
        H, C = emb[0][0], rew[0][1]
        w = tf_checkpoint._load_by_plan(path, dnn_plan(H, C), tf_checkpoint.dnn_variable_names(
            dict(DNN_CFG, category_hash_size=H, class_num=C)), name_map)
    elif path.endswith(".h5"):
        w = _h5_table(path)
    else:
        with np.load(path) as z:
            w = {k: z[k] for k in z.files}
    return _check_table(w, path)


class behavior_model(object):
    """rl4rs/policy/behavior_model.py over the dnn graph.  config: the script's config (action_size, page_items,
    item_feature_size); modelfile: see load_behavior_weights.  action_probs returns f32 [B]."""

    def __init__(self, config, modelfile, device=None, use_kernels=None):
        self.config = dict(config)
        self.page_items = int(config.get("page_items", 9))
        self.item_feature_size = int(config.get("item_feature_size", 40))
        if not 1 <= self.page_items <= NCAT - NHEAD:
            raise ValueError("page_items %d: the behaviour net's 21 category slots hold 11 user ids and 1..10 items"
                             % self.page_items)
        w, self.H, self.C = load_behavior_weights(modelfile, config.get("variable_name_map"))
        A = int(config.get("action_size", 284))
        if self.C < A:
            raise ValueError("the behaviour net has %d classes, fewer than action_size %d" % (self.C, A))
        if self.C < 149:
            raise ValueError("the behaviour net has %d classes: action_probs' third slice y[:, 148:] needs at least 149"
                             % self.C)
        if device is None:
            device = "cuda" if torch.cuda.is_available() else "cpu"
        self.device = torch.device(device)
        self.use_kernels = (self.device.type == "cuda") if use_kernels is None else bool(use_kernels)
        names = [n for n, _, _ in dnn_plan(self.H, self.C)]
        self.flat = torch.from_numpy(np.concatenate([w[n].reshape(-1) for n in names])).to(self.device)
        self.w, o = {}, 0
        for n in names:                                   # views of the flat vector, in the kernels' order
            self.w[n] = self.flat[o:o + w[n].size].view(w[n].shape)
            o += w[n].size
        if self.use_kernels:
            self.lib = _capi.load_library()
            assert self.lib.r4_ope_num_params(self.H, self.C) == self.flat.numel()
        self._records, self._pages = None, {}

    # ---- inputs ------------------------------------------------------------------------------------
    def parse(self, records):
        """Records -> (head i32 [B, 11], items i32 [B, P K], feat f32 [B, P 5K]) as record2input + feature_extraction
        build them for every page: user_protrait[:10] and sequence_id as ints, the exposed items, and the first 5 of
        each item's item_feature_size features."""
        if len(records) and not isinstance(records[0], str):
            raise ValueError("behavior_model needs the record strings: the env's log holds row indices only (a log ingested "
                             "from arrays keeps no item_feature); ingest it from the text log")
        K, F = self.page_items, self.item_feature_size
        heads, items, feats = [], [], []
        for r in records:
            _, _, sequence_id, exposed, _, _, portrait, item_feature, _ = FeatureUtil.record_split(r)
            if len(exposed) % K or len(item_feature) != len(exposed) * F:
                raise ValueError("a record has %d exposed items and %d item features: expected whole pages of %d items "
                                 "and %d features per item" % (len(exposed), len(item_feature), K, F))
            heads.append([int(x) for x in portrait[:10]] + [sequence_id])
            items.append(exposed)
            feats.append(np.asarray(item_feature, dtype=np.float32).reshape(-1, F)[:, :NITEMF].reshape(-1))
        if len({len(h) for h in heads}) != 1 or len(heads[0]) != NHEAD or len({len(i) for i in items}) != 1:
            raise ValueError("the records must all have 10 portrait ids and the same number of pages")
        to = lambda x, dt: torch.as_tensor(np.asarray(x, dtype=dt), device=self.device)
        return to(heads, np.int32), to(items, np.int32), to(feats, np.float32)

    def _prepare(self, records):
        """Parse and upload the records once per reset (a new records object); forget the cached pages."""
        if records is not self._records:
            self._inputs = self.parse(records)
            self._records, self._pages = records, {}
            self.P = self._inputs[1].shape[1] // self.page_items

    def page_block(self, records, page):
        """The page's renormalised slices f32 [B, C - 1] on the device (column c - 1 = y[c] over its slice's sum),
        computed once per (reset, page)."""
        self._prepare(records)
        if not 0 <= page < self.P:
            raise ValueError("page %d: the records have %d pages" % (page, self.P))
        if page not in self._pages:
            self._pages[page] = self._forward_kernels(page) if self.use_kernels else self._forward_twin(page)
        return self._pages[page]

    # ---- the forward -------------------------------------------------------------------------------
    def _forward_kernels(self, page):
        head, items, feat = self._inputs
        B = head.shape[0]
        out = torch.empty(B, self.C - 1, dtype=torch.float32, device=self.device)
        scratch = torch.empty(self.lib.r4_ope_behavior_scratch_size(B, self.C), dtype=torch.float32, device=self.device)
        rc = self.lib.r4_ope_behavior(B, self.H, self.C, self.page_items, self.P, page, ptr(self.flat), ptr(head), ptr(items),
                                      ptr(feat), ptr(out), ptr(scratch), _capi.stream(self.device))
        _capi.check(self.lib, None, rc, "r4_ope_behavior")
        return out

    @torch.no_grad()
    def logits_twin(self, page):
        """The net's logits [B, C] for the page (torch)."""
        head, items, feat = self._inputs
        K, w, elu = self.page_items, self.w, torch.nn.functional.elu
        B = head.shape[0]
        ids = torch.zeros(B, NCAT, dtype=torch.int64, device=self.device)
        ids[:, :NHEAD] = head
        ids[:, NHEAD:NHEAD + K] = items[:, page * K:(page + 1) * K]
        cat = w["emb_cat"][ids.clamp(0, self.H - 1)].sum(1) / NCAT
        dense = torch.zeros(B, NDENSE, dtype=torch.float32, device=self.device)
        dense[:, :NITEMF * K] = feat[:, page * NITEMF * K:(page + 1) * NITEMF * K]
        x = elu(elu(dense @ w["dense_w1"] + w["dense_b1"]) @ w["dense_w2"] + w["dense_b2"])
        a = elu(torch.cat([cat, x], 1) @ w["fc_w"] + w["fc_b"])
        o = elu(a @ w["obs_w"] + w["obs_b"])
        return o @ w["rew_w"] + w["rew_b"]

    def _forward_twin(self, page):
        z = self.logits_twin(page)
        return slice_probs(z)

    # ---- the reference's surface -------------------------------------------------------------------
    def action_probs(self, records, action, layer, page=0):
        """behavior_model.action_probs: the behaviour probability of `action` [B] in the slice of `layer` -> f32 [B]."""
        block = self.page_block(records, page)
        a = torch.as_tensor(np.asarray(action), device=self.device).long().reshape(-1)
        if a.numel() != block.shape[0]:
            raise ValueError("%d actions for %d records" % (a.numel(), block.shape[0]))
        col = block_col(layer, a)
        if bool((col > block.shape[1] - 1).any()):          # checked on the host: no device-side index fault
            raise IndexError("an action beyond the behaviour net's %d classes (action_probs' slice of layer %d)"
                             % (self.C, layer))
        return block[torch.arange(block.shape[0], device=self.device), col].cpu().numpy()


def slice_probs(z):
    """k_ope_softmax in torch: softmax of logits z [B, C] (exp in f32, the sum in f64), each of y[1:40], y[40:148],
    y[148:] over its own f64 sum -> f32 [B, C - 1]."""
    e = torch.exp(z - z.max(1, keepdim=True).values)
    y = (e.double() / e.double().sum(1, keepdim=True)).float()[:, 1:].double()
    parts = [y[:, :39], y[:, 39:147], y[:, 147:]]
    return torch.cat([p / p.sum(1, keepdim=True) for p in parts], 1).float()


def block_col(layer, a):
    """The block column action_probs reads for `layer` (csrc/r4_ope.cuh block_col): the slice and the reference's clip."""
    if layer == 1:
        return (a - 1).clamp(0, 38)
    if layer == 2:
        return 39 + (a - 40).clamp(0, 107)
    return 147 + (a - 148).clamp(0, 233)


# ---- the per-step gather ---------------------------------------------------------------------------
class StepBuffers(object):
    """The five [T, B] columns an epoch fills, on the device where the step's inputs live: the policy's probability of
    the offline action, its behaviour probability, the policy's value at its own action (f32), the simulated and the
    offline reward (f64)."""

    def __init__(self, T, B, device, use_kernels):
        z = lambda dt: torch.zeros(T, B, dtype=dt, device=device)
        self.T, self.B, self.device = T, B, torch.device(device)
        self.pol, self.beh, self.val = z(torch.float32), z(torch.float32), z(torch.float32)
        self.rew, self.offr = z(torch.float64), z(torch.float64)
        self.use_kernels = use_kernels and self.device.type == "cuda"
        if self.use_kernels:
            self.lib = _capi.load_library()

    def gather(self, t, probs, logits, off, beh, layer, own, values, reward, off_reward):
        """Column t.  probs f32 [B, A] (logits: masked logits, softmaxed here); off i32 [B] the offline action; beh the
        page block f32 [B, C - 1] read at `layer`, or the behaviour probabilities f32 [B]; values f32 [B, A] read at own
        i32 [B], or f32 [B] (own None); reward, off_reward f64 [B]."""
        dev = self.device
        f32 = lambda x: torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x, device=dev).to(torch.float32).contiguous()
        i32 = lambda x: torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x, device=dev).to(torch.int32).reshape(-1).contiguous()
        f64 = lambda x: torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x, device=dev).to(torch.float64).reshape(-1).contiguous()
        probs, off, values, reward, off_reward = f32(probs), i32(off), f32(values), f64(reward), f64(off_reward)
        beh = f32(beh)
        own = i32(own) if own is not None else None
        self._check(t, probs, off, beh, own, values, reward, off_reward)
        B, A = probs.shape
        if self.use_kernels and beh.dim() == 2:
            rc = self.lib.r4_ope_step(t, self.T, B, A, beh.shape[1] + 1, layer, ptr(probs), int(bool(logits)), ptr(off),
                                      ptr(beh), ptr(own), ptr(values), int(own is not None), ptr(reward), ptr(off_reward),
                                      ptr(self.pol), ptr(self.beh), ptr(self.val), ptr(self.rew), ptr(self.offr),
                                      _capi.stream(dev))
            _capi.check(self.lib, None, rc, "r4_ope_step")
            return
        rows = torch.arange(B, device=dev)
        ok = (off >= 0) & (off < A)
        a = off.long().clamp(0, A - 1)
        if logits:
            e = torch.exp(probs - probs.max(1, keepdim=True).values)
            p = (e[rows, a].double() / e.double().sum(1)).float()
        else:
            p = probs[rows, a]
        nan = torch.tensor(float("nan"), device=dev)
        self.pol[t] = torch.where(ok, p, nan)
        self.beh[t] = torch.where(ok, beh[rows, block_col(layer, off.long()).clamp(max=beh.shape[1] - 1)], nan) \
            if beh.dim() == 2 else beh
        if own is not None:
            g = own.long()
            self.val[t] = torch.where((g >= 0) & (g < A), values[rows, g.clamp(0, A - 1)], nan)
        else:
            self.val[t] = values.reshape(-1)
        self.rew[t], self.offr[t] = reward, off_reward

    def _check(self, t, probs, off, beh, own, values, reward, off_reward):
        """Every input of column t must have the buffers' B rows (the kernel writes t B + b for each of its rows)."""
        B = self.B
        if not 0 <= t < self.T:
            raise ValueError("step %d of a %d-step episode" % (t, self.T))
        if probs.dim() != 2 or probs.shape[0] != B:
            raise ValueError("the policy gave %s probabilities for a batch of %d (config batch_size): the env's batch "
                             "must be batch_size" % (tuple(probs.shape), B))
        A = probs.shape[1]
        shapes = {"offline action": (off, (B,)), "offline reward": (off_reward, (B,)), "reward": (reward, (B,)),
                  "values": (values, (B, A) if own is not None else (B,))}
        if own is not None:
            shapes["own action"] = (own, (B,))
        for name, (x, want) in shapes.items():
            if tuple(x.shape) != want:
                raise ValueError("the step's %s has shape %s, expected %s (batch_size %d)" % (name, tuple(x.shape), want, B))
        if beh.shape[0] != B or beh.dim() not in (1, 2):
            raise ValueError("the behaviour probabilities have shape %s for a batch of %d" % (tuple(beh.shape), B))

    def host(self):
        """The five buffers as NumPy arrays [T, B] (one copy each)."""
        return [x.cpu().numpy() for x in (self.pol, self.beh, self.val, self.rew, self.offr)]


# ---- the policies --------------------------------------------------------------------------------
def _is_continuous(policy, config):
    from .policy import GaussianPolicy
    from .trainer import DDPGTrainer
    p = getattr(policy, "policy", policy)
    return bool(config.get("support_conti_env", False) or getattr(p, "continuous", False) or getattr(p, "conti", False)
                or isinstance(p, DDPGTrainer) or isinstance(getattr(p, "policy", None), GaussianPolicy))


def _step_inputs(policy, obs):
    """One step of the policy -> (env action, probs or logits [B, A], logits?, own action or None, values, value fix):
    policy_model's device fetch, or the reference's three calls (predict_with_mask, action_probs, predict_q) for any other
    object with that surface."""
    if hasattr(policy, "_ope_fetch"):
        return policy._ope_fetch(obs)
    action = policy.predict_with_mask(obs)
    return action, policy.action_probs(obs), False, None, policy.predict_q(obs, action), None


def _null_span(name):
    return contextlib.nullcontext()


def episode_products(p):
    """np.multiply.reduce(p * 100, axis=1) as offline_evaluation.py:47-48 forms it: in p's dtype, in step order."""
    return np.multiply.reduce(p * 100, axis=1)


def epoch_metrics(pol, beh, val, rew, offr):
    """offline_evaluation.py:39-71 on the copied [T, B] buffers -> (CIPS, DR, WIPS, SeqDR), each (value, half-width)."""
    episode_reward = np.sum(rew, axis=0)
    action_probs, behavior_probs = pol.swapaxes(0, 1), beh.swapaxes(0, 1)
    off_rewards = offr.swapaxes(0, 1)
    off_rewards_sum = np.sum(off_rewards, axis=1)
    rewards_hat, q_values = rew.swapaxes(0, 1), val.swapaxes(0, 1)
    apm, bpm = episode_products(action_probs), episode_products(behavior_probs)
    cips = OPE.eval_CIPS(off_rewards_sum, apm, bpm)
    dr = OPE.eval_doubly_robust(episode_reward, np.average(q_values, 1), off_rewards_sum, apm, bpm)
    wips = OPE.eval_WIPS(off_rewards, action_probs, behavior_probs)
    sdr = OPE.eval_seq_doubly_robust(rewards_hat, q_values, off_rewards, action_probs, behavior_probs)
    return cips, dr, wips, sdr


def ope_eval(config, eval_env, algo, sample_model=None, use_kernels=None, timer=None):
    """offline_evaluation.ope_eval: `epoch` episodes of max_steps steps at batch_size, the policy acting with its mask;
    with a sample_model, each epoch's CIPS, DR, WIPS and SeqDR.  Prints the reference's lines and returns the metrics
    [epoch, 4, 2].  use_kernels=False runs the torch gather on the CUDA env; timer(name) -> a context manager that times
    the named part of a step (tools/ope_time.py)."""
    policy = policy_model(algo, config)
    if _is_continuous(policy, config):
        raise NotImplementedError("ope: continuous-action policies are not evaluated (the reference indexes their "
                                  "probabilities with a continuous offline_action, offline_evaluation.py:27-28)")
    span = timer or _null_span
    metrics = []
    epoch, B, T = config["epoch"], config["batch_size"], config["max_steps"]
    page_items = config.get("page_items", 9)
    for i in range(epoch):
        with span("env"):
            obs = eval_env.reset()
        bufs = None
        print('test batch at ', i)
        for j in range(T):
            with span("act"):
                action, probs, logits, own, values, fix = _step_inputs(policy, obs)
            if sample_model is not None:
                with span("env"):
                    off_action = eval_env.offline_action                 # before the step (offline_evaluation.py:25)
                layer, page = j // 3 + 1, j // page_items
                if isinstance(sample_model, behavior_model):
                    with span("parse"):
                        sample_model._prepare(eval_env.samples.records)
                    with span("behavior"):
                        beh = sample_model.page_block(eval_env.samples.records, page)
                else:
                    beh = sample_model.action_probs(eval_env.samples.records, off_action, layer, page=page)
            with span("env"):
                obs, reward, done, info = eval_env.step(action)
                off_reward = eval_env.offline_reward                     # after the step (offline_evaluation.py:33-34)
            if sample_model is not None:
                with span("gather"):
                    if bufs is None:
                        dev = probs.device if torch.is_tensor(probs) else torch.device("cpu")
                        uk = dev.type == "cuda" if use_kernels is None else bool(use_kernels)
                        bufs = StepBuffers(T, B, dev, uk)
                    bufs.gather(j, probs, logits, off_action, beh, layer, own, values, reward, off_reward)
        if sample_model is not None:
            with span("estimators"):
                pol, bh, val, rew, offr = bufs.host()
                if fix is not None:
                    val = fix(val)
                metrics.append(epoch_metrics(pol, bh, val, rew, offr))
    out = np.array(metrics)
    print('IS', 'DR', 'WIPS', 'SeqDR', sep=' ')
    print(np.average(out, axis=0))
    print(np.std(out, axis=0))
    return out
