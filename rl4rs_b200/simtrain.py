"""Training the DIEN user simulator on the logged data: ``script/supervised_train.py <train> <test> <model_file> dien 0`` without
TensorFlow, from log text to the Saver checkpoint ``SlateRecEnv`` restores through ``config['model_file']``.

  item_samples(lines_or_path, config) -> ItemSamples   the samples of ``data_preprocess.py tfrecord_item`` (:91-131 with
                                                      ``FeatureUtil.feature_extraction``, datautil.py:34-69), kept per record
  get_model(config, 'dien')          -> SimulatorTrainer: fit / evaluate / weights / save / save_state / load_state
  supervised_train(train, test, model_file, model_type, is_slate_label)   the script, in its argument order

On a CUDA device one optimiser step is one library call (r4_simtrain_step: the forward with saved activations, the
backward, the weight and embedding gradients and Keras's Adam, csrc/r4_simtrain.cuh) and the samples stay on the device.
On the CPU the torch twin ``SimulatorNet`` runs the same algorithm.  The Keras / TF1 training semantics restated here are
listed in INTEGRATION.md section 8 as not verified (TensorFlow and deepctr are not in this project's environment).
"""
import ctypes as C
import math

import numpy as np
import torch

from . import synth
from .utils import tf_checkpoint
from .utils.datautil import FeatureUtil

NOT_BUILT = {"dnn": "the dnn simulator", "widedeep": "the widedeep simulator", "lstm": "the lstm simulator"}
# the fit schedule of supervised_train.py:38-42 and the Keras defaults it leaves (INTEGRATION.md section 8)
BATCH_SIZE = 256
STEPS_PER_EPOCH = 600000 // BATCH_SIZE
VALIDATION_STEPS = 400000 // BATCH_SIZE
EPOCHS = 20
PATIENCE = 3
DROPOUT = 0.2
ADAM = {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7}
CLIP = 1e-7
NUM_THRESHOLDS = 200
MAXLEN, SEQ_NUM, EMB, NCAT, NDENSE = 64, 2, 128, 21, 432
_FIXED = {"maxlen": MAXLEN, "seq_num": SEQ_NUM, "emb_size": EMB, "hidden_units": 128, "dense_feature_num": NDENSE,
          "category_feature_num": NCAT, "class_num": 2}


def _check_config(config):
    for k, v in _FIXED.items():
        if config.get(k, v) != v:
            raise ValueError("simulator training is built for %s = %r (got %r)" % (k, v, config[k]))
    return int(config.get("category_hash_size", 100000))


# ---- samples --------------------------------------------------------------------------------------------------------
class ItemSamples(object):
    """The item samples of a log, stored per page record (9 samples each).  Sample i is (record i // 9, item i % 9):
      cat   i32[21]     = user_cat (10) + [sequence_id] + items (9) + [items[j]]
      dense f32[432]    = user_dense (32) + item_feature (360) + item_feature[40 j : 40 j + 40]
      seq   i32[2, 64]  = seq[record]  (user_seqfeature | the earlier pages' items, pre-padded / pre-truncated)
      label             = feedback[record, j]"""

    FIELDS = ("user_cat", "user_dense", "sequence_id", "items", "feedback", "item_feature", "seq")

    def __init__(self, hash_size, **kw):
        self.hash_size = int(hash_size)
        for k in self.FIELDS:
            setattr(self, k, kw[k])

    @property
    def n_records(self):
        return self.items.shape[0]

    def __len__(self):
        return 9 * self.n_records

    def features(self, idx):
        """Samples idx -> (cat i32[n, 21], dense f32[n, 432], seq i32[n, 2, 64], label i64[n])."""
        idx = np.asarray(idx, dtype=np.int64)
        r, j = idx // 9, idx % 9
        cat = np.concatenate([self.user_cat[r], self.sequence_id[r, None], self.items[r], self.items[r, j][:, None]], 1)
        fj = self.item_feature.reshape(-1, 9, 40)[r, j]
        dense = np.concatenate([self.user_dense[r], self.item_feature[r], fj], 1)
        return (cat.astype(np.int32), dense.astype(np.float32), self.seq[r].astype(np.int32),
                self.feedback[r, j].astype(np.int64))

    def save(self, path):
        np.savez(path, hash_size=np.int64(self.hash_size), **{k: getattr(self, k) for k in self.FIELDS})

    @staticmethod
    def load(path):
        z = np.load(path)
        return ItemSamples(int(z["hash_size"]), **{k: z[k] for k in ItemSamples.FIELDS})


def _pad(ids, maxlen=MAXLEN):
    """keras pad_sequences: pre-pad with 0, keep the last maxlen ids."""
    out = np.zeros(maxlen, np.int64)
    ids = np.asarray(ids, dtype=np.int64)[-maxlen:]
    if len(ids):
        out[maxlen - len(ids):] = ids
    return out


def item_samples(lines_or_path, config):
    """Log text (path or list of page records, session-contiguous; header and empty lines skipped) -> ItemSamples, as
    ``data_preprocess.py tfrecord_item`` builds them (before its shuffle).  Every id must lie in [0, category_hash_size):
    anything else raises ValueError."""
    H = _check_config(config)
    if isinstance(lines_or_path, str):
        with open(lines_or_path, "r") as f:
            lines = f.read().split("\n")
    else:
        lines = list(lines_or_path)
    sessions, tmp, prev = [], [], None
    for record in lines:
        if len(record) < 1 or "timestamp" in record:
            continue
        sid = record.split("@")[1]
        if prev is not None and sid != prev:
            sessions.append(tmp)
            tmp = []
        tmp.append(record)
        prev = sid
    if tmp:
        sessions.append(tmp)
    cols = {k: [] for k in ItemSamples.FIELDS}
    for sess in sessions:
        fields = [FeatureUtil.record_split(r) for r in sess]
        for i, (_, _, sequence_id, items, feedback, useq, portrait, ifeat, _) in enumerate(fields):
            if sequence_id - 1 != i:
                raise AssertionError("session %s: record %d has sequence_id %d" % (sess[0].split("@")[1], i, sequence_id))
            if len(items) != 9 or len(feedback) != 9 or len(ifeat) != 360 or len(portrait) != 42:
                raise ValueError("record %r: expected 9 items / feedbacks, 360 item features and a 42-value portrait" % sess[i][:40])
            prev_items = [it for f in fields[:i] for it in f[3]] if i > 0 else [0]
            cols["user_cat"].append([int(x) for x in portrait[:10]])
            cols["user_dense"].append(portrait[10:])
            cols["sequence_id"].append(sequence_id)
            cols["items"].append(items)
            cols["feedback"].append(feedback)
            cols["item_feature"].append(ifeat)
            cols["seq"].append([_pad(useq), _pad(prev_items)])
    arr = {
        "user_cat": np.asarray(cols["user_cat"], np.int64).reshape(-1, 10),
        "user_dense": np.asarray(cols["user_dense"], np.float64).reshape(-1, 32).astype(np.float32),
        "sequence_id": np.asarray(cols["sequence_id"], np.int64).reshape(-1),
        "items": np.asarray(cols["items"], np.int64).reshape(-1, 9),
        "feedback": np.asarray(cols["feedback"], np.int64).reshape(-1, 9),
        "item_feature": np.asarray(cols["item_feature"], np.float64).reshape(-1, 360).astype(np.float32),
        "seq": np.asarray(cols["seq"], np.int64).reshape(-1, SEQ_NUM, MAXLEN),
    }
    for k in ("user_cat", "sequence_id", "items", "seq"):
        a = arr[k]
        if a.size and (a.min() < 0 or a.max() >= H):
            raise ValueError("%s holds ids outside [0, category_hash_size = %d): min %d, max %d" % (k, H, a.min(), a.max()))
        arr[k] = a.astype(np.int32)
    if arr["feedback"].size and (arr["feedback"].min() < 0 or arr["feedback"].max() > 1):
        raise ValueError("user_feedback must be 0 or 1")
    arr["feedback"] = arr["feedback"].astype(np.uint8)
    return ItemSamples(H, **arr)


def _load_samples(src, config):
    if isinstance(src, ItemSamples):
        return src
    if isinstance(src, str) and src.endswith(".npz"):
        s = ItemSamples.load(src)
        if s.hash_size > _check_config(config):
            raise ValueError("%s was built for category_hash_size %d > %d" % (src, s.hash_size, config["category_hash_size"]))
        return s
    return item_samples(src, config)


# ---- the torch twin -------------------------------------------------------------------------------------------------
def layer_plan(config):
    """[(W-table name, shape)] in the flat parameter order (tf_checkpoint.dien_layer_plan, the C-ABI's layout)."""
    return [(name, tuple(shape)) for name, _, shape in tf_checkpoint.dien_layer_plan(config)]


def flatten(weights, config):
    return np.concatenate([np.asarray(weights[k], np.float32).reshape(-1) for k, _ in layer_plan(config)])


def unflatten(flat, config):
    out, o = {}, 0
    for k, shape in layer_plan(config):
        n = int(np.prod(shape))
        out[k] = flat[o:o + n].reshape(shape)
        o += n
    return out


def keep_scale(keep, rate):
    """u8 keep bits [n, 256] (layer-major) -> the two layers' inverted-dropout scales, each [n, 128]."""
    k = keep.to(torch.float64) / (1.0 - rate)
    return k[:, :128], k[:, 128:]


class SimulatorNet(torch.nn.Module):
    """nets/dien.py in training mode over a flat parameter vector: the CPU path of the trainer and the autograd reference of
    the kernels.  forward(cat, dense, seq, keep, rate) -> (probs [n, 2], obs [n, 256]); keep (u8 [n, 256] or None: no dropout)."""

    def __init__(self, config, flat=None, dtype=torch.float32, seed=synth.WEIGHT_SEED):
        super().__init__()
        self.config = dict(config)
        if flat is None:
            flat = flatten(synth.make_weights(config, seed=seed), config)
        self.flat = torch.nn.Parameter(torch.as_tensor(np.asarray(flat)).to(dtype).clone())

    def tensors(self):
        return unflatten(self.flat, self.config)

    @staticmethod
    def _gru(x, wg, bg, wc, bc, scores=None):
        n, T, _ = x.shape
        Hd = wc.shape[1]
        h = x.new_zeros(n, Hd)
        outs = []
        for t in range(T):
            xt = x[:, t]
            g = torch.sigmoid(torch.cat([xt, h], 1) @ wg + bg)
            r, u = g[:, :Hd], g[:, Hd:]
            c = torch.tanh(torch.cat([xt, r * h], 1) @ wc + bc)
            if scores is not None:
                u = (1.0 - scores[:, t:t + 1]) * u
            h = u * h + (1.0 - u) * c
            outs.append(h)
        return torch.stack(outs, 1), h

    def forward(self, cat, dense, seq, keep=None, rate=DROPOUT):
        w = self.tensors()
        dt, dev = self.flat.dtype, self.flat.device

        def t(x, dtype):
            return (x if torch.is_tensor(x) else torch.as_tensor(np.asarray(x))).to(dev, dtype)
        cat, seq, dense = t(cat, torch.int64), t(seq, torch.int64), t(dense, dt)
        n = cat.shape[0]
        ec = w["emb_cat"][cat]
        p = torch.softmax(ec @ ec.transpose(1, 2), -1)
        c1 = (p @ ec).mean(1)
        x = torch.nn.functional.elu(dense @ w["dense_w1"] + w["dense_b1"])
        k0 = k1 = None
        if keep is not None:
            k0, k1 = keep_scale(t(keep, torch.uint8), rate)
            x = x * k0.to(dt)
        x = torch.nn.functional.elu(x @ w["dense_w2"] + w["dense_b2"])
        if keep is not None:
            x = x * k1.to(dt)
        q = w["emb_seq"][cat[:, -10:]].mean(1)
        hs = []
        for i in range(SEQ_NUM):
            xs = w["emb_seq"][seq[:, i]]
            H, _ = self._gru(xs, w["gru%d_wg" % i], w["gru%d_bg" % i], w["gru%d_wc" % i], w["gru%d_bc" % i])
            qq = q[:, None, :].expand_as(H)
            a = torch.cat([qq, H, qq - H, qq * H], -1)
            a = torch.sigmoid(a @ w["att%d_w1" % i] + w["att%d_b1" % i])
            a = torch.sigmoid(a @ w["att%d_w2" % i] + w["att%d_b2" % i])
            s = (a @ w["att%d_k" % i] + w["att%d_b" % i])[..., 0]
            _, h = self._gru(H, w["augru%d_wg" % i], w["augru%d_bg" % i], w["augru%d_wc" % i], w["augru%d_bc" % i], s)
            hs.append(h)
        allf = torch.cat(hs + [x, c1, ec.reshape(n, -1)], -1)
        obs = torch.nn.functional.elu(allf @ w["obs_w"] + w["obs_b"])
        probs = torch.softmax(obs @ w["rew_w"] + w["rew_b"], -1)
        return probs, obs


def keras_bce(probs, labels):
    """Keras binary_crossentropy of softmax probabilities against one_hot(labels, 2): p clipped to [1e-7, 1 - 1e-7] (zero
    gradient where clipped), the mean over both columns and the batch."""
    y = torch.nn.functional.one_hot(torch.as_tensor(labels, dtype=torch.int64, device=probs.device), 2).to(probs.dtype)
    pc = probs.clamp(CLIP, 1.0 - CLIP)
    return -(y * torch.log(pc) + (1.0 - y) * torch.log(1.0 - pc)).mean()


@torch.no_grad()
def keras_adam_(p, g, m, v, step, lr=ADAM["lr"], beta1=ADAM["beta1"], beta2=ADAM["beta2"], eps=ADAM["eps"]):
    """Keras OptimizerV2 Adam (ResourceApplyAdam) in place: m += (g - m)(1 - b1); v += (g^2 - v)(1 - b2);
    p -= lr sqrt(1 - b2^t) / (1 - b1^t) m / (sqrt(v) + eps)  -- eps outside the bias correction, unlike torch.optim.Adam."""
    alpha = lr * math.sqrt(1.0 - beta2 ** step) / (1.0 - beta1 ** step)
    m.add_((g - m) * (1.0 - beta1))
    v.add_((g * g - v) * (1.0 - beta2))
    p.sub_(alpha * m / (v.sqrt() + eps))


def auc_bins(p):
    """The number of Keras AUC thresholds (200: -1e-7, i / 199 for i = 1..198, 1 + 1e-7, as float32) each p exceeds."""
    thr = np.concatenate([[-1e-7], np.arange(1, NUM_THRESHOLDS - 1) / (NUM_THRESHOLDS - 1.0), [1.0 + 1e-7]]).astype(np.float32)
    p = np.asarray(p, np.float32).reshape(-1)
    return (p[:, None] > thr[None, :]).sum(1)


class Metrics(object):
    """Keras's epoch metrics: mean batch loss, binary accuracy at 0.5 over both columns, AUC (200 thresholds, ROC by the
    trapezoid rule) over the flattened one-hot columns -- from the f64[405] accumulator layout of r4_simtrain_grad."""

    def __init__(self):
        self.acc = np.zeros(3 + 2 * (NUM_THRESHOLDS + 1))

    def add(self, probs, labels, loss_rows):
        p = np.asarray(probs, np.float32)
        y = np.eye(2)[np.asarray(labels, np.int64)]
        self.acc[0] += float(np.sum(loss_rows))
        self.acc[1] += float(((p > 0.5).astype(np.float64) == y).mean(1).sum())
        self.acc[2] += p.shape[0]
        b = auc_bins(p)
        pos = y.reshape(-1) > 0
        self.acc[3:3 + NUM_THRESHOLDS + 1] += np.bincount(b[pos], minlength=NUM_THRESHOLDS + 1)
        self.acc[4 + NUM_THRESHOLDS:] += np.bincount(b[~pos], minlength=NUM_THRESHOLDS + 1)

    def result(self):
        a = self.acc
        nb = NUM_THRESHOLDS + 1
        pos, neg = a[3:3 + nb], a[3 + nb:]
        tp = np.array([pos[k + 1:].sum() for k in range(NUM_THRESHOLDS)])
        fp = np.array([neg[k + 1:].sum() for k in range(NUM_THRESHOLDS)])
        P, N = pos.sum(), neg.sum()
        tpr = tp / P if P > 0 else np.zeros_like(tp)
        fpr = fp / N if N > 0 else np.zeros_like(fp)
        auc = float(np.sum((fpr[:-1] - fpr[1:]) * (tpr[:-1] + tpr[1:]) / 2.0))
        n = max(a[2], 1.0)
        return {"loss": a[0] / n, "acc": a[1] / n, "auc": auc}


# ---- the trainer ----------------------------------------------------------------------------------------------------
def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class _Stream(object):
    """An endless stream of minibatches cut from consecutive seeded permutations of the sample set (tf.data's
    shuffle(10000).repeat() cannot be reproduced; INTEGRATION.md section 8)."""

    def __init__(self, n, batch, seed, device):
        self.n, self.batch, self.device = n, batch, device
        self.gen = torch.Generator(device=device)
        self.gen.manual_seed(int(seed))
        self.buf = torch.empty(0, dtype=torch.int64, device=device)

    def next(self):
        while self.buf.numel() < self.batch:
            self.buf = torch.cat([self.buf, torch.randperm(self.n, generator=self.gen, device=self.device)])
        out, self.buf = self.buf[:self.batch], self.buf[self.batch:]
        return out


class SimulatorTrainer(object):
    """The compiled `dien` simulator of supervised_train.py: Keras Adam (lr 1e-3), binary_crossentropy, dropout 0.2 in the
    dense tower, metrics AUC and acc.  device 'cuda[:k]' runs the kernels, 'cpu' the torch twin."""

    def __init__(self, config, device=None, seed=synth.WEIGHT_SEED, data_seed=0, weights=None):
        self.config = dict(config)
        self.H = _check_config(self.config)
        self.config["category_hash_size"] = self.H
        self.device = torch.device(device or ("cuda" if torch.cuda.is_available() else "cpu"))
        self.data_seed = int(data_seed)
        w = weights if weights is not None else synth.make_weights(self.config, seed=seed)
        flat = torch.from_numpy(flatten(w, self.config)).to(self.device)
        self.step = 0
        self.m = torch.zeros_like(flat)
        self.v = torch.zeros_like(flat)
        self._uploaded = {}
        if self.device.type == "cuda":
            from . import _capi
            self.lib = _capi.load_library()
            if self.lib.r4_simtrain_num_params(self.H) != flat.numel():
                raise ValueError("category_hash_size %d is outside the library's range" % self.H)
            self.params = flat
            self.grad = torch.zeros_like(flat)
            self.scratch, self.scratch_n = None, 0
            self.acc = torch.zeros(3 + 2 * (NUM_THRESHOLDS + 1), dtype=torch.float64, device=self.device)
            self.stats = torch.zeros(2, dtype=torch.float32, device=self.device)
        else:
            self.net = SimulatorNet(self.config, flat.numpy(), torch.float32)

    # -- parameters --
    def flat_params(self):
        return (self.params if self.device.type == "cuda" else self.net.flat.data).detach()

    def weights(self):
        """The W-table {name: float32 array} (what save_dien_checkpoint writes and the env loads)."""
        flat = self.flat_params().cpu().numpy()
        return {k: np.array(v) for k, v in unflatten(flat, self.config).items()}

    def save(self, model_file):
        """A TF1 Saver-format checkpoint at the prefix model_file (SlateRecEnv's config['model_file'])."""
        return tf_checkpoint.save_dien_checkpoint(model_file, self.weights(), self.config)

    def save_state(self, path):
        np.savez(path, params=self.flat_params().cpu().numpy(), m=self.m.cpu().numpy(), v=self.v.cpu().numpy(),
                 step=np.int64(self.step), hash_size=np.int64(self.H))

    def load_state(self, path):
        z = np.load(path)
        if int(z["hash_size"]) != self.H:
            raise ValueError("state was saved at category_hash_size %d, not %d" % (int(z["hash_size"]), self.H))
        self.flat_params().copy_(torch.from_numpy(z["params"]))
        self.m.copy_(torch.from_numpy(z["m"]))
        self.v.copy_(torch.from_numpy(z["v"]))
        self.step = int(z["step"])

    # -- device data --
    def _data(self, samples):
        key = id(samples)
        if key not in self._uploaded:
            if samples.hash_size > self.H:
                raise ValueError("samples were checked against category_hash_size %d > %d" % (samples.hash_size, self.H))
            from . import _capi
            ts = [torch.from_numpy(np.ascontiguousarray(getattr(samples, k))).to(self.device) for k in ItemSamples.FIELDS]
            self._uploaded[key] = (samples, ts, _capi.SimTrainData(*[t.data_ptr() for t in ts]))
        return self._uploaded[key][2]

    def _scratch(self, n):
        if self.scratch is None or self.scratch_n < n:
            size = self.lib.r4_simtrain_scratch_size(n)
            if size < 0:
                raise ValueError("batch size %d is outside 1..4096" % n)
            self.scratch = torch.empty(size, dtype=torch.uint8, device=self.device)
            self.scratch_n = n
        return self.scratch

    def _check(self, rc, what):
        from . import _capi
        _capi.check(self.lib, None, rc, what)

    # -- one step / one evaluation batch --
    def train_step(self, samples, idx, counter=None, rate=DROPOUT, metrics=None):
        """One Adam step on the samples idx (int64, on the trainer's device).  The dropout draw is keyed by (data_seed,
        counter = the step by default)."""
        self.step += 1
        counter = self.step if counter is None else counter
        n = int(idx.numel())
        if self.device.type == "cuda":
            d = self._data(samples)
            rc = self.lib.r4_simtrain_step(self.H, _p(self.params), _p(self.grad), _p(self.m), _p(self.v), C.byref(d), _p(idx), n,
                                           self.data_seed, counter, rate, self.step, ADAM["lr"], ADAM["beta1"], ADAM["beta2"],
                                           ADAM["eps"], _p(self._scratch(n)), _p(self.stats), _p(self.acc),
                                           C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
            self._check(rc, "r4_simtrain_step")
            return
        cat, dense, seq, y = samples.features(idx.numpy())
        gen = torch.Generator().manual_seed(self.data_seed * 1000003 + counter)
        keep = (torch.rand(n, 256, generator=gen) >= rate).to(torch.uint8) if rate > 0 else None
        probs, _ = self.net(cat, dense, seq, keep, rate)
        loss = keras_bce(probs, y)
        self.net.flat.grad = None
        loss.backward()
        keras_adam_(self.net.flat.data, self.net.flat.grad, self.m, self.v, self.step)
        if metrics is not None:
            p = probs.detach().numpy()
            metrics.add(p, y, _bce_rows(p, y))

    def eval_batch(self, samples, idx, metrics=None):
        """probs f32[n, 2] of the samples idx without dropout (accumulating the metrics on the CUDA path into self.acc)."""
        n = int(idx.numel())
        if self.device.type == "cuda":
            d = self._data(samples)
            probs = torch.empty(n, 2, dtype=torch.float32, device=self.device)
            rc = self.lib.r4_simtrain_eval(self.H, _p(self.params), C.byref(d), _p(idx), n, _p(self._scratch(n)), _p(probs),
                                           _p(self.acc), C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
            self._check(rc, "r4_simtrain_eval")
            return probs
        cat, dense, seq, y = samples.features(idx.numpy())
        with torch.no_grad():
            probs, _ = self.net(cat, dense, seq, None)
        p = probs.numpy()
        if metrics is not None:
            metrics.add(p, y, _bce_rows(p, y))
        return probs

    def _run(self, fn, samples, stream, steps):
        m = Metrics()
        if self.device.type == "cuda":
            self.acc.zero_()
            for _ in range(steps):
                fn(samples, stream.next())
            m.acc = self.acc.cpu().numpy()
        else:
            for _ in range(steps):
                fn(samples, stream.next(), metrics=m)
        return m.result()

    def evaluate(self, samples, steps=None, batch_size=BATCH_SIZE):
        """Loss / acc / AUC over the samples in order (steps batches, default: all whole batches and the remainder)."""
        samples = _load_samples(samples, self.config)
        n = len(samples)
        m = Metrics()
        if self.device.type == "cuda":
            self.acc.zero_()
        nb = steps if steps is not None else (n + batch_size - 1) // batch_size
        for b in range(nb):
            idx = torch.arange(b * batch_size, min(n, (b + 1) * batch_size), device=self.device)
            if idx.numel():
                self.eval_batch(samples, idx, metrics=m)
        if self.device.type == "cuda":
            m.acc = self.acc.cpu().numpy()
        return m.result()

    def fit(self, train, test, epochs=EPOCHS, steps_per_epoch=STEPS_PER_EPOCH, validation_steps=VALIDATION_STEPS,
            patience=PATIENCE, batch_size=BATCH_SIZE, verbose=0):
        """Keras fit with EarlyStopping(val_loss, patience, mode='min') that keeps the last epoch's weights.  Returns the
        history {loss, auc, acc, val_loss, val_auc, val_acc}: one entry per epoch run."""
        train = _load_samples(train, self.config)
        test = _load_samples(test, self.config)
        dev = self.device if self.device.type == "cuda" else torch.device("cpu")
        key = (len(train), len(test), batch_size)
        if getattr(self, "_streams", (None,))[0] != key:          # a later fit on the same sets continues their streams
            self._streams = (key, _Stream(len(train), batch_size, self.data_seed, dev),
                             _Stream(len(test), batch_size, self.data_seed + 1, dev))
        _, tr, va = self._streams
        hist = {k: [] for k in ("loss", "auc", "acc", "val_loss", "val_auc", "val_acc")}
        best, wait = math.inf, 0
        for ep in range(epochs):
            r = self._run(self.train_step, train, tr, steps_per_epoch)
            rv = self._run(self.eval_batch, test, va, validation_steps)
            for k in ("loss", "auc", "acc"):
                hist[k].append(r[k])
                hist["val_" + k].append(rv[k])
            if verbose:
                print("epoch %d: loss %.4f auc %.4f acc %.4f val_loss %.4f val_auc %.4f val_acc %.4f"
                      % (ep + 1, r["loss"], r["auc"], r["acc"], rv["loss"], rv["auc"], rv["acc"]))
            if rv["loss"] < best:
                best, wait = rv["loss"], 0
            else:
                wait += 1
                if wait >= patience:
                    break
        return hist


def _bce_rows(p, y):
    p = np.clip(np.asarray(p, np.float64), CLIP, 1.0 - CLIP)
    yy = np.eye(2)[np.asarray(y, np.int64)]
    return -(yy * np.log(p) + (1.0 - yy) * np.log(1.0 - p)).mean(1)


def get_model(config, model_type="dien", **kw):
    """rl4rs.nets.<model_type>.get_model for training: only 'dien' is built."""
    if model_type in NOT_BUILT:
        raise NotImplementedError("%s: training %s is not built in this project" % (model_type, NOT_BUILT[model_type]))
    if model_type != "dien":
        raise NotImplementedError("%s: training the slate-label and other nets is not built in this project" % model_type)
    return SimulatorTrainer(config, **kw)


def supervised_train(train_file, test_file, model_file, model_type="dien", is_slate_label=0, config=None, device=None,
                     verbose=2, **fit_kw):
    """script/supervised_train.py in its argument order.  train_file / test_file: log text (path or lines) or an ItemSamples
    .npz, where the script took TFRecords.  Trains, saves the Saver checkpoint at model_file and returns (trainer, history)."""
    if int(is_slate_label):
        raise NotImplementedError("is_slate_label = 1: training the slate-label nets is not built in this project")
    cfg = {"epoch": EPOCHS, "maxlen": 64, "batch_size": BATCH_SIZE, "class_num": 2, "dense_feature_num": 432,
           "category_feature_num": 21, "category_hash_size": 100000, "seq_num": 2, "emb_size": 128, "hidden_units": 128,
           "action_size": 284}
    cfg.update(config or {})
    model = get_model(cfg, model_type, device=device)
    train, test = _load_samples(train_file, cfg), _load_samples(test_file, cfg)
    fit_kw.setdefault("epochs", int(cfg["epoch"]))
    fit_kw.setdefault("batch_size", int(cfg["batch_size"]))
    hist = model.fit(train, test, verbose=verbose, **fit_kw)
    model.save(model_file)
    return model, hist
