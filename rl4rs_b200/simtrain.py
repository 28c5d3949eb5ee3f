"""Training the DIEN user simulator on the logged data: ``script/supervised_train.py <train> <test> <model_file> dien 0`` without
TensorFlow, from log text to the Saver checkpoint ``SlateRecEnv`` restores through ``config['model_file']``; and the
slate-label nets on the same backbone, ``supervised_train.py ... dien_slate 1`` / ``dien_slate_multiclass 1``.

  item_samples(lines_or_path, config) -> ItemSamples   the samples of ``data_preprocess.py tfrecord_item`` (:91-131 with
                                                      ``FeatureUtil.feature_extraction``, datautil.py:34-69), kept per record
  slate_samples(lines_or_path, config) -> SlateSamples the samples of ``tfrecord_slate``: one per record, the same store
  get_model(config, 'dien' | 'dien_slate' | 'dien_slate_multiclass') -> SimulatorTrainer: fit / evaluate / weights / save /
                                                      save_state / load_state
  supervised_train(train, test, model_file, model_type, is_slate_label)   the script, in its argument order

On a CUDA device one optimiser step is one library call (r4_simtrain_head_step: the forward with saved activations, the
backward, the weight and embedding gradients and Keras's Adam, csrc/r4_simtrain.cuh) and the samples stay on the device.
On the CPU the torch twin ``SimulatorNet`` runs the same algorithm.  The Keras / TF1 training semantics restated here are
listed in INTEGRATION.md section 8 as not verified (TensorFlow and deepctr are not in this project's environment).
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _capi, synth
from ._capi import ptr
from .utils import tf_checkpoint
from .utils.datautil import FeatureUtil

NOT_BUILT = {"dnn": "the dnn simulator", "widedeep": "the widedeep simulator", "lstm": "the lstm simulator"}
# the nets get_model trains -> the library's head (R4_SIMHEAD_*): nets/dien.py, dien_slate.py, dien_slate_multiclass.py
HEADS = {"dien": 0, "dien_slate": 1, "dien_slate_multiclass": 2}
CLASSES = (2, 9, 22)                       # simulator_reward's width per head
HISTORY = (("loss", "auc", "acc"), ("loss", "auc", "precision", "recall"), ("loss", "acc"))
# the slate-label nets whose backbones (dnn, widedeep, lstm) or training (adversarial) are not built
NOT_BUILT_SLATE = ("dnn_slate", "dnn_slate_multiclass", "widedeep_slate", "widedeep_slate_multiclass", "lstm_slate",
                   "lstm_slate_multiclass", "adversarial_slate")
# dien_slate_multiclass.py:8-11: the class of a page's click pattern y[9] is y . SLATE2LABEL (0..21)
SLATE2LABEL = np.array([1, 2, 4, 1, 2, 4, 1, 2, 4], np.int64)
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


def _check_config(config, head=0):
    for k, v in _FIXED.items():
        if k == "class_num" and head:                  # the slate nets fix their own width (dien_slate.py:37)
            continue
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

    @classmethod
    def load(cls, path):
        z = np.load(path)
        return cls(int(z["hash_size"]), **{k: z[k] for k in ItemSamples.FIELDS})

    @classmethod
    def view(cls, samples):
        """The same per-record store seen as cls's samples (no copy)."""
        return samples if type(samples) is cls else cls(samples.hash_size, **{k: getattr(samples, k) for k in ItemSamples.FIELDS})


class SlateSamples(ItemSamples):
    """The slate samples of a log (``data_preprocess.py tfrecord_slate`` with ``feature_extraction``): one per page record,
    over the same store as ItemSamples.  Sample i is record i:
      cat   i32[21]     = user_cat (10) + [sequence_id] + items (9) + [0]   (pad_sequences post-padding to 21)
      dense f32[432]    = user_dense (32) + item_feature (360) + 40 zeros   (post-padding to 432)
      seq   i32[2, 64]  = seq[record]
      label u8[9]       = feedback[record]"""

    def __len__(self):
        return self.n_records

    def features(self, idx):
        """Samples idx -> (cat i32[n, 21], dense f32[n, 432], seq i32[n, 2, 64], label u8[n, 9])."""
        r = np.asarray(idx, dtype=np.int64)
        n = len(r)
        cat = np.concatenate([self.user_cat[r], self.sequence_id[r, None], self.items[r], np.zeros((n, 1), np.int64)], 1)
        dense = np.concatenate([self.user_dense[r], self.item_feature[r], np.zeros((n, 40), np.float32)], 1)
        return (cat.astype(np.int32), dense.astype(np.float32), self.seq[r].astype(np.int32),
                self.feedback[r].astype(np.uint8))


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


def slate_samples(lines_or_path, config):
    """Log text -> SlateSamples, as ``data_preprocess.py tfrecord_slate`` builds them (before its shuffle); the ids are
    checked as item_samples checks them."""
    return SlateSamples.view(item_samples(lines_or_path, dict(config, class_num=2)))


def _load_samples(src, config, head=0):
    cls = SlateSamples if head else ItemSamples
    if isinstance(src, ItemSamples):
        return cls.view(src)
    if isinstance(src, str) and src.endswith(".npz"):
        s = cls.load(src)
        if s.hash_size > _check_config(config, head):
            raise ValueError("%s was built for category_hash_size %d > %d" % (src, s.hash_size, config["category_hash_size"]))
        return s
    return slate_samples(src, config) if head else item_samples(src, config)


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


def head_weights(config, head=0, seed=synth.WEIGHT_SEED, **kw):
    """synth.make_weights for a head: the dien W-table, with simulator_reward [256, C] + [C] drawn as Keras initialises a
    Dense kernel (Glorot uniform) and bias (zeros) for the slate heads; stress / bias_noise apply to it as to the others."""
    w = synth.make_weights(dict(config, class_num=2), seed=seed, **kw)
    if head:
        C = CLASSES[head]
        rs = np.random.RandomState(int(seed) * 7 + head)
        lim = math.sqrt(6.0 / (256 + C))
        w["rew_w"] = (rs.uniform(-lim, lim, (256, C)) * kw.get("stress", 1.0)).astype(np.float32)
        w["rew_b"] = rs.normal(0.0, kw.get("bias_noise", 0.0), C).astype(np.float32) if kw.get("bias_noise") else np.zeros(C, np.float32)
    return w


def keep_scale(keep, rate):
    """u8 keep bits [n, 256] (layer-major) -> the two layers' inverted-dropout scales, each [n, 128]."""
    k = keep.to(torch.float64) / (1.0 - rate)
    return k[:, :128], k[:, 128:]


class SimulatorNet(torch.nn.Module):
    """nets/dien.py in training mode over a flat parameter vector: the CPU path of the trainer and the autograd reference of
    the kernels.  forward(cat, dense, seq, keep, rate) -> (probs [n, C], obs [n, 256]); keep (u8 [n, 256] or None: no dropout).
    head (HEADS) picks the output: 0 softmax over 2 (dien.py), 1 sigmoid over 9 (dien_slate.py), 2 softmax over 22
    (dien_slate_multiclass.py); logits(...) -> (z [n, C], obs) is the forward before that activation."""

    def __init__(self, config, flat=None, dtype=torch.float32, seed=synth.WEIGHT_SEED, head=0):
        super().__init__()
        self.config = dict(config, class_num=CLASSES[head]) if head else dict(config)
        self.head = int(head)
        if flat is None:
            flat = flatten(head_weights(self.config, self.head, seed=seed), self.config)
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
        z, obs = self.logits(cat, dense, seq, keep, rate)
        return (torch.sigmoid(z) if self.head == 1 else torch.softmax(z, -1)), obs

    def logits(self, cat, dense, seq, keep=None, rate=DROPOUT):
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
        return obs @ w["rew_w"] + w["rew_b"], obs


def keras_bce(probs, labels):
    """Keras binary_crossentropy of softmax probabilities against one_hot(labels, 2): p clipped to [1e-7, 1 - 1e-7] (zero
    gradient where clipped), the mean over both columns and the batch."""
    y = torch.nn.functional.one_hot(torch.as_tensor(labels, dtype=torch.int64, device=probs.device), 2).to(probs.dtype)
    pc = probs.clamp(CLIP, 1.0 - CLIP)
    return -(y * torch.log(pc) + (1.0 - y) * torch.log(1.0 - pc)).mean()


def slate2label(labels):
    """The click pattern's class of each page: labels [n, 9] . [1, 2, 4, 1, 2, 4, 1, 2, 4] (dien_slate_multiclass.py:8-11)."""
    return np.asarray(labels, np.int64) @ SLATE2LABEL


def slate_bce_rows(logits, labels):
    """dien_slate's binary_crossentropy per sample from the logits of its Sigmoid output (no clip): the mean over the 9
    columns of max(z, 0) - z y + log(1 + exp(-|z|))."""
    y = torch.as_tensor(np.asarray(labels), device=logits.device).to(logits.dtype)
    return torch.nn.functional.binary_cross_entropy_with_logits(logits, y, reduction="none").mean(1)


def slate_cce_rows(logits, labels):
    """dien_slate_multiclass's my_loss_fn per sample from the logits of its Softmax output (no clip): categorical
    cross-entropy against one_hot(slate2label(labels), 22)."""
    cls = torch.as_tensor(slate2label(labels), device=logits.device)
    return torch.nn.functional.cross_entropy(logits, cls, reduction="none")


def loss_rows(head, logits, labels):
    """The per-sample loss of a slate head (1, 2) from its logits; the batch loss is their mean."""
    return slate_bce_rows(logits, labels) if head == 1 else slate_cce_rows(logits, labels)


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


def _auc(pos, neg):
    """Keras AUC (ROC, trapezoid rule over the 200 thresholds) from the positives' and negatives' bin counts."""
    tp = np.array([pos[k + 1:].sum() for k in range(NUM_THRESHOLDS)])
    fp = np.array([neg[k + 1:].sum() for k in range(NUM_THRESHOLDS)])
    P, N = pos.sum(), neg.sum()
    tpr = tp / P if P > 0 else np.zeros_like(tp)
    fpr = fp / N if N > 0 else np.zeros_like(fp)
    return float(np.sum((fpr[:-1] - fpr[1:]) * (tpr[:-1] + tpr[1:]) / 2.0))


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
        n = max(a[2], 1.0)
        return {"loss": a[0] / n, "acc": a[1] / n, "auc": _auc(a[3:3 + nb], a[3 + nb:])}


class SlateMetrics(object):
    """dien_slate's epoch metrics: mean batch loss, AUC() over all 9 columns, Precision() and Recall() at p > 0.5 (0 when
    nothing is predicted / labelled positive, as Keras's div_no_nan) -- from the f64[408] accumulator of the slate head:
    {loss sum, binary accuracy sum, samples, positives[201], negatives[201], TP, FP, FN}."""

    SIZE = 3 + 2 * (NUM_THRESHOLDS + 1) + 3

    def __init__(self):
        self.acc = np.zeros(self.SIZE)

    def add(self, probs, labels, loss_rows):
        p = np.asarray(probs, np.float32)
        y = np.asarray(labels, np.int64) != 0
        pos = p > 0.5
        nb = NUM_THRESHOLDS + 1
        self.acc[0] += float(np.sum(loss_rows))
        self.acc[1] += float((pos == y).mean(1).sum())
        self.acc[2] += p.shape[0]
        b = auc_bins(p)
        self.acc[3:3 + nb] += np.bincount(b[y.reshape(-1)], minlength=nb)
        self.acc[3 + nb:3 + 2 * nb] += np.bincount(b[~y.reshape(-1)], minlength=nb)
        self.acc[-3:] += [np.sum(pos & y), np.sum(pos & ~y), np.sum(~pos & y)]

    def result(self):
        a, nb = self.acc, NUM_THRESHOLDS + 1
        tp, fp, fn = a[-3:]
        n = max(a[2], 1.0)
        return {"loss": a[0] / n, "auc": _auc(a[3:3 + nb], a[3 + nb:3 + 2 * nb]),
                "precision": tp / (tp + fp) if tp + fp > 0 else 0.0, "recall": tp / (tp + fn) if tp + fn > 0 else 0.0}


class MulticlassMetrics(object):
    """dien_slate_multiclass's epoch metrics: mean batch loss and my_acc_metrics (categorical accuracy: the first argmax of
    p at the click pattern's class) -- from the f64[3] accumulator {loss sum, hits, samples}."""

    SIZE = 3

    def __init__(self):
        self.acc = np.zeros(self.SIZE)

    def add(self, probs, labels, loss_rows):
        p = np.asarray(probs, np.float32)
        self.acc += [float(np.sum(loss_rows)), float(np.sum(np.argmax(p, 1) == slate2label(labels))), p.shape[0]]

    def result(self):
        n = max(self.acc[2], 1.0)
        return {"loss": self.acc[0] / n, "acc": self.acc[1] / n}


METRICS = (Metrics, SlateMetrics, MulticlassMetrics)


# ---- the trainer ----------------------------------------------------------------------------------------------------
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
    dense tower, metrics AUC and acc.  device 'cuda[:k]' runs the kernels, 'cpu' the torch twin.  head 1 / 2 (HEADS) is the
    compiled dien_slate / dien_slate_multiclass on SlateSamples: the same backbone and Adam, their own head, loss and
    metrics (HISTORY)."""

    def __init__(self, config, device=None, seed=synth.WEIGHT_SEED, data_seed=0, weights=None, head=0):
        if head not in (0, 1, 2):
            raise ValueError("head must be 0 (dien), 1 (dien_slate) or 2 (dien_slate_multiclass), not %r" % (head,))
        self.head = int(head)
        self.config = dict(config, class_num=CLASSES[head]) if head else dict(config)
        self.H = _check_config(self.config, self.head)
        self.config["category_hash_size"] = self.H
        self.device = torch.device(device or ("cuda" if torch.cuda.is_available() else "cpu"))
        self.data_seed = int(data_seed)
        w = weights if weights is not None else head_weights(self.config, self.head, seed=seed)
        flat = torch.from_numpy(flatten(w, self.config)).to(self.device)
        if self.head and flat.numel() != sum(int(np.prod(s)) for _, s in layer_plan(self.config)):
            raise ValueError("the weights do not fit the %d-wide head" % CLASSES[head])
        self.step = 0
        self.m = torch.zeros_like(flat)
        self.v = torch.zeros_like(flat)
        self._uploaded = {}
        if self.device.type == "cuda":
            self.lib = _capi.load_library()
            if self.lib.r4_simtrain_head_num_params(self.head, self.H) != flat.numel():
                raise ValueError("category_hash_size %d is outside the library's range" % self.H)
            self.params = flat
            self.grad = torch.zeros_like(flat)
            self.scratch, self.scratch_n = None, 0
            self.acc = torch.zeros(METRICS[self.head].SIZE if self.head else 3 + 2 * (NUM_THRESHOLDS + 1), dtype=torch.float64,
                                   device=self.device)
            self.stats = torch.zeros(2, dtype=torch.float32, device=self.device)
        else:
            self.net = SimulatorNet(self.config, flat.numpy(), torch.float32, head=self.head)

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
                 step=np.int64(self.step), hash_size=np.int64(self.H), **({"head": np.int64(self.head)} if self.head else {}))

    def load_state(self, path):
        z = np.load(path)
        if int(z["hash_size"]) != self.H:
            raise ValueError("state was saved at category_hash_size %d, not %d" % (int(z["hash_size"]), self.H))
        head = int(z["head"]) if "head" in z else 0
        if head != self.head:
            raise ValueError("state was saved for head %d, not %d" % (head, self.head))
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
            ts = [torch.from_numpy(np.ascontiguousarray(getattr(samples, k))).to(self.device) for k in ItemSamples.FIELDS]
            self._uploaded[key] = (samples, ts, _capi.SimTrainData(*[t.data_ptr() for t in ts]))
        return self._uploaded[key][2]

    def _scratch(self, n):
        if self.scratch is None or self.scratch_n < n:
            size = self.lib.r4_simtrain_head_scratch_size(self.head, n)
            if size < 0:
                raise ValueError("batch size %d is outside 1..4096" % n)
            self.scratch = torch.empty(size, dtype=torch.uint8, device=self.device)
            self.scratch_n = n
        return self.scratch

    def _check(self, rc, what):
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
            rc = self.lib.r4_simtrain_head_step(self.head, self.H, ptr(self.params), ptr(self.grad), ptr(self.m), ptr(self.v),
                                                C.byref(d), ptr(idx), n, self.data_seed, counter, rate, self.step, ADAM["lr"],
                                                ADAM["beta1"], ADAM["beta2"], ADAM["eps"], ptr(self._scratch(n)), ptr(self.stats),
                                                ptr(self.acc), _capi.stream(self.device))
            self._check(rc, "r4_simtrain_step")
            return
        cat, dense, seq, y = samples.features(idx.numpy())
        gen = torch.Generator().manual_seed(self.data_seed * 1000003 + counter)
        keep = (torch.rand(n, 256, generator=gen) >= rate).to(torch.uint8) if rate > 0 else None
        if self.head:
            z, _ = self.net.logits(cat, dense, seq, keep, rate)
            rows = loss_rows(self.head, z, y)
            self.net.flat.grad = None
            rows.mean().backward()
            keras_adam_(self.net.flat.data, self.net.flat.grad, self.m, self.v, self.step)
            if metrics is not None:
                metrics.add(self._activate(z).detach().numpy(), y, rows.detach().numpy())
            return
        probs, _ = self.net(cat, dense, seq, keep, rate)
        loss = keras_bce(probs, y)
        self.net.flat.grad = None
        loss.backward()
        keras_adam_(self.net.flat.data, self.net.flat.grad, self.m, self.v, self.step)
        if metrics is not None:
            p = probs.detach().numpy()
            metrics.add(p, y, _bce_rows(p, y))

    def _activate(self, z):
        return torch.sigmoid(z) if self.head == 1 else torch.softmax(z, -1)

    def eval_batch(self, samples, idx, metrics=None):
        """probs f32[n, C] of the samples idx without dropout (accumulating the metrics on the CUDA path into self.acc)."""
        n = int(idx.numel())
        if self.device.type == "cuda":
            d = self._data(samples)
            probs = torch.empty(n, CLASSES[self.head], dtype=torch.float32, device=self.device)
            rc = self.lib.r4_simtrain_head_eval(self.head, self.H, ptr(self.params), C.byref(d), ptr(idx), n, ptr(self._scratch(n)),
                                                ptr(probs), ptr(self.acc), _capi.stream(self.device))
            self._check(rc, "r4_simtrain_eval")
            return probs
        cat, dense, seq, y = samples.features(idx.numpy())
        if self.head:
            with torch.no_grad():
                z, _ = self.net.logits(cat, dense, seq, None)
                probs = self._activate(z)
            if metrics is not None:
                metrics.add(probs.numpy(), y, loss_rows(self.head, z, y).numpy())
            return probs
        with torch.no_grad():
            probs, _ = self.net(cat, dense, seq, None)
        p = probs.numpy()
        if metrics is not None:
            metrics.add(p, y, _bce_rows(p, y))
        return probs

    def _run(self, fn, samples, stream, steps):
        m = METRICS[self.head]()
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
        """The head's metrics (HISTORY: loss / acc / AUC for dien) over the samples in order (steps batches, default: all
        whole batches and the remainder)."""
        samples = _load_samples(samples, self.config, self.head)
        n = len(samples)
        m = METRICS[self.head]()
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
        history {loss, auc, acc, val_loss, val_auc, val_acc} (the slate heads: HISTORY[head] and their val_): one entry per
        epoch run."""
        train = _load_samples(train, self.config, self.head)
        test = _load_samples(test, self.config, self.head)
        dev = self.device if self.device.type == "cuda" else torch.device("cpu")
        key = (len(train), len(test), batch_size)
        if getattr(self, "_streams", (None,))[0] != key:          # a later fit on the same sets continues their streams
            self._streams = (key, _Stream(len(train), batch_size, self.data_seed, dev),
                             _Stream(len(test), batch_size, self.data_seed + 1, dev))
        _, tr, va = self._streams
        keys = HISTORY[self.head]
        hist = {k: [] for k in keys + tuple("val_" + k for k in keys)}
        best, wait = math.inf, 0
        for ep in range(epochs):
            r = self._run(self.train_step, train, tr, steps_per_epoch)
            rv = self._run(self.eval_batch, test, va, validation_steps)
            for k in keys:
                hist[k].append(r[k])
                hist["val_" + k].append(rv[k])
            if verbose:
                print("epoch %d: " % (ep + 1) + " ".join(["%s %.4f" % (k, r[k]) for k in keys] +
                                                         ["val_%s %.4f" % (k, rv[k]) for k in keys]))
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
    """rl4rs.nets.<model_type>.get_model for training: 'dien', 'dien_slate' and 'dien_slate_multiclass' are built."""
    if model_type in NOT_BUILT:
        raise NotImplementedError("%s: training %s is not built in this project" % (model_type, NOT_BUILT[model_type]))
    if model_type in NOT_BUILT_SLATE:
        raise NotImplementedError("%s: training this slate-label net is not built in this project (only dien_slate and "
                                  "dien_slate_multiclass are)" % model_type)
    if model_type not in HEADS:
        raise NotImplementedError("%s: training the slate-label and other nets is not built in this project" % model_type)
    return SimulatorTrainer(config, head=HEADS[model_type], **kw)


def supervised_train(train_file, test_file, model_file, model_type="dien", is_slate_label=0, config=None, device=None,
                     verbose=2, **fit_kw):
    """script/supervised_train.py in its argument order.  train_file / test_file: log text (path or lines) or an ItemSamples
    .npz, where the script took TFRecords.  Trains, saves the Saver checkpoint at model_file and returns (trainer, history).
    is_slate_label = 1 reads slate samples and trains dien_slate / dien_slate_multiclass; those nets need it (in the
    reference the item samples' labels do not fit their heads)."""
    slate_net = model_type in HEADS and HEADS[model_type] != 0
    if int(is_slate_label) and not slate_net:
        if model_type in NOT_BUILT_SLATE:
            get_model({}, model_type)
        raise NotImplementedError("is_slate_label = 1 with %s: only dien_slate and dien_slate_multiclass train on slate "
                                  "labels in this project" % model_type)
    if slate_net and not int(is_slate_label):
        raise ValueError("%s trains on slate labels: is_slate_label must be 1, not %r" % (model_type, is_slate_label))
    cfg = {"epoch": EPOCHS, "maxlen": 64, "batch_size": BATCH_SIZE, "class_num": 2, "dense_feature_num": 432,
           "category_feature_num": 21, "category_hash_size": 100000, "seq_num": 2, "emb_size": 128, "hidden_units": 128,
           "action_size": 284}
    cfg.update(config or {})
    model = get_model(cfg, model_type, device=device)
    train, test = _load_samples(train_file, model.config, model.head), _load_samples(test_file, model.config, model.head)
    fit_kw.setdefault("epochs", int(cfg["epoch"]))
    fit_kw.setdefault("batch_size", int(cfg["batch_size"]))
    hist = model.fit(train, test, verbose=verbose, **fit_kw)
    model.save(model_file)
    return model, hist
