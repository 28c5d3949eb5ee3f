"""Slate-label simulator training on the CPU: the slate samples against the reference's own tfrecord_slate stage, the
dien_slate / dien_slate_multiclass graphs and losses of the reference against the twin's heads, the metrics against direct
NumPy computations, the host-only entry points against the restated layout, the routing and error paths of get_model /
supervised_train, teacher-student learning and the Saver round trip."""
import os
import random
import sys
import types

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import simtrain_ref as R  # noqa: E402
import simtrain_slate_ref as SR  # noqa: E402

from oracle import ref_harness  # noqa: E402
from rl4rs_b200 import simtrain, synth  # noqa: E402
from rl4rs_b200.utils import tf_checkpoint  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "simtrain", "slate_samples.npz")
needs_reference = pytest.mark.skipif(not ref_harness.reference_available(), reason="reference tree absent")


# ---- samples --------------------------------------------------------------------------------------------------------
def test_slate_samples_match_reference_tfrecord_slate():
    z = np.load(GOLDEN)
    s = simtrain.slate_samples(list(z["lines"]), {"category_hash_size": 100000})
    assert isinstance(s, simtrain.SlateSamples) and len(s) == s.n_records == z["cat"].shape[0] == 18
    cat, dense, seq, y = s.features(np.arange(len(s)))
    random.seed(int(z["shuffle_seed"]))
    perm = list(range(len(s)))
    random.shuffle(perm)                                  # the script's random.shuffle(records), undone
    assert np.array_equal(z["cat"], cat[perm]) and np.array_equal(z["dense"], dense[perm])
    assert np.array_equal(z["seq"], seq[perm]) and np.array_equal(z["slate_label"], y[perm])
    assert cat.shape == (18, 21) and dense.shape == (18, 432) and y.shape == (18, 9) and y.dtype == np.uint8
    assert not cat[:, 20].any() and not dense[:, 392:].any()              # the pad id 0 and the 40 zero features
    assert np.array_equal(cat[:, 11:20], s.items) and np.array_equal(y, s.feedback)


def test_slate_samples_share_the_item_store(tmp_path):
    lines = list(np.load(GOLDEN)["lines"])
    items = simtrain.item_samples(lines, {"category_hash_size": 100000})
    s = simtrain.slate_samples(lines, {"category_hash_size": 100000})
    for k in simtrain.ItemSamples.FIELDS:
        assert np.array_equal(getattr(s, k), getattr(items, k))
    assert len(items) == 9 * len(s)
    p = str(tmp_path / "s.npz")
    items.save(p)
    t = simtrain.SlateSamples.load(p)
    assert type(t) is simtrain.SlateSamples and type(simtrain.ItemSamples.load(p)) is simtrain.ItemSamples
    for a, b in zip(t.features(np.arange(len(t))), s.features(np.arange(len(s)))):
        assert np.array_equal(a, b)
    with pytest.raises(ValueError):
        simtrain.slate_samples(lines, {"category_hash_size": 1000})


# ---- the reference's graphs and losses over the stand-ins -----------------------------------------------------------
def _np_keras_cce(y, p):
    """Keras backend categorical_crossentropy on probabilities (not a Softmax op's output): normalise, clip, -sum y log p."""
    p = p / p.sum(-1, keepdims=True)
    return -(y * np.log(np.clip(p, 1e-7, 1 - 1e-7))).sum(-1)


@pytest.fixture
def stub(monkeypatch):
    """oracle/tf_eager_stub with what the slate nets touch besides dien.py's graph: Dense(activation='sigmoid'), the
    metric classes of their compile calls, and the tf ops of my_loss_fn / my_acc_metrics (NumPy)."""
    from oracle import tf_eager_stub as st
    call = st.Dense.call

    def dense_call(self, x):
        if self.act == "sigmoid":
            w, b = self.weight("kernel", (x.shape[-1], self.units)), self.weight("bias", (self.units,))
            return st._sigmoid(x @ w + b)
        return call(self, x)
    monkeypatch.setattr(st.Dense, "call", dense_call)
    make = st._modules

    def modules():
        mods = make()
        tf, keras = mods["tensorflow"], mods["tensorflow.keras"]
        metric = type("Metric", (), {"__init__": lambda self, *a, **k: None})
        keras.metrics = types.SimpleNamespace(
            AUC=metric, Precision=metric, Recall=metric,
            categorical_accuracy=lambda y, p: (np.argmax(y, -1) == np.argmax(p, -1)).astype(np.float32))
        keras.losses = types.SimpleNamespace(categorical_crossentropy=_np_keras_cce)
        tf.einsum = np.einsum
        tf.int64 = np.int64
        tf.cast = lambda x, dtype: np.asarray(x).astype(dtype)
        tf.constant = lambda v, dtype=None: np.asarray(v, dtype=dtype)
        tf.one_hot = lambda i, depth: np.eye(depth)[np.asarray(i)]
        return mods
    monkeypatch.setattr(st, "_modules", modules)
    return st


def _graph_inputs(n, H, seed):
    s = SR.make_samples(n, H, seed=seed)
    return s, s.features(np.arange(n))


@needs_reference
@pytest.mark.parametrize("head", SR.HEADS)
def test_reference_slate_graph_matches_the_plan_and_the_twin(stub, head, tmp_path):
    H = 600
    cfg = dict(maxlen=64, dense_feature_num=432, category_feature_num=21, class_num=2, seq_num=2, emb_size=128,
               hidden_units=128, category_hash_size=H, batch_size=8)
    c = SR.cfg(H, head)
    w = simtrain.head_weights(c, head, seed=5, stress=2.0, bias_noise=0.1, bounded_scores=True)
    rd = tf_checkpoint.TensorBundleReader(tf_checkpoint.save_dien_checkpoint(str(tmp_path / "m"), w, c))
    ck = {name: rd.get_tensor(name) for name in rd.variables()}
    s, (cat, dense, seq, _) = _graph_inputs(6, H, 3)
    r = stub.run_reference_graph(SR.NAMES[head], cfg, ck, seq.astype(np.float32), dense, cat)
    assert not r["unused"]
    created = sorted((sc, tuple(sh)) for sc, _, sh in r["variables"])
    assert created == sorted((sc, tuple(sh)) for _, sc, sh in tf_checkpoint.dien_layer_plan(c))
    net = simtrain.SimulatorNet(c, simtrain.flatten(w, c), torch.float64, head=head)
    with torch.no_grad():
        p, o = net(cat, dense, seq)
    assert r["probs"].shape == (6, simtrain.CLASSES[head])
    np.testing.assert_allclose(o.numpy(), r["obs"], rtol=0, atol=1e-11 * max(1.0, np.abs(r["obs"]).max()))
    np.testing.assert_allclose(p.numpy(), r["probs"], rtol=0, atol=1e-12)


@needs_reference
def test_reference_loss_and_accuracy_equal_the_twin_restatement(stub):
    import importlib
    with stub._swapped_modules():
        ref = importlib.import_module("rl4rs.nets.dien_slate_multiclass")
        loss_fn, acc_fn = ref.my_loss_fn, ref.my_acc_metrics
        pats = (np.arange(512)[:, None] >> np.arange(9)[None, :]) & 1      # every click pattern
        rs = np.random.RandomState(0)
        pats = np.concatenate([pats, (rs.random_sample((300, 9)) < 0.3).astype(np.int64)])
        z = rs.normal(0, 2.0, (len(pats), 22))
        p = torch.softmax(torch.from_numpy(z), -1).numpy()
        cls = simtrain.slate2label(pats)
        assert cls.min() == 0 and cls.max() == 21 and len(np.unique(cls[:512])) == 22
        ref_loss = loss_fn(pats, p)
        ref_acc = acc_fn(pats, p)
    ours = simtrain.slate_cce_rows(torch.from_numpy(z), pats).numpy()
    np.testing.assert_allclose(ours, ref_loss, rtol=1e-12, atol=0)
    m = simtrain.MulticlassMetrics()
    m.add(p.astype(np.float32), pats, ours)
    assert m.acc[1] == ref_acc.sum() and m.acc[2] == len(pats)


def test_slate_bce_is_keras_binary_crossentropy_from_logits():
    rs = np.random.RandomState(1)
    z = rs.normal(0, 3.0, (50, 9))
    y = (rs.random_sample((50, 9)) < 0.4).astype(np.uint8)
    p = 1 / (1 + np.exp(-z))
    ref = -(y * np.log(p) + (1 - y) * np.log(1 - p)).mean(1)
    np.testing.assert_allclose(simtrain.slate_bce_rows(torch.from_numpy(z), y).numpy(), ref, rtol=1e-12)
    big = simtrain.slate_bce_rows(torch.tensor([[60.0] * 9, [-60.0] * 9]), np.array([[0] * 9, [1] * 9]))
    assert np.allclose(big.numpy(), 60.0)                             # the logits path: no clip at -log(1e-7)


# ---- metrics --------------------------------------------------------------------------------------------------------
def test_slate_metrics_against_numpy():
    rs = np.random.RandomState(3)
    p = rs.random_sample((400, 9)).astype(np.float32)
    p[:5] = 0.5                                                       # the edge: p == 0.5 is negative
    y = (rs.random_sample((400, 9)) < p).astype(np.uint8)
    m = simtrain.SlateMetrics()
    m.add(p[:150], y[:150], np.ones(150))
    m.add(p[150:], y[150:], np.ones(250) * 3)
    r = m.result()
    pos, yy = p.reshape(-1) > 0.5, y.reshape(-1) > 0
    assert r["precision"] == pytest.approx((pos & yy).sum() / pos.sum(), abs=1e-15)
    assert r["recall"] == pytest.approx((pos & yy).sum() / yy.sum(), abs=1e-15)
    assert r["loss"] == pytest.approx((150 + 750) / 400)
    thr = np.concatenate([[-1e-7], np.arange(1, 199) / 199.0, [1 + 1e-7]]).astype(np.float32)
    pp = p.reshape(-1)
    tp = np.array([((pp > t) & yy).sum() for t in thr], float)
    fp = np.array([((pp > t) & ~yy).sum() for t in thr], float)
    tpr, fpr = tp / yy.sum(), fp / (~yy).sum()
    assert r["auc"] == pytest.approx(np.sum((fpr[:-1] - fpr[1:]) * (tpr[:-1] + tpr[1:]) / 2), abs=1e-12)
    e = simtrain.SlateMetrics()
    e.add(np.full((2, 9), 0.5, np.float32), np.zeros((2, 9)), np.zeros(2))
    assert e.result()["precision"] == 0.0 and e.result()["recall"] == 0.0        # Keras div_no_nan


def test_multiclass_accuracy_takes_the_first_argmax():
    p = np.zeros((3, 22), np.float32)
    p[0, [3, 5]] = 0.5                                        # tie: the first index wins (tf.argmax)
    p[1, 0] = 1.0
    p[2, 21] = 1.0
    y = np.zeros((3, 9), np.int64)
    y[0, [0, 1]] = 1                                          # class 3
    y[2] = 1                                                  # class 21
    m = simtrain.MulticlassMetrics()
    m.add(p, y, np.array([1.0, 2.0, 3.0]))
    assert m.result() == {"loss": 2.0, "acc": 1.0}
    y[0] = [0, 0, 0, 1, 0, 1, 0, 0, 0]                        # 1 + 4: class 5, the second of the tie
    m = simtrain.MulticlassMetrics()
    m.add(p, y, np.zeros(3))
    assert m.result()["acc"] == pytest.approx(2 / 3)


# ---- host-only entry points -----------------------------------------------------------------------------------------
def _lib():
    from rl4rs_b200 import _capi
    return _capi.load_library()


@pytest.mark.parametrize("H", [1, 9, 100000, 4000000])
def test_head_num_params(H):
    lib = _lib()
    assert lib.r4_simtrain_head_num_params(0, H) == lib.r4_simtrain_num_params(H) == R.num_params(H)
    for head in SR.HEADS:
        assert lib.r4_simtrain_head_num_params(head, H) == SR.num_params(H, head)
    if H == 9:
        assert SR.num_params(H, 1) == simtrain.flatten(simtrain.head_weights(SR.cfg(9, 1), 1), SR.cfg(9, 1)).size


@pytest.mark.parametrize("n", list(range(1, 131)) + [4095, 4096])
def test_head_scratch_size_is_the_end_of_the_layout(n):
    lib = _lib()
    assert lib.r4_simtrain_head_scratch_size(0, n) == lib.r4_simtrain_scratch_size(n) == R.scratch_bytes(n)
    for head in SR.HEADS:
        assert lib.r4_simtrain_head_scratch_size(head, n) == SR.scratch_bytes(n, head)


def test_head_size_functions_reject_out_of_range():
    lib = _lib()
    for head in (-1, 3, 100):
        assert lib.r4_simtrain_head_num_params(head, 100) == -1 and lib.r4_simtrain_head_scratch_size(head, 10) == -1
    for head in (0, 1, 2):
        assert lib.r4_simtrain_head_num_params(head, 0) == -1 and lib.r4_simtrain_head_num_params(head, 4000001) == -1
        assert lib.r4_simtrain_head_scratch_size(head, 0) == -1 and lib.r4_simtrain_head_scratch_size(head, 4097) == -1


# ---- routing and errors ---------------------------------------------------------------------------------------------
def test_routing_and_errors():
    cfg = {"category_hash_size": 50}
    for name, head in (("dien_slate", 1), ("dien_slate_multiclass", 2)):
        m = simtrain.get_model(dict(cfg, class_num=2), name, device="cpu")
        assert m.head == head and m.config["class_num"] == simtrain.CLASSES[head]
        assert m.weights()["rew_w"].shape == (256, simtrain.CLASSES[head])
        with pytest.raises(ValueError, match="is_slate_label"):
            simtrain.supervised_train("a", "b", "c", name, 0)
    for name in simtrain.NOT_BUILT_SLATE:
        with pytest.raises(NotImplementedError, match=name):
            simtrain.get_model(cfg, name)
        with pytest.raises(NotImplementedError, match=name):
            simtrain.supervised_train("a", "b", "c", name, 1)
    with pytest.raises(NotImplementedError, match="is_slate_label"):
        simtrain.supervised_train("a", "b", "c", "dien", 1)
    with pytest.raises(ValueError):
        simtrain.get_model(cfg, "dien_slate", device="cpu", weights=synth.make_weights(cfg))      # a 2-wide head


# ---- learning and checkpoints ---------------------------------------------------------------------------------------
def _fit_patterns(n_records, H):
    """The 22-way check's sets: the teacher's decisions (p > 0.5) as clicks, validated on the first third of the training
    records.  From a few thousand random records the 22 click patterns do not generalise within a test's few hundred
    steps (the student fits the training records while the held-out loss stays near the constant predictor's); what this
    checks is that the 22-way loss, its gradient and Adam fit the patterns a teacher draws."""
    tr = SR.make_samples(n_records, H, seed=1)
    SR.teacher_labels(tr, H, draw=False)
    return tr, simtrain.SlateSamples(H, **{k: getattr(tr, k)[:n_records // 3] for k in simtrain.ItemSamples.FIELDS})


@pytest.mark.parametrize("head", SR.HEADS)
def test_teacher_student_learns_on_cpu(head):
    H = 60
    if head == 1:
        tr, te = SR.make_samples(800, H, seed=1), SR.make_samples(200, H, seed=2)
        SR.teacher_labels(tr, H)
        SR.teacher_labels(te, H, label_seed=3)
    else:
        tr, te = _fit_patterns(600, H)
    m = simtrain.get_model({"category_hash_size": H}, SR.NAMES[head], device="cpu",
                           weights=simtrain.head_weights(SR.cfg(H, head), head, seed=123, bounded_scores=True))
    init = m.evaluate(te)["loss"]
    h = m.fit(tr, te, epochs=4, steps_per_epoch=20, validation_steps=4, batch_size=48)
    keys = simtrain.HISTORY[head]
    assert set(h) == set(keys) | {"val_" + k for k in keys}
    best = min(h["val_loss"])
    if head == 1:
        const = R.constant_loss(te.feedback)
        assert max(h["val_auc"]) > 0.8, h["val_auc"]
    else:
        f = np.bincount(simtrain.slate2label(te.feedback), minlength=22) / len(te)
        const = -float(np.sum(f[f > 0] * np.log(f[f > 0])))
        assert max(h["val_acc"]) > f.max(), (h["val_acc"], f.max())
    assert best < 0.85 * init and best < const, (init, const, h["val_loss"])


@pytest.mark.parametrize("head", SR.HEADS)
def test_supervised_train_saves_a_checkpoint_that_reloads_bit_exact(head, tmp_path):
    H = 300
    s = SR.make_samples(40, H, seed=6)
    p = str(tmp_path / "slate.npz")
    s.save(p)
    prefix = str(tmp_path / "model")
    m, h = simtrain.supervised_train(p, p, prefix, SR.NAMES[head], 1, config={"category_hash_size": H}, device="cpu",
                                     verbose=0, epochs=1, steps_per_epoch=2, validation_steps=1, batch_size=16)
    assert set(h) == set(simtrain.HISTORY[head]) | {"val_" + k for k in simtrain.HISTORY[head]}
    back = tf_checkpoint.load_dien_checkpoint(prefix, SR.cfg(H, head))
    ref = m.weights()
    assert set(back) == set(ref) and back["rew_w"].shape == (256, simtrain.CLASSES[head])
    for k in ref:
        assert back[k].dtype == np.float32 and np.array_equal(back[k], ref[k]), k
    st = str(tmp_path / "state.npz")
    m.save_state(st)
    m2 = simtrain.get_model({"category_hash_size": H}, SR.NAMES[head], device="cpu", seed=1)
    m2.load_state(st)
    assert m2.step == m.step and torch.equal(m2.flat_params(), m.flat_params()) and torch.equal(m2.m, m.m)
    with pytest.raises(ValueError, match="head"):
        simtrain.get_model({"category_hash_size": H}, SR.NAMES[3 - head], device="cpu").load_state(st)


def test_twin_gradient_matches_finite_differences():
    """The slate heads' float64 autograd (the kernels' reference) against central differences on the head weights."""
    H = 40
    s = SR.make_samples(6, H, seed=9)
    for head in SR.HEADS:
        c = SR.cfg(H, head)
        flat = simtrain.flatten(simtrain.head_weights(c, head, seed=4, bounded_scores=True), c).astype(np.float64)
        idx = np.arange(6)
        _, g, _ = SR.ref_grad(head, c, flat, s, idx, None, 0.0)
        o = len(flat) - simtrain.CLASSES[head] * 257                # rew_w then rew_b at the end of the layout
        for k in (o, o + 3, len(flat) - 1):
            e = np.zeros_like(flat)
            e[k] = 1e-6
            lp = SR.ref_grad(head, c, flat + e, s, idx, None, 0.0)[0]
            lm = SR.ref_grad(head, c, flat - e, s, idx, None, 0.0)[0]
            assert abs((lp - lm) / 2e-6 - g[k]) <= 1e-6 * max(1.0, abs(g[k])), (head, k)
