"""Backbone training on the CPU (dnn, widedeep, lstm, adversarial_slate): the reference's slate graphs over the eager
stand-ins against the twins, the twins' item heads against the NumPy oracles, the Saver round trip through each net's
plan, the host-only entry points against a restated layout, routing and errors, the hard-sigmoid kink convention and a
teacher-student fit per backbone."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import simtrain_nets_ref as NR  # noqa: E402

from oracle import ref_harness  # noqa: E402
from rl4rs_b200 import simtrain  # noqa: E402
from rl4rs_b200.utils import tf_checkpoint  # noqa: E402

needs_reference = pytest.mark.skipif(not ref_harness.reference_available(), reason="reference tree absent")


def _lib():
    from rl4rs_b200 import _capi
    return _capi.load_library()


# ---- the reference's graphs over the stand-ins ----------------------------------------------------------------------
@pytest.fixture
def stub(monkeypatch):
    """oracle/tf_eager_stub with Dense(activation='sigmoid'), the metric classes of the compile calls and the tf ops of
    my_loss_fn / my_acc_metrics and adversarial_slate's loss3 (NumPy)."""
    import types
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
        keras.metrics = types.SimpleNamespace(AUC=metric, Precision=metric, Recall=metric,
                                              categorical_accuracy=lambda y, p: None)
        keras.losses = types.SimpleNamespace(categorical_crossentropy=lambda y, p: None, binary_crossentropy=lambda y, p: None)
        tf.einsum = np.einsum
        tf.int64, tf.float32 = np.int64, np.float32
        tf.cast = lambda x, dtype: np.asarray(x).astype(dtype)
        tf.constant = lambda v, dtype=None: np.asarray(v, dtype=dtype)
        tf.one_hot = lambda i, depth: np.eye(depth)[np.asarray(i)]
        tf.exp, tf.log = np.exp, np.log
        tf.reduce_sum = lambda x, axis=None: np.sum(x, axis=axis)
        return mods
    monkeypatch.setattr(st, "_modules", modules)
    return st


GRAPH_CFG = dict(maxlen=64, dense_feature_num=432, category_feature_num=21, class_num=2, seq_num=2, emb_size=128,
                 hidden_units=128, batch_size=8)


@needs_reference
@pytest.mark.parametrize("net,head", [p for p in NR.PAIRS if p[1] in (1, 2)])
def test_reference_slate_graph_matches_the_plan_and_the_twin(stub, net, head, tmp_path):
    H = 600
    c = NR.cfg(H, head)
    w = simtrain.net_weights(c, net, head, seed=5, stress=2.0, bias_noise=0.1)
    rd = tf_checkpoint.TensorBundleReader(simtrain.SAVERS[net](str(tmp_path / "m"), w, c))
    ck = {name: rd.get_tensor(name) for name in rd.variables()}
    if net == 1:                                   # dnn's second Embedding: the graph creates it, nothing reads it
        ck["embedding_1/embeddings"] = np.zeros((H, 128), np.float32)
    s = NR.make_samples(6, H, head, seed=3)
    cat, dense, seq, _ = s.features(np.arange(6))
    r = stub.run_reference_graph(NR.NAMES[(net, head)], dict(GRAPH_CFG, category_hash_size=H), ck, seq.astype(np.float32),
                                 dense, cat)
    plan = simtrain.PLANS[net](c)
    created = sorted((sc, tuple(sh)) for sc, _, sh in r["variables"])
    if net == 1:                                   # dnn's second Embedding is created, feeds nothing and is not held
        created = [v for v in created if v[0] != "embedding_1"]
        assert r["unused"] == []
    assert created == sorted((sc, tuple(sh)) for _, sc, sh in plan)
    tw = simtrain.twin(c, net, simtrain.flatten(w, c, net), torch.float64, head=head)
    with torch.no_grad():
        p, o = tw(cat, dense, seq)
    assert r["probs"].shape == (6, simtrain.CLASSES[head])
    np.testing.assert_allclose(o.numpy(), r["obs"], rtol=0, atol=1e-11 * max(1.0, np.abs(r["obs"]).max()))
    np.testing.assert_allclose(p.numpy(), r["probs"], rtol=0, atol=1e-12)


@pytest.mark.parametrize("net", [1, 2, 3])
def test_twin_item_heads_match_the_oracles(net):
    from oracle.dnn_np import DnnOracle
    from oracle.lstm_np import LstmOracle
    from oracle.widedeep_np import WideDeepOracle
    H = 300
    c = NR.cfg(H, 0)
    w = simtrain.net_weights(c, net, 0, seed=4, stress=2.0, bias_noise=0.1)
    s = NR.make_samples(5, H, 0, seed=3)
    cat, dense, seq, _ = s.features(np.arange(len(s)))
    tw = simtrain.twin(c, net, simtrain.flatten(w, c, net), torch.float64)
    with torch.no_grad():
        p, o = tw(cat, dense, seq)
    oo, op = {1: DnnOracle, 2: WideDeepOracle, 3: LstmOracle}[net](w, np.float64).forward(seq, dense, cat)
    np.testing.assert_allclose(p.numpy(), op, rtol=0, atol=1e-12)
    np.testing.assert_allclose(o.numpy(), oo, rtol=0, atol=1e-11 * max(1.0, np.abs(oo).max()))


def test_adversarial_loss_restated():
    rs = np.random.RandomState(2)
    z = rs.normal(0, 2.0, (40, 9))
    y = (rs.random_sample((40, 9)) < 0.3).astype(np.uint8)
    p = 1 / (1 + np.exp(-z))
    bce = -(y * np.log(p) + (1 - y) * np.log(1 - p)).mean(1)
    q = np.exp(p) / np.exp(p).sum(1, keepdims=True)
    ref = 0.1 * bce + (q * (1 - y)).sum(1)
    np.testing.assert_allclose(simtrain.adversarial_rows(torch.from_numpy(z), y).numpy(), ref, rtol=1e-12)


# ---- checkpoints ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("net,head", NR.PAIRS)
def test_checkpoint_round_trip(net, head, tmp_path):
    H = 70
    c = NR.cfg(H, head)
    w = simtrain.net_weights(c, net, head, seed=8, bias_noise=0.1)
    prefix = simtrain.SAVERS[net](str(tmp_path / "m"), w, c)
    back = simtrain.LOADERS[net](prefix, c)
    assert [k for k, _ in simtrain.layer_plan(c, net)] == list(back)
    for k in back:
        assert back[k].dtype == np.float32 and np.array_equal(back[k], w[k]), k


# ---- host-only entry points -----------------------------------------------------------------------------------------
PARAMS_100K = {(1, 0): 13004034, (1, 1): 13005833, (1, 2): 13009174, (2, 0): 25743874, (2, 1): 25765385, (2, 2): 25805334,
               (3, 0): 26787970, (3, 1): 26789769, (3, 2): 26793110, (4, 3): 25676553}


@pytest.mark.parametrize("H", [1, 9, 100000, 4000000])
def test_net_num_params(H):
    lib = _lib()
    for net, head in NR.PAIRS:
        assert lib.r4_simtrain_net_num_params(net, head, H) == NR.num_params(net, H, head), (net, head)
        if H == 100000:
            assert lib.r4_simtrain_net_num_params(net, head, H) == PARAMS_100K[(net, head)]
        if H == 9:
            c = NR.cfg(H, head)
            assert NR.num_params(net, H, head) == simtrain.flatten(simtrain.net_weights(c, net, head), c, net).size
    for head in (0, 1, 2):
        assert lib.r4_simtrain_net_num_params(0, head, H) == lib.r4_simtrain_head_num_params(head, H)


@pytest.mark.parametrize("n", [1, 2, 63, 64, 65, 255, 257, 4096])
def test_net_scratch_size_is_the_end_of_the_layout(n):
    lib = _lib()
    for net, head in NR.PAIRS:
        assert lib.r4_simtrain_net_scratch_size(net, head, n) == NR.scratch_bytes(net, n, head), (net, head)
    for head in (0, 1, 2):
        assert lib.r4_simtrain_net_scratch_size(0, head, n) == lib.r4_simtrain_head_scratch_size(head, n)


def test_net_size_functions_reject_bad_pairs():
    lib = _lib()
    for net, head in [(0, 3), (1, 3), (2, 3), (3, 3), (4, 0), (4, 1), (4, 2), (5, 0), (-1, 1), (1, -1), (1, 4)]:
        assert lib.r4_simtrain_net_num_params(net, head, 100) == -1 and lib.r4_simtrain_net_scratch_size(net, head, 10) == -1
    for net, head in NR.PAIRS:
        assert lib.r4_simtrain_net_num_params(net, head, 0) == -1 and lib.r4_simtrain_net_num_params(net, head, 4000001) == -1
        assert lib.r4_simtrain_net_scratch_size(net, head, 0) == -1 and lib.r4_simtrain_net_scratch_size(net, head, 4097) == -1
    assert lib.r4_simtrain_head_num_params(3, 100) == -1


# ---- routing and errors ---------------------------------------------------------------------------------------------
def test_routing_and_errors():
    cfg = {"category_hash_size": 50}
    assert simtrain.NOT_BUILT_SLATE == ()
    for name, (net, head) in simtrain.SLATE_NETS.items():
        m = simtrain.get_model(dict(cfg, class_num=2), name, device="cpu")
        assert (m.net, m.head) == (net, head) and m.config["class_num"] == simtrain.CLASSES[head]
        assert m.weights()["rew_w"].shape[1] == simtrain.CLASSES[head]
        with pytest.raises(ValueError, match="is_slate_label"):
            simtrain.supervised_train("a", "b", "c", name, 0)
    for name in ("dnn", "widedeep", "lstm"):
        with pytest.raises(NotImplementedError, match=name):
            simtrain.get_model(cfg, name)
        with pytest.raises(NotImplementedError, match=name):
            simtrain.supervised_train("a", "b", "c", name, 0)
        with pytest.raises(NotImplementedError, match="is_slate_label"):
            simtrain.supervised_train("a", "b", "c", name, 1)
    with pytest.raises(ValueError):
        simtrain.SimulatorTrainer(cfg, device="cpu", net=4, head=1)
    with pytest.raises(ValueError):
        simtrain.SimulatorTrainer(cfg, device="cpu", net=2, head=3)
    assert simtrain.get_model(cfg, "dien_slate", device="cpu").net == simtrain.NET_DIEN


# ---- the hard-sigmoid kink ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_hard_sigmoid_argument_at_the_kink_is_exact(dtype):
    b = dtype(2.5)
    plain = dtype(dtype(0.2) * b) + dtype(0.5)
    fused = dtype(np.float64(dtype(0.2)) * np.float64(b) + 0.5) if dtype == np.float32 else dtype(0.2) * b + dtype(0.5)
    assert plain == 1.0 and fused == 1.0
    assert dtype(dtype(0.2) * dtype(2.6)) + dtype(0.5) > 1.0


def test_kink_slope_is_taken_at_both_ends():
    U = 128
    x = torch.zeros(3, 5, 128, dtype=torch.float64)
    k = torch.zeros(128, 3 * U, dtype=torch.float64)
    rk = torch.zeros(U, 3 * U, dtype=torch.float64)
    for zb, nonzero in ((2.5, True), (2.6, False)):
        b = torch.zeros(3 * U, dtype=torch.float64)
        b[:U] = zb
        b[2 * U:] = 0.3
        b.requires_grad_(True)
        m = []
        h = simtrain.keras_gru(x, k, rk, b, m)
        h.sum().backward()
        assert (b.grad[:U].abs().max() > 0) == nonzero, zb
        if zb == 2.5:
            assert min(m) == 0.0 and float(h.detach().abs().max()) == 0.0     # z = 1 exactly: h stays h0


# ---- learning -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("net", NR.NETS)
def test_teacher_student_learns_on_cpu(net):
    H = 60
    head = 3 if net == 4 else 1
    tr, te = NR.make_samples(500, H, head, seed=1), NR.make_samples(150, H, head, seed=2)
    c = NR.cfg(H, head)
    w = simtrain.net_weights(c, net, head, seed=7, stress=3.0, bias_noise=0.2)
    for s, ls in ((tr, 1), (te, 3)):
        p = NR.ref_probs(net, head, c, simtrain.flatten(w, c, net), s, np.arange(len(s)))
        s.feedback = (np.random.RandomState(ls).random_sample(p.shape) < p).astype(np.uint8)
    m = simtrain.get_model({"category_hash_size": H}, NR.NAMES[(net, head)], device="cpu",
                           weights=simtrain.net_weights(c, net, head, seed=123))
    init = m.evaluate(te)["loss"]
    h = m.fit(tr, te, epochs=8, steps_per_epoch=15, validation_steps=3, batch_size=48)
    assert set(h) == set(simtrain.HISTORY[head]) | {"val_" + k for k in simtrain.HISTORY[head]}
    assert max(h["val_auc"]) > 0.75, h["val_auc"]
    assert min(h["val_loss"]) < 0.95 * init, (init, h["val_loss"])


@pytest.mark.parametrize("name", ["dnn_slate_multiclass", "lstm_slate", "adversarial_slate"])
def test_supervised_train_saves_through_the_plan(name, tmp_path):
    H = 300
    net, head = simtrain.SLATE_NETS[name]
    s = NR.make_samples(30, H, 1, seed=6)
    p = str(tmp_path / "slate.npz")
    s.save(p)
    prefix = str(tmp_path / "model")
    m, h = simtrain.supervised_train(p, p, prefix, name, 1, config={"category_hash_size": H}, device="cpu", verbose=0,
                                     epochs=1, steps_per_epoch=2, validation_steps=1, batch_size=16)
    back = simtrain.LOADERS[net](prefix, NR.cfg(H, head))
    for k, v in m.weights().items():
        assert np.array_equal(back[k], v), k
    st = str(tmp_path / "state.npz")
    m.save_state(st)
    m2 = simtrain.get_model({"category_hash_size": H}, name, device="cpu", seed=1)
    m2.load_state(st)
    assert torch.equal(m2.flat_params(), m.flat_params())
    other = "dnn_slate" if name != "dnn_slate_multiclass" else "dien_slate_multiclass"
    with pytest.raises(ValueError):
        simtrain.get_model({"category_hash_size": H}, other, device="cpu").load_state(st)
