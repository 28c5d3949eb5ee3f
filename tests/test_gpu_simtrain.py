"""Simulator-training kernels on the GPU: per-tensor gradient parity with the float64 autograd reference, forward parity with
r4_dien_forward and the f32 oracle, Keras Adam, determinism, agreement with the torch twin, and end-to-end training into a
checkpoint the CUDA env restores."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import simtrain_ref as R  # noqa: E402
from golden_util import assert_close_rel, record_margin  # noqa: E402

from oracle.dien_np import DienOracle  # noqa: E402
from rl4rs_b200 import simtrain, synth  # noqa: E402

pytestmark = pytest.mark.gpu

H = 3000
CFG = {"category_hash_size": H}
TOL = 1e-4
# The attention MLPs' and emb_cat's gradients are sums of nearly cancelling terms, so their fp32 rounding is set by the terms
# rather than the sum: on page 1 the second sequence is 64 copies of the padding id, so its 64 attention rows per sample are
# nearly equal and their d(score) terms cancel; with small embeddings the category self-attention is nearly uniform and its
# softmax backward P (a - P a) is a difference of nearly equal numbers.  Measured on an H100: up to 7.9e-4 (att1_w1, n = 1)
# and 2.2e-4 (emb_cat) of the tensor's largest element.
TOL_CANCEL = 1e-3


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


@pytest.fixture(scope="module")
def samples():
    return R.make_samples(300, H, seed=11)


def _weights(kind):
    if kind == "default":
        return synth.make_weights(CFG, seed=21, bounded_scores=True)
    return synth.make_weights(CFG, seed=22, stress=2.0, bias_noise=0.1, bounded_scores=True)


def _kernel_grad(tr, samples, idx, rate, keep_in=None):
    """One r4_simtrain_grad -> (grad f64, stats, keep bits)."""
    n = len(idx)
    d = tr._data(samples)
    grad = torch.zeros_like(tr.params)
    keep_out = torch.zeros(n, 256, dtype=torch.uint8, device="cuda")
    stats = torch.zeros(2, dtype=torch.float32, device="cuda")
    ki = None if keep_in is None else torch.from_numpy(keep_in).cuda()
    it = torch.from_numpy(np.asarray(idx, np.int64)).cuda()
    rc = tr.lib.r4_simtrain_grad(H, _p(tr.params), C.byref(d), _p(it), n, 5, 77, rate, _p(ki), _p(keep_out),
                                 _p(tr._scratch(n)), _p(grad), _p(stats), None, None)
    tr._check(rc, "r4_simtrain_grad")
    torch.cuda.synchronize()
    return grad.double().cpu().numpy(), stats.cpu().numpy(), keep_out.cpu().numpy()


@pytest.mark.parametrize("kind", ["default", "stress"])
@pytest.mark.parametrize("n", [1, 7, 8, 9, 33, 63, 64, 65, 256, 257])
@pytest.mark.parametrize("rate", [0.0, 0.2])
def test_gradient_parity_per_tensor(samples, kind, n, rate):
    w = _weights(kind)
    tr = simtrain.SimulatorTrainer(CFG, device="cuda", weights=w)
    idx = np.random.RandomState(n).permutation(len(samples))[:n]
    g, stats, keep = _kernel_grad(tr, samples, idx, rate)
    flat = simtrain.flatten(w, CFG)
    loss, ref, probs = R.ref_grad(CFG, flat, samples, idx, keep if rate > 0 else None, rate)
    assert np.all(np.minimum(probs, 1 - probs) > 1e-7 + 1e-6), "a row is within 1e-6 of the loss clip"
    assert abs(stats[0] - loss) <= 1e-5 * abs(loss) + 1e-6        # one sample's loss can be ~1e-3: fp32 log(p) near p = 1
    if rate > 0:
        assert 0.7 < keep.mean() < 0.9
    gt, rt = simtrain.unflatten(g, CFG), simtrain.unflatten(ref, CFG)
    cat, _, seq, _ = samples.features(idx)
    for name in gt:
        err = np.abs(gt[name] - rt[name]).max()
        bound = (TOL_CANCEL if name.startswith(("att", "emb_cat")) else TOL) * np.abs(rt[name]).max()
        record_margin("simtrain %s n%d %s drop%g" % (name, n, kind, rate), np.array([err]), np.array([bound + 1e-30]),
                      np.array([np.abs(rt[name]).max()]))
        assert err <= bound, (name, err, bound)
    touched = {"emb_cat": np.unique(cat), "emb_seq": np.unique(np.concatenate([seq.reshape(-1), cat[:, -10:].reshape(-1)]))}
    for name, ids in touched.items():
        mask = np.ones(H, bool)
        mask[ids] = False
        assert not np.any(gt[name][mask]), name                       # untouched rows exactly zero


def test_forward_parity_with_dien_forward_and_oracle(samples):
    from rl4rs_b200.env.slate import SlateRecEnv, SlateState
    w = _weights("stress")
    tr = simtrain.SimulatorTrainer(CFG, device="cuda", weights=w)
    idx = np.arange(200)
    probs = tr.eval_batch(samples, torch.arange(200, device="cuda")).cpu().numpy()
    cat, dense, seq, _ = samples.features(idx)
    _, p_ref = DienOracle(w, np.float32).forward(seq, dense, cat)
    assert_close_rel(probs, p_ref, what="simtrain eval probs")
    config = {"epoch": 1, "maxlen": 64, "batch_size": 8, "action_size": 284, "class_num": 2, "dense_feature_num": 432,
              "category_feature_num": 21, "category_hash_size": H, "seq_num": 2, "emb_size": 128, "hidden_units": 128,
              "max_steps": 9, "page_items": 9, "action_emb_size": 32, "is_eval": True, "cache_size": 8,
              "support_rllib_mask": True, "output_format": "numpy"}
    catalog = synth.make_catalog()
    env = SlateRecEnv(dict(config, catalog=catalog, log=synth.make_log(16, catalog=catalog, hash_size=H), weights=w),
                      state_cls=SlateState)
    _, p_env = env.engine.dien_forward(seq, dense, cat)
    assert_close_rel(probs, p_env.cpu().numpy(), what="simtrain eval vs r4_dien_forward")


def test_apply_is_keras_adam():
    tr = simtrain.SimulatorTrainer(CFG, device="cuda", weights=_weights("default"))
    rs = np.random.RandomState(0)
    np_ = tr.params.numel()
    g = (rs.normal(size=np_) * 1e-3).astype(np.float32)
    g[: H * 128 // 2] = 0.0                                             # half of emb_cat untouched
    m0 = (rs.normal(size=np_) * 1e-4).astype(np.float32)
    v0 = (rs.random_sample(np_) * 1e-6).astype(np.float32)
    p0 = tr.params.cpu().numpy().copy()
    grad = torch.from_numpy(g).cuda()
    tr.m.copy_(torch.from_numpy(m0)); tr.v.copy_(torch.from_numpy(v0))
    rc = tr.lib.r4_simtrain_apply(H, _p(tr.params), _p(grad), _p(tr.m), _p(tr.v), 3, 1e-3, 0.9, 0.999, 1e-7, None)
    tr._check(rc, "r4_simtrain_apply")
    p, m, v = (torch.from_numpy(x.astype(np.float64)) for x in (p0, m0, v0))
    simtrain.keras_adam_(p, torch.from_numpy(g.astype(np.float64)), m, v, 3)
    got = tr.params.cpu().numpy().astype(np.float64)
    assert np.abs(got - p.numpy()).max() <= 1e-6 * np.abs(p.numpy()).max()
    assert np.abs(tr.v.cpu().numpy() - v.numpy()).max() <= 1e-6 * np.abs(v.numpy()).max()
    L = simtrain.unflatten(grad.cpu().numpy(), CFG)
    assert not L["emb_cat"].any() and not L["emb_seq"].any()            # embedding gradient rows cleared
    assert np.array_equal(L["obs_w"], simtrain.unflatten(g, CFG)["obs_w"])


def test_twenty_steps_bit_identical(samples):
    outs = []
    for _ in range(2):
        tr = simtrain.SimulatorTrainer(CFG, device="cuda", weights=_weights("default"), data_seed=3)
        st = simtrain._Stream(len(samples), 64, 3, torch.device("cuda"))
        for _ in range(20):
            tr.train_step(samples, st.next())
        torch.cuda.synchronize()
        outs.append((tr.params.cpu().numpy(), tr.acc.cpu().numpy()))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])


def test_kernel_and_twin_losses_agree(samples):
    w = _weights("default")
    tr = simtrain.SimulatorTrainer(CFG, device="cuda", weights=w)
    net = simtrain.SimulatorNet(CFG, simtrain.flatten(w, CFG), torch.float32)
    m, v = torch.zeros_like(net.flat.data), torch.zeros_like(net.flat.data)
    rs = np.random.RandomState(4)
    for step in range(1, 4):
        idx = rs.permutation(len(samples))[:128]
        g, stats, keep = _kernel_grad(tr, samples, idx, 0.2)
        gk = torch.from_numpy(g.astype(np.float32)).cuda()
        rc = tr.lib.r4_simtrain_apply(H, _p(tr.params), _p(gk), _p(tr.m), _p(tr.v), step, 1e-3, 0.9, 0.999, 1e-7, None)
        tr._check(rc, "r4_simtrain_apply")
        cat, dense, seq, y = samples.features(idx)
        probs, _ = net(cat, dense, seq, keep, 0.2)
        loss = simtrain.keras_bce(probs, y)
        net.flat.grad = None
        loss.backward()
        simtrain.keras_adam_(net.flat.data, net.flat.grad, m, v, step)
        # step 1 starts from the same parameters; after it Adam's per-element normalisation turns rounding-level differences
        # of near-zero gradient elements into lr-sized steps, so the two trajectories separate slowly
        tol = 1e-5 if step == 1 else 1e-3
        lv = float(loss.detach())
        assert abs(lv - stats[0]) <= tol * abs(lv), (step, lv, stats[0])


def test_teacher_student_on_gpu_and_env_restores_checkpoint(tmp_path):
    cfg = {"category_hash_size": 60}
    tr_s, te_s = R.make_samples(1500, 60, seed=1), R.make_samples(100, 60, seed=2)
    R.teacher_labels(tr_s, cfg, stress=3.0)
    R.teacher_labels(te_s, cfg, stress=3.0, label_seed=3)
    m = simtrain.get_model(cfg, device="cuda", weights=synth.make_weights(cfg, seed=123, bounded_scores=True))
    init = m.evaluate(te_s)["loss"]
    h = m.fit(tr_s, te_s, epochs=6, steps_per_epoch=20, validation_steps=14, batch_size=64)
    best = min(h["val_loss"])
    assert best < 0.85 * init and best < R.constant_loss(te_s.feedback), (init, h["val_loss"])
    assert max(h["val_auc"]) > 0.8

    from rl4rs_b200.env.slate import SlateRecEnv, SlateState
    config = {"epoch": 1, "maxlen": 64, "batch_size": 128, "action_size": 284, "class_num": 2, "dense_feature_num": 432,
              "category_feature_num": 21, "category_hash_size": 5000, "seq_num": 2, "emb_size": 128, "hidden_units": 128,
              "max_steps": 9, "page_items": 9, "action_emb_size": 32, "is_eval": True, "cache_size": 128,
              "support_rllib_mask": True, "output_format": "numpy"}
    s = R.make_samples(64, 5000, seed=5)
    m2 = simtrain.get_model(config, device="cuda", weights=synth.make_weights(config, seed=4, bounded_scores=True))
    m2.fit(s, s, epochs=1, steps_per_epoch=5, validation_steps=1, batch_size=64)
    prefix = str(tmp_path / "sim")
    m2.save(prefix)
    catalog = synth.make_catalog()
    log = synth.make_log(256, catalog=catalog, hash_size=5000)
    env = SlateRecEnv(dict(config, catalog=catalog, log=log, model_file=prefix), state_cls=SlateState)
    w = m2.weights()
    rs = np.random.RandomState(6)
    seq = np.zeros((128, 2, 64), np.int32)
    seq[:, 0, 20:] = rs.randint(1, 284, (128, 44))
    dense = rs.normal(0, 1, (128, 432)).astype(np.float32)
    cat = rs.randint(0, 5000, (128, 21)).astype(np.int32)
    obs, probs = env.engine.dien_forward(seq, dense, cat)
    o_ref, p_ref = DienOracle(w, np.float32).forward(seq, dense, cat)
    assert_close_rel(obs.cpu().numpy(), o_ref, what="trained checkpoint env obs")
    assert_close_rel(probs.cpu().numpy(), p_ref, what="trained checkpoint env probs")
