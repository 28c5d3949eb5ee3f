"""Simulator training on the CPU: the item samples against the reference's own tfrecord_item stage, the float64 twin against
the NumPy oracle, the loss / dropout / Keras Adam restatements, teacher-student learning, checkpoints and the error paths."""
import math
import os
import random
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import simtrain_ref as R  # noqa: E402

from oracle.dien_np import DienOracle  # noqa: E402
from rl4rs_b200 import simtrain, synth  # noqa: E402
from rl4rs_b200.env.slate import SlateRecEnv  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "simtrain", "item_samples.npz")


def test_item_samples_match_reference_tfrecord_item():
    z = np.load(GOLDEN)
    s = simtrain.item_samples(list(z["lines"]), {"category_hash_size": 100000})
    assert len(s) == z["cat"].shape[0] == 9 * 18
    cat, dense, seq, y = s.features(np.arange(len(s)))
    random.seed(int(z["shuffle_seed"]))
    perm = list(range(len(s)))
    random.shuffle(perm)                                  # the script's random.shuffle(records), undone
    assert np.array_equal(z["cat"], cat[perm])
    assert np.array_equal(z["dense"], dense[perm])
    assert np.array_equal(z["seq"], seq[perm])
    assert np.array_equal(z["label"], y[perm])
    assert (seq[:, 0, 0] != 0).any() and (seq[:, 1, -1] == 0).any() and (seq[:, 1, -27] != 0).any()


def test_item_samples_save_load_and_bad_ids(tmp_path):
    lines = list(np.load(GOLDEN)["lines"])
    s = simtrain.item_samples(lines, {"category_hash_size": 100000})
    p = str(tmp_path / "s.npz")
    s.save(p)
    t = simtrain.ItemSamples.load(p)
    for k in simtrain.ItemSamples.FIELDS:
        assert np.array_equal(getattr(s, k), getattr(t, k))
    with pytest.raises(ValueError):
        simtrain.item_samples(lines, {"category_hash_size": 1000})      # portrait ids above 1000
    f = lines[0].split("@")
    f[3] = "-1," + f[3].split(",", 1)[1]
    with pytest.raises(ValueError):
        simtrain.item_samples(["@".join(f)], {"category_hash_size": 100000})


@pytest.mark.parametrize("stress", [1.0, 2.0])
def test_twin_forward_matches_oracle_f64(stress):
    cfg = {"category_hash_size": 700}
    s = R.make_samples(6, 700, seed=4)
    kw = dict(stress=stress, bias_noise=0.1, bounded_scores=True) if stress != 1.0 else {}
    w = synth.make_weights(cfg, seed=5, **kw)
    cat, dense, seq, _ = s.features(np.arange(len(s)))
    net = simtrain.SimulatorNet(cfg, simtrain.flatten(w, cfg), torch.float64)
    with torch.no_grad():
        p, o = net(cat, dense, seq)
    ob, pr = DienOracle({k: v.astype(np.float64) for k, v in w.items()}, np.float64).forward(seq, dense, cat)
    assert np.abs(p.numpy() - pr).max() <= 1e-11
    assert np.abs(o.numpy() - ob).max() <= 1e-11 * max(1.0, np.abs(ob).max())


def test_loss_clip_and_gradient():
    p = torch.tensor([[0.3, 0.7], [1e-9, 1 - 1e-9], [0.5, 0.5]], dtype=torch.float64, requires_grad=True)
    y = np.array([1, 1, 0])
    loss = simtrain.keras_bce(p, y)
    pc = np.clip(p.detach().numpy(), 1e-7, 1 - 1e-7)
    yy = np.eye(2)[y]
    ref = -(yy * np.log(pc) + (1 - yy) * np.log(1 - pc)).mean()
    assert abs(float(loss.detach()) - ref) < 1e-12
    loss.backward()
    g = p.grad.numpy()
    assert np.all(g[1] == 0.0)                                            # clipped: no gradient
    assert abs(g[0, 1] - (0.7 - 1) / (0.7 * 0.3) / 6) < 1e-12


def test_dropout_scaling():
    keep = np.zeros((2, 256), np.uint8)
    keep[0, :3] = 1
    keep[1, 128:] = 1
    k0, k1 = simtrain.keep_scale(torch.from_numpy(keep), 0.2)
    assert float(k0[0, 0]) == pytest.approx(1.25) and float(k0[0, 3]) == 0.0 and float(k1[0].sum()) == 0.0
    assert float(k1[1].sum()) == pytest.approx(128 * 1.25)
    cfg = {"category_hash_size": 300}
    s = R.make_samples(2, 300, seed=1)
    cat, dense, seq, _ = s.features(np.arange(4))
    net = simtrain.SimulatorNet(cfg, dtype=torch.float64)
    with torch.no_grad():
        full = net(cat, dense, seq, np.ones((4, 256), np.uint8), 0.0)[0]
        plain = net(cat, dense, seq)[0]
        dropped = net(cat, dense, seq, np.ones((4, 256), np.uint8), 0.2)[0]
    assert torch.equal(full, plain) and not torch.allclose(dropped, plain)


def test_keras_adam_formula_differs_from_torch():
    rs = np.random.RandomState(0)
    p0, g = rs.normal(size=50), rs.normal(size=50) * 1e-6       # small gradients: eps placement matters
    p, m, v = (torch.tensor(x) for x in (p0.copy(), np.zeros(50), np.zeros(50)))
    pr, mr, vr = p0.copy(), np.zeros(50), np.zeros(50)
    for t in (1, 2, 3):
        simtrain.keras_adam_(p, torch.tensor(g), m, v, t)
        mr += (g - mr) * 0.1
        vr += (g * g - vr) * 0.001
        pr -= 1e-3 * math.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t) * mr / (np.sqrt(vr) + 1e-7)
    assert np.abs(p.numpy() - pr).max() < 1e-15
    q = torch.tensor(p0.copy(), requires_grad=True)
    opt = torch.optim.Adam([q], lr=1e-3, eps=1e-7)
    for _ in range(3):
        q.grad = torch.tensor(g)
        opt.step()
    assert np.abs(q.detach().numpy() - pr).max() > 1e-6


def test_auc_matches_trapezoid_on_thresholds():
    rs = np.random.RandomState(2)
    p1 = rs.random_sample(400).astype(np.float32)
    y = (rs.random_sample(400) < p1).astype(np.int64)
    probs = np.stack([1 - p1, p1], 1)
    m = simtrain.Metrics()
    m.add(probs, y, np.zeros(400))
    thr = np.concatenate([[-1e-7], np.arange(1, 199) / 199.0, [1 + 1e-7]]).astype(np.float32)
    yy, pp = np.eye(2)[y].reshape(-1), probs.reshape(-1)
    tp = np.array([((pp > t) & (yy > 0)).sum() for t in thr], float)
    fp = np.array([((pp > t) & (yy == 0)).sum() for t in thr], float)
    tpr, fpr = tp / yy.sum(), fp / (1 - yy).sum()
    ref = np.sum((fpr[:-1] - fpr[1:]) * (tpr[:-1] + tpr[1:]) / 2)
    r = m.result()
    assert r["auc"] == pytest.approx(ref, abs=1e-12)
    assert r["acc"] == pytest.approx(((probs > 0.5) == np.eye(2)[y]).mean(), abs=1e-12)


def test_teacher_student_learns_on_cpu():
    cfg = {"category_hash_size": 60}
    tr, te = R.make_samples(1500, 60, seed=1), R.make_samples(100, 60, seed=2)
    R.teacher_labels(tr, cfg, stress=3.0)
    R.teacher_labels(te, cfg, stress=3.0, label_seed=3)
    m = simtrain.get_model(cfg, device="cpu", weights=synth.make_weights(cfg, seed=123, bounded_scores=True))
    init = m.evaluate(te)["loss"]
    h = m.fit(tr, te, epochs=4, steps_per_epoch=20, validation_steps=14, batch_size=64)
    assert set(h) == {"loss", "auc", "acc", "val_loss", "val_auc", "val_acc"}
    best = min(h["val_loss"])
    const = R.constant_loss(te.feedback)
    assert best < 0.85 * init and best < const, (init, const, h["val_loss"])
    assert max(h["val_auc"]) > 0.8


def test_early_stopping_keeps_last_epoch(monkeypatch):
    cfg = {"category_hash_size": 300}
    m = simtrain.get_model(cfg, device="cpu")
    s = R.make_samples(4, 300)
    seq = iter([1.0, 0.9, 0.95, 0.97, 0.99, 0.5])
    monkeypatch.setattr(m, "_run", lambda fn, *a: {"loss": 0.0, "acc": 0.0, "auc": 0.0} if fn == m.train_step else
                        {"loss": next(seq), "acc": 0.0, "auc": 0.0})
    h = m.fit(s, s, epochs=6, steps_per_epoch=1, validation_steps=1, patience=3)
    assert h["val_loss"] == [1.0, 0.9, 0.95, 0.97, 0.99]                    # 3 epochs without improvement


def test_save_roundtrip_through_env_loader(tmp_path):
    cfg = {"category_hash_size": 400}
    m = simtrain.get_model(cfg, device="cpu", seed=9)
    s = R.make_samples(8, 400)
    m.fit(s, s, epochs=1, steps_per_epoch=1, validation_steps=1, batch_size=16)
    prefix = str(tmp_path / "model")
    m.save(prefix)
    w = SlateRecEnv.load_model_file(prefix, dict(cfg, algo="dien"))
    ref = m.weights()
    assert set(w) == set(ref)
    for k in ref:
        assert w[k].dtype == np.float32 and np.array_equal(w[k], ref[k]), k
    st = str(tmp_path / "state.npz")
    m.save_state(st)
    m2 = simtrain.get_model(cfg, device="cpu", seed=1)
    m2.load_state(st)
    assert m2.step == m.step and torch.equal(m2.flat_params(), m.flat_params()) and torch.equal(m2.v, m.v)


def test_unbuilt_models_raise():
    for t in ("dnn", "widedeep", "lstm"):
        with pytest.raises(NotImplementedError, match=t):
            simtrain.get_model({"category_hash_size": 10}, t)
    with pytest.raises(NotImplementedError, match="is_slate_label"):
        simtrain.supervised_train("a", "b", "c", "dien", 1)
    with pytest.raises(ValueError):
        simtrain.get_model({"category_hash_size": 10, "emb_size": 64}, "dien", device="cpu")


def test_size_functions_reject_out_of_range():
    from rl4rs_b200 import _capi
    lib = _capi.load_library()
    assert lib.r4_simtrain_num_params(100000) == 27413956
    assert lib.r4_simtrain_num_params(5000) == simtrain.flatten(synth.make_weights({"category_hash_size": 5000}),
                                                                 {"category_hash_size": 5000}).size
    assert lib.r4_simtrain_num_params(0) == -1 and lib.r4_simtrain_num_params(4000001) == -1
    assert lib.r4_simtrain_scratch_size(0) == -1 and lib.r4_simtrain_scratch_size(4097) == -1
    assert 0 < lib.r4_simtrain_scratch_size(1) < lib.r4_simtrain_scratch_size(256) < lib.r4_simtrain_scratch_size(4096)
