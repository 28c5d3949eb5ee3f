"""CPU: batch RL on the logged dataset (rl4rs_b200/batchrl.py over the torch twin policy.BatchRLNet) -- dispatch and error
paths, the transition builder, the losses and targets against NumPy float64 restatements, learning on synthetic data,
and checkpoints.  The kernels are checked against the same twin in tests/test_gpu_batchrl.py."""
import math

import numpy as np
import pytest
import torch

A = 284


def synthetic_dataset(K=266, E=80, L=10, seed=0, action_fn=None):
    """E episodes of L entries in the writer's layout: obs = random | 9 prev actions | cur_steps, the reward of entry j's
    action in entry j + 1, terminal on the last entry."""
    rs = np.random.RandomState(seed)
    obs = rs.randn(E, L, K).astype(np.float32)
    obs[:, :, K - 10:K - 1] = rs.randint(0, A, (E, L, 9))
    obs[:, :, K - 1] = np.arange(L)[None]
    act = rs.randint(0, A, (E, L)).astype(np.float32) if action_fn is None else action_fn(obs)
    rew = rs.rand(E, L).astype(np.float32)
    rew[:, 0] = 0
    term = np.zeros((E, L), np.float32)
    term[:, -1] = 1
    return {"observations": obs.reshape(-1, K), "actions": act.reshape(-1, 1), "rewards": rew.reshape(-1),
            "terminals": term.reshape(-1), "discrete_action": np.asarray(True)}


def _cfg(**kw):
    from rl4rs_b200 import synth
    return dict({"action_size": A, "page_items": 9, "catalog": synth.make_catalog(), "CQL_alpha": 1, "gpu": False}, **kw)


def _model(algo, ds=None, **hp):
    from rl4rs_b200 import batchrl
    m = batchrl.get_model(_cfg(), algo)
    m.hp.update(hp)
    m.batch_size = int(m.hp["batch_size"])
    assert m.device.type == "cpu" and not m.use_kernels
    if ds is not None:
        m.build_with_dataset(ds)
    return m


# ---- dispatch ----------------------------------------------------------------------------------------------
def test_dispatch_and_error_paths():
    from rl4rs_b200 import batchrl
    for algo, cls in (("BC", batchrl.DiscreteBC), ("BCQ", batchrl.DiscreteBCQ), ("CQL", batchrl.DiscreteCQL)):
        assert isinstance(batchrl.get_model(_cfg(), algo), cls)
    assert batchrl.get_model(_cfg(CQL_alpha=3), "CQL").hp["alpha"] == 3.0
    for algo in ("BCQ-conti", "CQL-conti", "MOPO", "COMBO", "dynamics"):
        with pytest.raises(NotImplementedError, match=algo):
            batchrl.get_model(_cfg(), algo)
    for algo in ("DQN", "bc", "CQL_rawstate"):
        with pytest.raises(AssertionError):
            batchrl.get_model(_cfg(), algo)
    with pytest.raises(NotImplementedError, match="ope"):
        batchrl.ope_eval()
    with pytest.raises(NotImplementedError, match="soft_opc"):
        batchrl.d3rlpy_eval()
    # the script's own masks win over the catalog's
    lm = np.zeros((4, A), np.int64)
    lm[:3, 5] = 1
    m = batchrl.get_model(_cfg(location_mask=lm, special_items=[7]), "BC")
    m.build_with_dataset(synthetic_dataset(E=2))
    assert int(m.net.location_mask.sum()) == 3 and int(m.net.special.sum()) == 1 and int(m.net.special[7]) == 1
    ds = synthetic_dataset(E=2)
    ds["actions"] = ds["actions"] + 0.5
    with pytest.raises(ValueError, match="discrete"):
        _model("BC").fit(ds)


# ---- the transition list ---------------------------------------------------------------------------------
def test_transition_builder_unequal_episodes():
    from rl4rs_b200.batchrl import transitions_host
    #          ep 0 (3)  ep 1 (1)  ep 2 (5)        unfinished tail
    term = [0, 0, 1, 1, 0, 0, 0, 0, 1, 0, 0]
    assert transitions_host(term).tolist() == [0, 1, 4, 5, 6, 7]
    assert transitions_host([0, 0]).tolist() == []
    ds = synthetic_dataset(E=3, L=4)
    ds["terminals"] = np.array([0, 1, 0, 0, 0, 0, 0, 1, 0, 0, 1, 1], np.float32)
    from rl4rs_b200.batchrl import DeviceDataset
    d = DeviceDataset(ds, "cpu")
    assert d.transitions.tolist() == [0, 2, 3, 4, 5, 6, 8, 9]
    o, a, r, o2, t = d.batch(torch.tensor([1, 5, 7]))
    assert torch.equal(o2, torch.as_tensor(ds["observations"][[3, 7, 10]]))
    assert r.tolist() == ds["rewards"][[3, 7, 10]].tolist() and t.tolist() == [0, 1, 1]


@pytest.mark.parametrize("seq", [False, True])
def test_transitions_of_the_writer_output(oracle_engine, seq):
    """The writer over the stand-in engine: 9 transitions per Slate episode, 36 per SeqSlate-36 episode."""
    from test_gpu_parity import _synthetic
    from rl4rs_b200 import dataset
    from rl4rs_b200.batchrl import transitions_host
    B, epochs = 8, 2
    cfg, cat, log, w = _synthetic(B, seq, max_steps=36 if seq else 9)
    np.random.seed(0)
    fn = dataset.data_generate_rl4rs_b if seq else dataset.data_generate_rl4rs_a
    out = fn(dict(cfg, catalog=cat, log=log, weights=w), epochs=epochs)
    T = 36 if seq else 9
    assert transitions_host(out["terminals"]).numel() == epochs * B * T


@pytest.fixture()
def oracle_engine(monkeypatch):
    import rl4rs_b200.engine as engine_mod
    from oracle_engine import OracleEngine
    monkeypatch.setattr(engine_mod, "Engine", OracleEngine)


# ---- masks, losses and targets against NumPy float64 --------------------------------------------------------
def _np_keep(x, lm, special):
    prev = x[:, -10:-1].astype(np.int64)
    layer = x[:, -1].astype(np.int64) % 9 // 3
    mask = lm[layer].copy()
    for i in range(9):
        mask[np.arange(len(x)), prev[:, i]] = 0
    for i in range(len(x)):
        if len(np.intersect1d(prev[i], special)) > 0:
            mask[i][special] = 0
    return mask >= 0.01


def _np_mnet(x, p, pre, keep):
    x = x.astype(np.float64)
    h = np.maximum(x @ p[pre + "w1"] + p[pre + "b1"], 0)
    e = p[pre + "emb"][x[:, -10:].astype(np.int64)].reshape(len(x), -1)
    f = np.concatenate([h, e], 1) @ p[pre + "w2"] + p[pre + "b2"]
    f[~keep] = 0
    return f @ p[pre + "w3"] + p[pre + "b3"]


def _np_params(net, flat=None):
    return {k: v.detach().double().numpy() for k, v in net.params(flat).items()}


def _lsm(z):
    m = z.max(1, keepdims=True)
    return z - m - np.log(np.exp(z - m).sum(1, keepdims=True))


def _huber(d):
    return np.where(np.abs(d) < 1, 0.5 * d * d, np.abs(d) - 0.5)


def _batch(ds, special_rows=True):
    from rl4rs_b200.batchrl import DeviceDataset
    d = DeviceDataset(ds, "cpu")
    return d, d.batch(torch.arange(0, d.n, 3))


def test_masked_net_matches_numpy():
    ds = synthetic_dataset(E=30)
    m = _model("BCQ", ds)
    x = ds["observations"][:200].copy()
    sp = np.asarray(m.special_items)
    x[:40, -10] = sp[0]                      # special items present in some rows
    x[40:60, -10:-1] = 0                     # item 0 in unfilled slots
    x[60:80, -1] = np.arange(20) + 9         # SeqSlate cur_steps past the first page
    keep = _np_keep(x, m.location_mask, sp)
    assert np.array_equal(m.net.keep(torch.as_tensor(x)).numpy(), keep)
    assert not keep[:40][:, sp].any() and not keep[40:60, 0].any()
    p = _np_params(m.net)
    for pre, fn in (("q_", m.net.q), ("i_", m.net.imitator)):
        got = fn(torch.as_tensor(x)).detach().double().numpy()
        ref = _np_mnet(x, p, pre, keep)
        assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max()


@pytest.mark.parametrize("algo", ["BC", "BCQ", "CQL"])
def test_losses_and_targets_match_numpy(algo):
    ds = synthetic_dataset(E=40)
    m = _model(algo, ds)
    if algo != "BC":
        with torch.no_grad():
            m.net.target.add_(0.1 * torch.randn(m.net.n_target, generator=torch.Generator().manual_seed(1)))
    hp = m._hyper()
    _, (o, a, r, o2, t) = _batch(ds)
    loss, st = m.net.loss(o, a, r, o2, t, hp)
    on, on2, an = o.numpy(), o2.numpy(), a.numpy().astype(np.int64)
    rn, tn = r.numpy().astype(np.float64), t.numpy().astype(np.float64)
    rows = np.arange(len(on))
    p, pt = _np_params(m.net), _np_params(m.net, m.net.target)
    sp = np.asarray(m.special_items)
    k1, k2 = _np_keep(on, m.location_mask, sp), _np_keep(on2, m.location_mask, sp)

    def bc(z, beta):
        return -_lsm(z)[rows, an] + beta * (z * z).mean(1)
    if algo == "BC":
        ref = bc(_np_mnet(on, p, "i_", k1), 0.0).mean()
    else:
        if algo == "BCQ":
            q2 = _np_mnet(on2, p, "q_", k2)
            lp = _lsm(_np_mnet(on2, p, "i_", k2))
            filt = (q2 - q2.min(1, keepdims=True)) * ((lp - lp.max(1, keepdims=True)) > math.log(0.3))
            astar = filt.argmax(1)
            qt = _np_mnet(on2, pt, "q_", k2)[rows, astar]
            q = _np_mnet(on, p, "q_", k1)
            y = rn + 0.99 * (1 - tn) * qt
            ref = (_huber(q[rows, an] - y) + bc(_np_mnet(on, p, "i_", k1), 0.5)).mean()
        else:
            def c(x, pp):
                h = np.maximum(np.maximum(x.astype(np.float64) @ pp["w1"] + pp["b1"], 0) @ pp["w2"] + pp["b2"], 0)
                return h @ pp["w3"] + pp["b3"]
            astar = c(on2, p).argmax(1)
            y = (rn - m.reward_mean) / (m.reward_std + 1e-3) + 1.0 * (1 - tn) * c(on2, pt)[rows, astar]
            q = c(on, p)
            lse = np.log(np.exp(q - q.max(1, keepdims=True)).sum(1)) + q.max(1)
            ref = (_huber(q[rows, an] - y) + 1.0 * (lse - q[rows, an])).mean()
    assert abs(float(loss) - ref) <= 1e-5 * max(1.0, abs(ref)), (float(loss), ref)
    assert abs(float(st[0]) - ref) <= 1e-5 * max(1.0, abs(ref))


def test_reward_scaler_and_huber():
    ds = synthetic_dataset(E=20)
    m = _model("CQL", ds)
    from rl4rs_b200.batchrl import transitions_host
    r = ds["rewards"].astype(np.float64)[transitions_host(ds["terminals"]).numpy()]
    assert m.reward_scaler == "standard"
    assert abs(m.reward_mean - r.mean()) < 1e-12 and abs(m.reward_std - r.std()) < 1e-12
    h = m._hyper()
    assert h["reward_den"] == m.reward_std + 1e-3 and h["gamma"] == 1.0 and h["alpha"] == 1.0
    assert _model("BCQ")._hyper()["reward_den"] == 1.0 and _model("BCQ")._hyper()["gamma"] == 0.99
    d = torch.tensor([-3.0, -1.0, -0.5, 0.0, 0.999, 2.0], requires_grad=True)
    hub = torch.where(d.abs() < 1.0, 0.5 * d * d, d.abs() - 0.5)
    hub.sum().backward()
    assert np.allclose(hub.detach().numpy(), _huber(d.detach().numpy().astype(np.float64)))
    assert d.grad.tolist() == pytest.approx([-1.0, -1.0, -0.5, 0.0, 0.999, 1.0])


def test_target_copy_schedule():
    ds = synthetic_dataset(E=20)
    m = _model("CQL", ds, batch_size=32, target_update_interval=4)
    assert [s for s in range(1, 12) if m._copy_due(s)] == [1, 5, 9]
    assert not _model("BC", ds)._copy_due(1)


# ---- learning ----------------------------------------------------------------------------------------------
def test_bc_learns_a_fixed_logged_rule():
    def rule(obs):                  # the logged action is a fixed function of the observation
        return np.array([10, 50, 150, 200])[(obs[..., 0] > 0) * 2 + (obs[..., 1] > 0)].astype(np.float32)
    ds = synthetic_dataset(E=100, action_fn=rule)
    m = _model("BC", ds, batch_size=64)
    m.fit(ds, n_epochs=20)
    from rl4rs_b200.batchrl import DeviceDataset
    d = DeviceDataset(ds, "cpu")
    e = d.transitions
    got = torch.as_tensor(m.predict(d.obs[e].numpy()))
    assert float((got == d.action[e].long()).float().mean()) > 0.9


def _two_step(E=200, seed=0):
    """Two-step episodes (3 entries): step 0 logs action 3 (reward 1) or 4 (reward 0), step 1 logs 5 (reward 2); the
    observation tells the steps apart.  Returns Q(s0, 3) = 1 + g 2, Q(s0, 4) = g 2, Q(s1, 5) = 2."""
    rs = np.random.RandomState(seed)
    K = 266
    obs = np.zeros((E, 3, K), np.float32)
    obs[:, :, :4] = 0.1 * rs.randn(E, 3, 4)
    obs[:, 0, 4], obs[:, 1, 5], obs[:, 2, 6] = 1, 1, 1
    obs[:, :, K - 1] = np.arange(3)
    a0 = np.where(rs.rand(E) < 0.5, 3, 4)
    act = np.stack([a0, np.full(E, 5), np.zeros(E)], 1).astype(np.float32)
    rew = np.stack([np.zeros(E), (a0 == 3).astype(np.float64), np.full(E, 2.0)], 1).astype(np.float32)
    term = np.zeros((E, 3), np.float32)
    term[:, -1] = 1
    return {"observations": obs.reshape(-1, K), "actions": act.reshape(-1, 1), "rewards": rew.reshape(-1),
            "terminals": term.reshape(-1)}, obs


@pytest.mark.parametrize("algo", ["BCQ", "CQL"])
def test_q_values_approach_the_returns_of_a_two_step_mdp(algo):
    ds, obs = _two_step()
    m = _model(algo, ds, batch_size=50, learning_rate=3e-3, target_update_interval=20)
    m.fit(ds, n_epochs=60)
    pol = __import__("rl4rs_b200.batchrl", fromlist=["policy_model"]).policy_model(m, _cfg())
    g = m.hp["gamma"]
    q0 = pol.predict_q(obs[:50, 0], np.full(50, 3)).mean(), pol.predict_q(obs[:50, 0], np.full(50, 4)).mean()
    q1 = pol.predict_q(obs[:50, 1], np.full(50, 5)).mean()
    tol = 0.35
    assert abs(q1 - 2.0) < tol, q1
    if algo == "BCQ":
        assert abs(q0[0] - (1 + 2 * g)) < tol and abs(q0[1] - 2 * g) < tol, q0
    else:
        # the conservative term pulls the two logged actions of s0 towards each other (each is logged half the time);
        # their order and their mean stay those of the returns
        assert q0[0] > q0[1] + 0.2 and abs((q0[0] + q0[1]) / 2 - (0.5 + 2 * g)) < tol, q0
        q = m.act(obs[:50, 0], 1, want_values=True)[2]
        unlogged = torch.ones(A, dtype=torch.bool)
        unlogged[[3, 4]] = False
        assert float(q[:, unlogged].max()) < float(q[:, 4].min())


# ---- checkpoints -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("algo", ["BC", "BCQ", "CQL"])
def test_save_load_round_trip(algo, tmp_path):
    ds = synthetic_dataset(E=20)
    m = _model(algo, ds, batch_size=32)
    m.fit(ds, 1)
    path = str(tmp_path / "m.pt")
    m.save_model(path)
    m2 = _model(algo)
    m2.load_model(path)
    x = ds["observations"][:100]
    assert np.array_equal(m.predict(x), m2.predict(x))
    assert np.array_equal(m.predict_value(x, np.arange(100) % A), m2.predict_value(x, np.arange(100) % A))
    assert m2.step == m.step and torch.equal(m2.m, m.m) and torch.equal(m2.net.target, m.net.target)
    assert m2.reward_mean == m.reward_mean
    with pytest.raises(ValueError):
        _model("BC" if algo != "BC" else "CQL").load_model(path)


# ---- the reference's own encoder and eval rule ------------------------------------------------------------------
def _reference_obs(K, n, special, seed=0):
    """Random d3rl observations: simulator obs | 9 prev actions | cur_steps, with special items present in some rows and
    absent in others, item 0 in unfilled slots, and Slate (0..8) and SeqSlate (0..35) cur_steps."""
    rs = np.random.RandomState(seed)
    x = rs.randn(n, K)
    plain = np.setdiff1d(np.arange(1, A), special)
    prev = rs.choice(plain, (n, 9))
    cur = np.concatenate([rs.randint(0, 9, n // 2), rs.randint(0, 36, n - n // 2)])
    for i in range(n):
        prev[i, cur[i] % 9:] = 0                       # the window fills up along the page; later slots hold item 0
    with_special = rs.rand(n) < 0.4
    for i in np.nonzero(with_special)[0]:
        prev[i, rs.randint(0, 9)] = rs.choice(special)
    x[:, K - 10:K - 1] = prev
    x[:, K - 1] = cur
    return x, with_special


def test_reference_encoder_and_eval_rule_against_the_twin():
    """rl4rs/nets/cql/encoder.py CustomVectorEncoder.forward and rl4rs/policy/policy_model.py predict_with_mask, run from the
    reference tree under d3rlpy / RLlib stand-ins (tests/golden/make_batchrl_golden.py), against the twin: the encoder to
    float64 rounding, the eval rule's actions equal.  What the reference computes is stored under tests/golden/reference/."""
    import os
    import sys
    from golden_util import reference_result
    from rl4rs_b200.policy import BatchRLNet
    from rl4rs_b200.env.slate import SlateState
    from rl4rs_b200 import synth
    K, n = 266, 96
    special = [int(i) for i in synth.make_catalog().special_items]
    lm = SlateState._location_mask(A)
    cfg = {"page_items": 9, "location_mask": lm, "special_items": special}
    x, with_special = _reference_obs(K, n, special)
    assert with_special.any() and (~with_special).any() and (x[:, K - 1] >= 9).any() and (x[:, K - 10:K - 1] == 0).any()
    nets = {algo: BatchRLNet(algo, K, lm, special, A, "cpu", seed=s) for s, algo in enumerate(("BC", "BCQ", "CQL"))}
    xd = torch.as_tensor(x)
    xf = torch.as_tensor(x.astype(np.float32))
    with torch.no_grad():
        feats = {pre: nets["BCQ"].features(xd, pre, nets["BCQ"].flat.double()).numpy() for pre in ("q_", "i_")}
        acts, probs = {}, {}
        for algo, net in nets.items():
            a, pr, raw = net.act(xf, 0)
            acts[algo] = a.numpy()
            probs[algo] = (pr if algo == "BC" else raw).numpy()       # what _imitator / _q_func return
    p = {k: v.detach().double().numpy() for k, v in nets["BCQ"].params().items()}

    def reference():
        sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
        import make_batchrl_golden as ref
        out = {}
        for pre in ("q_", "i_"):
            out["features_" + pre] = ref.reference_encoder(dict(cfg), x, p[pre + "w1"], p[pre + "b1"], p[pre + "emb"],
                                                           p[pre + "w2"], p[pre + "b2"])
        for algo in nets:
            out["actions_" + algo] = ref.reference_predict_with_mask(dict(cfg), algo, x.astype(np.float32), probs[algo])
        return out
    out = reference_result("batchrl_encoder_eval_rule", reference)
    for pre in ("q_", "i_"):
        ref = out["features_" + pre]
        assert ref.shape == (n, A)
        assert np.abs(feats[pre] - ref).max() <= 1e-12 * np.abs(ref).max(), pre
        assert ((ref == 0) == (feats[pre] == 0)).all()          # the same entries zeroed
    assert (out["features_q_"][with_special][:, special] == 0).all()
    for algo in nets:
        np.testing.assert_array_equal(out["actions_" + algo], acts[algo], err_msg=algo)
