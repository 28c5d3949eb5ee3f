"""CPU: continuous-action CQL on the logged dataset (rl4rs_b200.batchrl.ContinuousCQL over the torch twin
policy.BatchRLContiNet) -- dispatch and error paths, the noise restatement, the twin's terms against NumPy float64, learning
on synthetic data, checkpoints and the train / eval stages over the oracle-backed engine.  The kernels are checked against
the same twin in tests/test_gpu_batchrl_conti.py."""
import math

import numpy as np
import pytest
import torch


def conti_dataset(K=266, D=32, E=40, L=10, seed=0, reward_fn=None):
    """E episodes of L entries with continuous actions f32 [N, D]; terminal on the last entry of each episode."""
    rs = np.random.RandomState(seed)
    obs = rs.randn(E, L, K).astype(np.float32)
    act = rs.uniform(-1, 1, (E, L, D)).astype(np.float32)
    rew = rs.rand(E, L).astype(np.float32)
    if reward_fn is not None:
        rew[:, 1:] = reward_fn(act[:, :-1])
    rew[:, 0] = 0
    term = np.zeros((E, L), np.float32)
    term[:, -1] = 1
    return {"observations": obs.reshape(-1, K), "actions": act.reshape(-1, D), "rewards": rew.reshape(-1),
            "terminals": term.reshape(-1), "discrete_action": np.asarray(False)}


def _cfg(**kw):
    return dict({"action_size": 284, "action_emb_size": 32, "support_conti_env": True, "CQL_alpha": 1, "gpu": False}, **kw)


def _model(ds=None, cfg=None, **hp):
    from rl4rs_b200 import batchrl
    m = batchrl.get_model(cfg or _cfg(), "CQL-conti")
    m.hp.update(hp)
    m.batch_size = int(m.hp["batch_size"])
    assert m.device.type == "cpu" and not m.use_kernels
    if ds is not None:
        m.build_with_dataset(ds)
    return m


# ---- dispatch ----------------------------------------------------------------------------------------------
def test_dispatch_and_dataset_kind_errors():
    from rl4rs_b200 import batchrl, synth
    assert isinstance(batchrl.get_model(_cfg(), "CQL-conti"), batchrl.ContinuousCQL)
    assert type(batchrl.get_model(_cfg(), "BCQ-conti")) is batchrl.ContinuousBCQ
    for algo in ("BCQ-conti", "CQL-conti"):
        with pytest.raises(NotImplementedError, match=algo + ".*support_conti_env"):
            batchrl.get_model(_cfg(support_conti_env=False), algo)
    for algo in ("MOPO", "COMBO", "dynamics"):
        with pytest.raises(NotImplementedError, match=algo):
            batchrl.get_model(_cfg(), algo)
    # D: action_emb_size, or action_size with one-hot actions
    assert batchrl.get_model(_cfg(), "CQL-conti").D == 32
    assert batchrl.get_model(_cfg(support_onehot_action=True), "CQL-conti").D == 284
    # a discrete dataset given to the continuous model, and the other way round
    from test_batchrl_cpu import synthetic_dataset
    with pytest.raises(ValueError, match="continuous"):
        _model().fit(synthetic_dataset(E=2))
    dcfg = {"action_size": 284, "page_items": 9, "catalog": synth.make_catalog(), "gpu": False}
    with pytest.raises(ValueError):                   # the discrete learners' existing error
        batchrl.get_model(dcfg, "BC").fit(conti_dataset(E=2))


def test_cql_alpha_is_dropped_as_d3rlpy_drops_it():
    """d3rlpy 0.91's continuous CQL has no `alpha` argument; the script's CQL_alpha does not reach it: initial alpha 1."""
    for a in (1, 3):
        m = _model(conti_dataset(E=2), cfg=_cfg(CQL_alpha=a))
        p = m.net.params(m.net.flat.detach())
        assert float(p["log_alpha"]) == 0.0 and float(p["log_temp"]) == 0.0
        assert "alpha" not in m.hp


# ---- the noise ---------------------------------------------------------------------------------------------
def test_draws_are_keyed_without_collisions():
    from rl4rs_b200.policy import cqlc_draws
    a = cqlc_draws(5, 7, 1, 64, 10, 284)
    assert a.shape == (64, 10, 284)
    assert np.array_equal(a, cqlc_draws(5, 7, 1, 64, 10, 284))
    assert np.array_equal(a[:3, :2, :5], cqlc_draws(5, 7, 1, 3, 2, 5))
    assert len(np.unique(a)) == a.size          # every (row, sample, dim) its own draw at D = 284
    # the normal draws carry 48 bits of the key's hash (the uniform ones 24, so those repeat by chance): distinct across
    # streams and steps
    streams = [cqlc_draws(5, 7, s, 8, 10, 284).ravel() for s in (0, 1, 3, 5)] + [cqlc_draws(5, 8, 1, 8, 10, 284).ravel()]
    allv = np.concatenate(streams)
    assert len(np.unique(allv)) == allv.size
    u = cqlc_draws(1, 1, 2, 256, 10, 32)
    assert u.min() >= -1 and u.max() < 1 and abs(u.mean()) < 0.02
    z = cqlc_draws(1, 1, 3, 256, 10, 32)
    assert abs(z.mean()) < 0.02 and abs(z.std() - 1) < 0.02


# ---- the twin against NumPy float64 ------------------------------------------------------------------------
def _np(p):
    return {k: v.detach().double().numpy() for k, v in p.items()}


def _mlp(p, pre, x):
    h = np.maximum(x @ p[pre + "w1"] + p[pre + "b1"], 0)
    return np.maximum(h @ p[pre + "w2"] + p[pre + "b2"], 0) @ p[pre + "w3"] + p[pre + "b3"]


def _softplus(x):
    return np.maximum(x, 0) + np.log1p(np.exp(-np.abs(x)))


def _sample(mu, ls_raw, eps):
    ls = np.clip(ls_raw, -20, 2)
    u = mu + np.exp(ls) * eps
    lp = (-0.5 * eps ** 2 - ls - 0.5 * np.log(2 * np.pi) - 2 * (np.log(2) - u - _softplus(-2 * u))).sum(-1)
    return np.tanh(u), lp


def _lse(v):
    m = v.max(-1, keepdims=True)
    return (m + np.log(np.exp(v - m).sum(-1, keepdims=True)))[..., 0]


def test_losses_match_numpy_float64():
    K, D, n, S = 20, 3, 16, 10
    ds = conti_dataset(K, D, E=4, L=6)
    m = _model(ds, cfg=_cfg(action_emb_size=D), batch_size=n)
    net = m.net
    data = m._device_data(ds)
    batch = data.batch(torch.arange(n))
    noise = net.noise(3, 1, n, S, dtype=torch.float64)
    hp = m._hyper()
    flat = net.flat.detach().double()
    with torch.no_grad():
        net.target.add_(0.01)
    losses, st = net.losses(batch, noise, hp, flat)
    p = _np(net.params(flat))
    tp = _np(net.target_params(None, torch.float64))
    obs, act, rew, nobs, term = [t.double().numpy() for t in batch]
    nz = {k: v.numpy() for k, v in noise.items()}
    o = _mlp(p, "a_", obs)
    mu, ls = o[:, :D], o[:, D:]
    # temperature
    _, lp_t = _sample(mu, ls, nz["temp"])
    assert np.isclose(float(losses["temp"]), -(np.exp(p["log_temp"][0]) * (lp_t - D)).mean(), rtol=1e-10)
    # conservative term (critic's draws) and TD
    q = lambda x, a, k, pp=p: _mlp(pp, "q%d_" % k, np.concatenate([x, a], -1))[..., 0]

    def cons(pol, uni):
        ap, lpp = _sample(mu[:, None], ls[:, None], pol)
        xr = np.repeat(obs[:, None], S, 1)
        tot = 0
        for k in (0, 1):
            v = np.concatenate([q(xr, ap, k) - lpp, q(xr, uni, k) - D * np.log(0.5)], 1)
            tot = tot + hp["conservative_weight"] * (_lse(v) - q(obs, act, k)) - hp["alpha_threshold"]
        return min(np.exp(p["log_alpha"][0]), 1e6) * tot.mean()
    assert np.isclose(float(losses["alpha"]), -cons(nz["alpha_policy"], nz["alpha_uniform"]), rtol=1e-10)
    a2 = np.tanh(_mlp(p, "a_", nobs)[:, :D])
    y = (rew - hp["reward_mean"]) / hp["reward_den"] + hp["gamma"] * (1 - term) * np.minimum(q(nobs, a2, 0, tp), q(nobs, a2, 1, tp))
    td = sum(((q(obs, act, k) - y) ** 2).mean() for k in (0, 1))
    assert np.isclose(float(losses["critic"]), td + cons(nz["critic_policy"], nz["critic_uniform"]), rtol=1e-10)
    # actor
    a_pi, lp_pi = _sample(mu, ls, nz["actor"])
    ref = (np.exp(p["log_temp"][0]) * lp_pi - np.minimum(q(obs, a_pi, 0), q(obs, a_pi, 1))).mean()
    assert np.isclose(float(losses["actor"]), ref, rtol=1e-10)
    assert np.isclose(float(st[4]), q(obs, act, 0).mean(), rtol=1e-10)


def test_logsumexp_max_subtraction_and_squashed_log_prob_at_extremes():
    from rl4rs_b200.policy import BatchRLContiNet
    net = BatchRLContiNet(4, 2, "cpu")
    # a Q near 1e4 overflows a plain exp; the max-subtracted logsumexp stays finite and exact
    p = net.params(net.flat.detach().double())
    with torch.no_grad():
        p["q0_b3"].fill_(1e4)
        p["q1_b3"].fill_(1e4)
    hp = {"conservative_weight": 5.0, "alpha_threshold": 10.0}
    obs = torch.randn(3, 4, dtype=torch.float64)
    act = torch.zeros(3, 2, dtype=torch.float64)
    mu, ls = torch.zeros(3, 2, dtype=torch.float64), torch.zeros(3, 2, dtype=torch.float64)
    pol = torch.randn(3, 10, 2, dtype=torch.float64)
    uni = torch.rand(3, 10, 2, dtype=torch.float64) * 2 - 1
    c, rows = net.conservative(p, obs, act, mu, ls, pol, uni, hp)
    assert torch.isfinite(c) and torch.isfinite(rows).all()
    # the squash: tanh(u) and the Jacobian form agree with log(1 - tanh(u)^2) where that is finite; finite at large |u|
    mu = torch.tensor([[0.3, -1.2], [8.0, -9.0]], dtype=torch.float64)
    ls = torch.tensor([[-0.5, 0.4], [30.0, -30.0]], dtype=torch.float64)
    eps = torch.tensor([[0.7, -0.2], [0.1, 0.5]], dtype=torch.float64)
    a, lp = net.sample(mu, ls, eps)
    ref_a, ref_lp = _sample(mu.numpy(), ls.numpy(), eps.numpy())
    assert np.allclose(a.numpy(), ref_a) and np.allclose(lp.numpy(), ref_lp)
    u = mu[0] + ls[0].exp() * eps[0]
    direct = (torch.distributions.Normal(mu[0], ls[0].exp()).log_prob(u) - torch.log(1 - torch.tanh(u) ** 2)).sum()
    assert torch.isclose(lp[0], direct) and torch.isfinite(lp[1])


def test_soft_update_and_group_updates():
    """One twin step: each group moves by its own Adam, the target moves by tau toward the updated critics."""
    ds = conti_dataset(20, 3, E=6, L=6)
    m = _model(ds, cfg=_cfg(action_emb_size=3), batch_size=16)
    net = m.net
    before, tgt0 = net.flat.detach().clone(), net.target.clone()
    m.train_step_twin(m._device_data(ds).batch(torch.arange(16)))
    after = net.flat.detach()
    for name in ("actor", "critic", "temp", "alpha"):
        assert not torch.equal(before[net.group(name)], after[net.group(name)]), name
    crit = after[net.group("critic")]
    assert torch.allclose(net.target, 0.005 * crit + 0.995 * tgt0, atol=1e-7)


# ---- learning ----------------------------------------------------------------------------------------------
def test_predict_moves_toward_the_rewarded_action_and_q_stays_conservative():
    """A one-step dataset with reward -|a - a*|^2: 300 steps move predict toward a* (distance down by half or more), and
    CQL keeps Q at uniform-random actions below Q at the logged ones."""
    K, D = 8, 2
    target = np.array([0.5, -0.4], np.float32)
    rs = np.random.RandomState(1)
    E = 2048
    obs = rs.randn(E, 2, K).astype(np.float32)
    act = np.clip(target + 0.3 * rs.randn(E, 2, D), -0.99, 0.99).astype(np.float32)
    rew = np.zeros((E, 2), np.float32)
    rew[:, 1] = -((act[:, 0] - target) ** 2).sum(-1)
    term = np.zeros((E, 2), np.float32)
    term[:, 1] = 1
    ds = {"observations": obs.reshape(-1, K), "actions": act.reshape(-1, D), "rewards": rew.reshape(-1),
          "terminals": term.reshape(-1), "discrete_action": np.asarray(False)}
    m = _model(ds, cfg=_cfg(action_emb_size=D), batch_size=64, actor_learning_rate=1e-3, critic_learning_rate=1e-3)
    x = ds["observations"][::2][:256]
    d0 = np.linalg.norm(m.predict(x) - target, axis=1).mean()
    m.fit(ds, n_epochs=10)
    d1 = np.linalg.norm(m.predict(x) - target, axis=1).mean()
    assert d1 < 0.5 * d0, (d0, d1)
    q_logged = m.predict_value(x, ds["actions"][::2][:256]).mean()
    q_rand = m.predict_value(x, np.random.RandomState(2).uniform(-1, 1, (256, D)).astype(np.float32)).mean()
    assert q_rand < q_logged, (q_rand, q_logged)


# ---- checkpoints -------------------------------------------------------------------------------------------
# ---- the train / eval stages over the oracle-backed engine -------------------------------------------------
@pytest.fixture()
def oracle_engine(monkeypatch):
    import rl4rs_b200.engine as engine_mod
    from oracle_engine import OracleEngine
    monkeypatch.setattr(engine_mod, "Engine", OracleEngine)


def test_generate_fit_evaluate_end_to_end(oracle_engine, tmp_path):
    from test_gpu_parity import _synthetic
    from rl4rs_b200 import batchrl, dataset
    B = 8
    cfg, cat, log, w = _synthetic(B, False)
    cfg = dict(cfg, catalog=cat, log=log, weights=w, CQL_alpha=1, support_conti_env=True, gpu=False)
    np.random.seed(0)
    ds = dataset.data_generate_rl4rs_a_conti(cfg, str(tmp_path / "ds.npz"), epochs=4)
    ds = batchrl.load_dataset(str(tmp_path / "ds.npz"))
    assert ds["actions"].shape[1] == cfg["action_emb_size"] and not bool(ds["discrete_action"])
    m = batchrl.get_model(cfg, "CQL-conti")
    m.hp["batch_size"] = m.batch_size = 32
    hist = m.fit(ds, n_epochs=1)
    assert all(np.isfinite(v) for v in hist[-1][1].values())
    avg = batchrl.evaluate(cfg, batchrl.policy_model(m, cfg), batch_size=B, episodes=1)
    assert np.isfinite(avg)


# ---- BCQ-conti ---------------------------------------------------------------------------------------------
def _bcq(ds=None, D=32, **hp):
    from rl4rs_b200 import batchrl
    m = batchrl.get_model(_cfg(action_emb_size=D), "BCQ-conti")
    m.hp.update(hp)
    m.batch_size = int(m.hp["batch_size"])
    assert m.device.type == "cpu" and not m.use_kernels
    if ds is not None:
        m.build_with_dataset(ds)
    return m


def test_bcq_losses_match_numpy_float64():
    """The VAE loss and KL, the perturbation and its clamp, the lambda-mixed max over the sampled actions, the actor loss."""
    K, D, n, S, L = 12, 3, 8, 100, 4
    ds = conti_dataset(K, D, E=4, L=5)
    m = _bcq(ds, D, batch_size=n, latent_size=L)
    net, hp = m.net, m._hyper()
    with torch.no_grad():
        net.target.add_(0.01)
    batch = m._device_data(ds).batch(torch.arange(n))
    noise = net.noise(3, 1, n, S, dtype=torch.float64)
    flat = net.flat.detach().double()
    losses, st = net.losses(batch, noise, hp, flat)
    p, tp = _np(net.params(flat)), _np(net.target_params(None, torch.float64))
    obs, act, rew, nobs, term = [t.double().numpy() for t in batch]
    nz = {k: v.numpy() for k, v in noise.items()}
    cat = lambda x, a: np.concatenate([x, a], -1)
    e = _mlp(p, "e_", cat(obs, act))
    mu, ls = e[:, :L], np.clip(e[:, L:], -20, 2)
    rec = np.tanh(_mlp(p, "d_", cat(obs, mu + np.exp(ls) * nz["vae"])))
    kl = (-ls + 0.5 * (np.exp(2 * ls) + mu ** 2) - 0.5).mean()
    assert np.isclose(float(losses["imitator"]), ((rec - act) ** 2).mean() + 0.5 * kl, rtol=1e-10)
    assert np.isclose(float(st[4]), ((rec - act) ** 2).mean(), rtol=1e-10)
    pert = lambda pp, x, a: np.clip(a + 0.05 * np.tanh(_mlp(pp, "a_", cat(x, a))), -1, 1)
    xr = np.repeat(nobs[:, None], S, 1)
    a_dec = np.tanh(_mlp(p, "d_", cat(xr, np.clip(nz["target"], -0.5, 0.5))))
    cand = pert(tp, xr, a_dec)
    qa, qb = _mlp(tp, "q0_", cat(xr, cand))[..., 0], _mlp(tp, "q1_", cat(xr, cand))[..., 0]
    v = (0.75 * np.minimum(qa, qb) + 0.25 * np.maximum(qa, qb)).max(1)
    y = rew + 0.99 * (1 - term) * v
    td = sum(((_mlp(p, "q%d_" % k, cat(obs, act))[:, 0] - y) ** 2).mean() for k in (0, 1))
    assert np.isclose(float(losses["critic"]), td, rtol=1e-10)
    a_s = np.tanh(_mlp(p, "d_", cat(obs, np.clip(nz["actor"], -0.5, 0.5))))
    assert np.isclose(float(losses["actor"]), -_mlp(p, "q0_", cat(obs, pert(p, obs, a_s)))[:, 0].mean(), rtol=1e-10)
    # the clamp of the perturbation: a base action at the edge stays inside [-1, 1]
    big = net.perturb(net.params(flat), "a_", torch.zeros(2, K, dtype=torch.float64),
                      torch.tensor([[1.0] * D, [-1.0] * D], dtype=torch.float64), 0.05)
    assert float(big.abs().max()) <= 1.0


def test_bcq_vae_learns_and_predict_moves_toward_the_rewarded_action():
    """One-step data with reward -|a - a*|^2 and logged actions around a*: the VAE reconstruction error falls by half or
    more, and predict's distance to a* falls by half or more."""
    K, D = 8, 2
    target = np.array([0.5, -0.4], np.float32)
    rs = np.random.RandomState(1)
    E = 1024
    obs = rs.randn(E, 2, K).astype(np.float32)
    act = np.clip(target + 0.3 * rs.randn(E, 2, D), -0.99, 0.99).astype(np.float32)
    rew = np.zeros((E, 2), np.float32)
    rew[:, 1] = -((act[:, 0] - target) ** 2).sum(-1)
    term = np.zeros((E, 2), np.float32)
    term[:, 1] = 1
    ds = {"observations": obs.reshape(-1, K), "actions": act.reshape(-1, D), "rewards": rew.reshape(-1),
          "terminals": term.reshape(-1), "discrete_action": np.asarray(False)}
    m = _bcq(ds, D, batch_size=64, n_action_samples=20)
    x = ds["observations"][::2][:256]
    batch = m._device_data(ds).batch(torch.arange(512))
    noise = m.net.noise(9, 1, 512, 20)
    mse = lambda: float(m.net.losses(batch, noise, m._hyper())[1][4])
    r0, d0 = mse(), np.linalg.norm(m.predict(x) - target, axis=1).mean()
    m.fit(ds, n_epochs=6)
    r1, d1 = mse(), np.linalg.norm(m.predict(x) - target, axis=1).mean()
    assert r1 < 0.5 * r0, (r0, r1)
    assert d1 < 0.5 * d0, (d0, d1)


@pytest.mark.parametrize("algo", ["BCQ-conti", "CQL-conti"])
def test_save_load_then_identical_predict_and_continued_fit(algo, tmp_path):
    from rl4rs_b200 import batchrl
    ds = conti_dataset(20, 3, E=20, L=6)
    def mk():
        m = batchrl.get_model(_cfg(action_emb_size=3), algo)
        m.hp.update(n_action_samples=10, batch_size=16)
        m.batch_size = 16
        return m
    m = mk()
    m.fit(ds, n_epochs=1)
    path = str(tmp_path / "m.pt")
    m.save_model(path)
    m2 = mk()
    m2.load_model(path)
    x = ds["observations"][:50]
    assert np.array_equal(m.predict(x), m2.predict(x))
    assert np.array_equal(m.predict_value(x, ds["actions"][:50]), m2.predict_value(x, ds["actions"][:50]))
    h1, h2 = m.fit(ds, n_epochs=1), m2.fit(ds, n_epochs=1)
    assert h1 == h2 and torch.equal(m.net.flat, m2.net.flat) and torch.equal(m.net.target, m2.net.target)
    assert torch.equal(m.m, m2.m) and m.step == m2.step


def test_bcq_generate_fit_evaluate_end_to_end(oracle_engine, tmp_path):
    from test_gpu_parity import _synthetic
    from rl4rs_b200 import batchrl, dataset
    B = 8
    cfg, cat, log, w = _synthetic(B, False)
    cfg = dict(cfg, catalog=cat, log=log, weights=w, support_conti_env=True, gpu=False)
    np.random.seed(0)
    ds = dataset.data_generate_rl4rs_a_conti(cfg, None, epochs=4)
    m = batchrl.get_model(cfg, "BCQ-conti")
    m.hp["batch_size"] = m.batch_size = 32
    hist = m.fit(ds, n_epochs=1)
    assert all(np.isfinite(v) for v in hist[-1][1].values())
    assert np.isfinite(batchrl.evaluate(cfg, batchrl.policy_model(m, cfg), batch_size=B, episodes=1))
