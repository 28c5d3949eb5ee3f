"""CPU: RAINBOW on the discrete env -- the get_rl_model dispatch, the parameter layout and init, the dueling distributional
forward, the projection and loss against NumPy float64, the n-step store, the per-tensor gradient clip, learning on a fake
env with the hard target schedule, checkpoints, and the world-size-2 learner over gloo."""
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from rl4rs_b200.policy import DistributionalQNetwork
from rl4rs_b200.trainer import RainbowTrainer, ReplayBuffer, get_rl_model

A, Z = 284, 8


class FakeEnv(object):
    """Torch-format env protocol on CPU with the plain observation (support_rllib_mask off): random obs [B, 256], reward 1
    per step for an even action, done on the last step."""

    def __init__(self, B, T=9, seed=0, **flags):
        self.config = dict({"max_steps": T, "batch_size": B, "action_size": A, "support_rllib_mask": False}, **flags)
        self.B, self.T = B, T
        self.g = torch.Generator().manual_seed(seed)
        self.sim = type("S", (), {"engine": type("E", (), {"device": torch.device("cpu")})()})()

    def reset(self):
        self.t = 0
        return torch.randn(self.B, 256, generator=self.g)

    def step(self, a):
        assert a.dtype == torch.int32 and a.shape == (self.B,)
        self.t += 1
        r = (a.to(torch.int64) % 2 == 0).to(torch.float32)
        return torch.randn(self.B, 256, generator=self.g), r, torch.full((self.B,), int(self.t >= self.T)), {}


def test_dispatch_and_errors():
    assert type(get_rl_model("RAINBOW", {}, env=FakeEnv(8), device="cpu")) is RainbowTrainer
    with pytest.raises(ValueError, match="support_rllib_mask"):
        get_rl_model("RAINBOW", {}, env=FakeEnv(8, support_rllib_mask=True), device="cpu")
    with pytest.raises(ValueError, match="support_conti_env"):
        get_rl_model("RAINBOW", {}, env=FakeEnv(8, support_conti_env=True), device="cpu")
    with pytest.raises(NotImplementedError):
        get_rl_model("RAINBOW_rawstate", {}, env=FakeEnv(8), device="cpu")
    with pytest.raises(NotImplementedError):
        get_rl_model("RAINBOW", {}, env=FakeEnv(8, rawstate_as_obs=True), device="cpu")
    for algo in ("DQN", "DQN_rawstate", "DDPG_conti", "SLATEQ", "RAINBOW_conti"):
        with pytest.raises(NotImplementedError):
            get_rl_model(algo, {}, env=FakeEnv(8), device="cpu")


def test_defaults_layout_and_init():
    tr = get_rl_model("RAINBOW", {"no_such_key": 1}, env=FakeEnv(200), device="cpu")
    c = tr.config
    assert (c["lr"], c["n_step"], c["num_atoms"], c["v_min"], c["v_max"], c["grad_clip"]) == (5e-4, 3, 8, 0.0, 1000.0, 40.0)
    assert (c["buffer_size"], c["learning_starts"], c["target_network_update_freq"]) == (100000, 1000, 500)
    assert tr.n_local == 1024 and tr.replay.prio is not None and tr.replay.action.dtype == torch.int32
    assert get_rl_model("RAINBOW", {}, env=FakeEnv(8), device="cpu").n_local == 72
    pol = tr.policy
    n = (256 * 256 + 256) * 2 + (256 * 128 + 128) * 2 + 128 * A * Z + A * Z + 128 * Z + Z
    assert pol.n_params == n == 491496 and len(pol.slices) == 12
    from rl4rs_b200 import _capi
    lib = _capi.load_library()
    assert lib.r4_rainbow_num_params(A, Z) == pol.n_params and lib.r4_rainbow_num_params(A, 33) == -1
    assert lib.r4_rainbow_scratch_size(A, Z, 576) > 576 * A * Z
    p = {k: v.detach() for k, v in pol.params().items()}
    for k in ("w1", "w2"):                                   # normc(1.0): unit column norms
        assert torch.allclose(p[k].norm(dim=0), torch.ones(256), atol=1e-5)
    for k, (fi, fo) in (("aw1", (256, 128)), ("aw2", (128, A * Z)), ("sw1", (256, 128)), ("sw2", (128, Z))):
        lim = (6.0 / (fi + fo)) ** 0.5                       # glorot uniform: |w| <= lim, variance lim^2 / 3
        assert float(p[k].abs().max()) <= lim and float(p[k].abs().max()) > 0.9 * lim
        assert abs(float(p[k].var()) - lim ** 2 / 3) < 0.1 * lim ** 2 / 3
    assert all(bool((p[k] == 0).all()) for k in ("b1", "b2", "ab1", "ab2", "sb1", "sb2"))
    assert torch.equal(pol.target, pol.flat.detach())
    assert torch.allclose(pol.z, torch.linspace(0, 1000, Z))


def _np_params(pol, flat=None):
    return {k: v.detach().double().numpy() for k, v in pol.params(flat).items()}


def _np_forward(p, obs, v_min=0.0, v_max=1000.0):
    h = np.tanh(np.tanh(obs @ p["w1"] + p["b1"]) @ p["w2"] + p["b2"])
    adv = (np.maximum(h @ p["aw1"] + p["ab1"], 0) @ p["aw2"] + p["ab2"]).reshape(len(obs), A, Z)
    score = np.maximum(h @ p["sw1"] + p["sb1"], 0) @ p["sw2"] + p["sb2"]
    logits = score[:, None, :] + adv - adv.mean(1, keepdims=True)
    e = np.exp(logits - logits.max(-1, keepdims=True))
    prob = e / e.sum(-1, keepdims=True)
    z = v_min + np.arange(Z) * (v_max - v_min) / (Z - 1)
    return logits, (prob * z).sum(-1)


def test_forward_matches_numpy():
    pol = DistributionalQNetwork(A, "cpu", seed=3)
    with torch.no_grad():
        pol.flat.add_(0.05 * torch.randn(pol.n_params, generator=torch.Generator().manual_seed(0)))
    obs = torch.randn(5, 256, generator=torch.Generator().manual_seed(1))
    logits, q = pol.forward(obs)
    rl, rq = _np_forward(_np_params(pol), obs.double().numpy())
    assert logits.shape == (5, A, Z) and q.shape == (5, A)
    np.testing.assert_allclose(logits.detach().numpy(), rl, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(q.detach().numpy(), rq, rtol=1e-4, atol=1e-3)


def _np_project(r, done, pt, gamma_n, v_min, v_max):
    dz = (v_max - v_min) / (Z - 1)
    z = v_min + np.arange(Z) * dz
    m = np.zeros_like(pt)
    for i in range(len(r)):
        for j in range(Z):
            rt = min(max(r[i] + gamma_n * (1 - done[i]) * z[j], v_min), v_max)
            b = (rt - v_min) / dz
            lb, ub = np.floor(b), np.ceil(b)
            m[i, int(lb)] += pt[i, j] * (ub - b + (1.0 if ub - lb < 0.5 else 0.0))
            m[i, int(ub)] += pt[i, j] * (b - lb)
    return m


def test_projection_edge_cases():
    pol = DistributionalQNetwork(A, "cpu", seed=0, v_min=-10.0, v_max=60.0)            # dz = 10: atoms at -10, 0, .., 60
    pt = torch.softmax(torch.randn(6, Z, generator=torch.Generator().manual_seed(2)), -1)
    r = torch.tensor([20.0, 3.5, -500.0, 500.0, 7.0, 0.0])
    done = torch.tensor([0, 0, 0, 0, 1, 1], dtype=torch.uint8)
    m = pol.project(r, done, pt, 1.0)
    ref = _np_project(r.double().numpy(), done.numpy(), pt.double().numpy(), 1.0, -10.0, 60.0)
    np.testing.assert_allclose(m.numpy(), ref, rtol=1e-6, atol=1e-7)
    assert torch.allclose(m.sum(1), torch.ones(6))
    # r = 20: b lands exactly on atoms (floor == ceil): each atom's mass moves two atoms up, the top three pile on v_max
    assert torch.allclose(m[0, 2:5], pt[0, :3]) and torch.allclose(m[0, 7], pt[0, 5:].sum())
    assert float(m[2, 0]) == pytest.approx(1.0) and float(m[3, 7]) == pytest.approx(1.0)   # clipped at both ends
    # done: the whole distribution collapses onto r, split between the neighbouring atoms (7 = 0.7 * 10 + 0.3 * 0)
    assert m[4, 1] == pytest.approx(0.3) and m[4, 2] == pytest.approx(0.7) and m[5, 1] == pytest.approx(1.0)


def test_loss_matches_numpy_with_double_q():
    pol = DistributionalQNetwork(A, "cpu", seed=5, v_max=10.0)
    g = torch.Generator().manual_seed(4)
    with torch.no_grad():
        pol.flat.add_(0.2 * torch.randn(pol.n_params, generator=g))
        pol.target.add_(0.5 * torch.randn(pol.n_params, generator=g))
    n = 12
    obs, nobs = torch.randn(n, 256, generator=g), torch.randn(n, 256, generator=g)
    act = torch.randint(0, A, (n,), generator=g, dtype=torch.int32)
    rew = torch.rand(n, generator=g) * 4
    done = (torch.rand(n, generator=g) < 0.3).to(torch.uint8)
    w = torch.rand(n, generator=g) + 0.5
    loss, td = pol.loss(obs, act, rew, nobs, done, w, 1.0, 1.0 / n)
    p, pt_ = _np_params(pol), _np_params(pol, pol.target)
    o, no = obs.double().numpy(), nobs.double().numpy()
    a_star = _np_forward(p, no, 0, 10)[1].argmax(1)
    assert (a_star != _np_forward(pt_, no, 0, 10)[1].argmax(1)).any()     # the online argmax is not the target's
    lt = _np_forward(pt_, no, 0, 10)[0][np.arange(n), a_star]
    pt = np.exp(lt - lt.max(-1, keepdims=True))
    pt /= pt.sum(-1, keepdims=True)
    m = _np_project(rew.double().numpy(), done.numpy(), pt, 1.0, 0.0, 10.0)
    sel = _np_forward(p, o, 0, 10)[0][np.arange(n), act.numpy()]
    logp = sel - sel.max(-1, keepdims=True)
    logp -= np.log(np.exp(logp).sum(-1, keepdims=True))
    rtd = -(m * logp).sum(-1)
    np.testing.assert_allclose(td.numpy(), rtd, rtol=1e-4, atol=1e-5)
    assert float(loss.detach()) == pytest.approx(float((w.double().numpy() * rtd).mean()), rel=1e-4)
    loss.backward()
    assert float(pol.flat.grad.abs().max()) > 0


def test_nstep_store_matches_numpy():
    g = torch.Generator().manual_seed(1)
    for T, B, C in ((9, 5, 100), (36, 3, 70)):
        gamma = 0.9
        rb = ReplayBuffer(C, None, torch.device("cpu"), True, alpha=0.6, n_step=3, gamma=gamma)
        ref_obs, ref_new, ref_r, ref_d, ref_a = (np.zeros((C, 256)), np.zeros((C, 256)), np.zeros(C), np.zeros(C),
                                                 np.zeros(C, np.int64))
        added = 0
        for ep in range(3):                            # 135 / 324 rows into 100 / 70 slots: wraps around
            obs, fin = torch.randn(T, B, 256, generator=g), torch.randn(B, 256, generator=g)
            act = torch.randint(0, A, (T, B), generator=g, dtype=torch.int32)
            rew = torch.randn(T, B, generator=g)
            done = torch.zeros(T, B, dtype=torch.uint8)
            done[-1] = 1
            rb.store(obs, fin, act, rew, done)
            nxt = np.concatenate([obs[1:].numpy(), fin[None].numpy()]).astype(np.float64)
            for t in range(T):
                for b in range(B):
                    s = (added + t * B + b) % C
                    t2 = min(t + 2, T - 1)
                    ref_obs[s], ref_new[s], ref_d[s], ref_a[s] = obs[t, b].numpy(), nxt[t2, b], done[t2, b], act[t, b]
                    ref_r[s] = sum(gamma ** j * float(rew[t + j, b]) for j in range(3) if t + j < T)
            added += T * B
            N = rb.size
            assert N == min(added, C)
            np.testing.assert_array_equal(rb.obs[:N].numpy(), ref_obs[:N].astype(np.float32))
            np.testing.assert_array_equal(rb.new_obs[:N].numpy(), ref_new[:N].astype(np.float32))
            np.testing.assert_array_equal(rb.action[:N].numpy(), ref_a[:N])
            np.testing.assert_array_equal(rb.done[:N].numpy(), ref_d[:N])
            np.testing.assert_allclose(rb.reward[:N].numpy(), ref_r[:N], rtol=1e-5, atol=1e-6)
        # the last n steps of an episode reach its end (the final obs, done = 1); the earlier ones do not
        last = torch.tensor([(added - B * k + b) % C for k in (1, 2, 3) for b in range(B)])
        earlier = torch.tensor([(added - B * k + b) % C for k in (4, 5) for b in range(B)])
        assert bool((rb.done[last] == 1).all()) and bool((rb.done[earlier] == 0).all())
        assert torch.equal(rb.new_obs[last], fin.repeat(3, 1))


def test_per_tensor_gradient_clip():
    pol = DistributionalQNetwork(A, "cpu", seed=0)
    g = torch.zeros(pol.n_params)
    norms = [100.0, 1.0, 39.0, 40.5, 3.0, 0.0, 400.0, 10.0, 41.0, 0.5, 2.0, 80.0]
    gen = torch.Generator().manual_seed(0)
    for (lo, hi), nrm in zip(pol.slices, norms):
        x = torch.randn(hi - lo, generator=gen)
        g[lo:hi] = x / x.norm() * nrm
    before = g.clone()
    pol.clip_per_tensor(g, 40.0)
    for (lo, hi), nrm in zip(pol.slices, norms):
        if nrm > 40:
            assert float(g[lo:hi].norm()) == pytest.approx(40.0, rel=1e-5)
            assert torch.allclose(g[lo:hi], before[lo:hi] * (40.0 / float(before[lo:hi].norm())), rtol=1e-5)
        else:
            assert torch.equal(g[lo:hi], before[lo:hi])


def test_learning_target_schedule_and_checkpoint():
    torch.manual_seed(0)
    B = 8
    cfg = {"lr": 1e-3, "v_max": 10.0, "learning_starts": B * 9 * 2, "buffer_size": 2000, "timesteps_per_iteration": B * 9 * 4,
           "train_batch_size": 128}
    env = FakeEnv(B, seed=3)
    tr = get_rl_model("RAINBOW", cfg, env=env, device="cpu")
    before = tr.evaluate(3)
    res = [tr.train() for _ in range(25)]
    assert res[0]["sgd_steps"] == 3 and all(r["sgd_steps"] == 4 for r in res[1:])      # none before learning_starts
    assert res[-1]["timesteps_total"] == 25 * 4 * B * 9 and res[-1]["replay_size"] == 2000
    assert np.isfinite(res[-1]["loss"]) and res[-1]["loss"] < res[0]["loss"]
    after = tr.evaluate(3)
    assert after > before + 2.0 and after >= 7.0, (before, after)    # 9 even actions in 9 steps is the best; chance 4.5
    # the hard copy: exactly after the steps at which 500 timesteps were sampled since the last copy
    copies = []
    batch = tr.replay.gather(torch.arange(128))
    for _ in range(12):
        tr.policy_ts += 72                                    # one 8 x 9 episode sampled per step
        t0, last = tr.policy.target.clone(), tr.last_target_update
        tr.sgd_step(torch.rand(128))
        copied = not torch.equal(tr.policy.target, t0)
        assert copied == (tr.policy_ts - last >= 500)
        if copied:
            assert torch.equal(tr.policy.target, tr.policy.flat.detach()) and tr.last_target_update == tr.policy_ts
            copies.append(tr.policy_ts)
    assert len(copies) >= 1 and all(b - a >= 500 for a, b in zip(copies, copies[1:]))
    d = tempfile.mkdtemp()
    path = tr.save(d)
    tr2 = get_rl_model("RAINBOW", cfg, env=FakeEnv(B, seed=3), device="cpu")
    tr2.restore(path)
    assert torch.equal(tr2.policy.flat, tr.policy.flat) and torch.equal(tr2.policy.target, tr.policy.target)
    assert (tr2.critic_steps, tr2.policy_ts, tr2.last_target_update, tr2.iteration, tr2.counter) == \
        (tr.critic_steps, tr.policy_ts, tr.last_target_update, tr.iteration, tr.counter)
    assert tr2.replay.size == 0
    o = env.reset()
    a = tr.compute_actions(o)
    assert a.shape == (B,) and a.dtype == np.int32 and a.min() >= 0 and a.max() < A
    np.testing.assert_array_equal(a, tr2.compute_actions({"obs": o.numpy()}))
    np.testing.assert_array_equal(a, tr.policy.forward(o)[1].argmax(1).numpy())
    rl = tr.compute_actions({i: o[i].numpy() for i in range(3)})
    assert sorted(rl) == [0, 1, 2] and all(rl[i] == a[i] for i in range(3))
    # SoftQ: reproducible from (seed, counter)
    c0 = tr.counter
    e1 = tr.compute_actions(o, explore=True)
    tr.counter = c0
    np.testing.assert_array_equal(e1, tr.compute_actions(o, explore=True))
    # both take one more step identically after the restore (Adam's state came back)
    for t in (tr, tr2):
        t.critic_steps += 1
        t.twin_step(*batch, None, False)
    assert torch.equal(tr2.policy.flat, tr.policy.flat)
    from test_trainer_conti_cpu import FakeContiEnv
    with pytest.raises(AssertionError):
        get_rl_model("DDPG", {}, env=FakeContiEnv(B), device="cpu").restore(path)


def test_softq_sampling_follows_softmax():
    pol = DistributionalQNetwork(A, "cpu", seed=1, v_max=3.0)     # Q in [0, 3]: softmax(Q) far from one-hot
    obs = torch.randn(1, 256).repeat(20000, 1)
    a, q = pol.act(obs, True, seed=7, counter=0)
    p = torch.softmax(q[0].double(), 0).numpy()
    freq = np.bincount(a.numpy(), minlength=A) / len(a)
    assert np.abs(freq - p).max() < 5 * np.sqrt(p.max() / len(a))
    assert torch.equal(a, pol.act(obs, True, seed=7, counter=0)[0]) and not torch.equal(a, pol.act(obs, True, 8, 0)[0])


def _worker(rank, world, init_file, out_dir):
    dist.init_process_group("gloo", init_method="file://" + init_file, rank=rank, world_size=world)
    tr = get_rl_model("RAINBOW", {"grad_clip": 0.05, "v_max": 10.0}, env=FakeEnv(8), device="cpu")
    batch = _batch(32, 9)
    per = 32 // world
    half = [x[rank * per:(rank + 1) * per] for x in batch]
    for step in range(2):
        tr.critic_steps += 1
        tr.twin_step(*half, torch.linspace(0.5, 1.5, 32)[rank * per:(rank + 1) * per], step == 0)
    torch.save({"flat": tr.policy.flat.detach(), "target": tr.policy.target}, os.path.join(out_dir, "r%d.pt" % rank))
    dist.destroy_process_group()


def _batch(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, 256, generator=g), torch.randint(0, A, (n,), generator=g, dtype=torch.int32),
            torch.rand(n, generator=g) * 5, torch.randn(n, 256, generator=g), (torch.rand(n, generator=g) < 0.3).to(torch.uint8))


def test_world_size_2_gloo_matches_single_learner():
    """Two ranks with half of a fixed batch each (and their halves of the weights) end on the parameters of one learner
    given the whole batch; the per-tensor clip (0.05 here, so it acts) sees the summed gradient."""
    d = tempfile.mkdtemp()
    mp.spawn(_worker, args=(2, os.path.join(d, "init"), d), nprocs=2, join=True)
    r0, r1 = torch.load(os.path.join(d, "r0.pt")), torch.load(os.path.join(d, "r1.pt"))
    assert torch.equal(r0["flat"], r1["flat"]) and torch.equal(r0["target"], r1["target"])
    single = get_rl_model("RAINBOW", {"grad_clip": 0.05, "v_max": 10.0}, env=FakeEnv(8), device="cpu")
    p0 = single.policy.flat.detach().clone()
    batch = _batch(32, 9)
    for step in range(2):
        single.critic_steps += 1
        single.twin_step(*batch, torch.linspace(0.5, 1.5, 32), step == 0)
    p = single.policy.flat.detach()
    assert (p - p0).abs().max() > 1e-4
    assert torch.allclose(r0["flat"], p, atol=2e-6) and torch.allclose(r0["target"], single.policy.target, atol=2e-6)
