"""CPU: DDPG / TD3 on the continuous-action env -- the get_rl_model dispatch, the exploration defaults (the DDPG quirk, OU,
TD3's random phase), the losses against the table's formulas, the torch replay against a NumPy float64 oracle, learning on
a fake continuous env, checkpoints, and the world-size-2 learner over gloo."""
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from rl4rs_b200.policy import DeterministicActorCritic
from rl4rs_b200.trainer import DDPGTrainer, ReplayBuffer, TD3Trainer, get_rl_model
from test_trainer_conti_cpu import FakeContiEnv
from test_trainer_cpu import FakeEnv

D = 32
OU = {"type": "OrnsteinUhlenbeckNoise"}


def test_dispatch_and_errors():
    conti = FakeContiEnv(8)
    assert type(get_rl_model("DDPG", {}, env=conti, device="cpu")) is DDPGTrainer
    assert type(get_rl_model("TD3", {}, env=conti, device="cpu")) is TD3Trainer
    for algo in ("DDPG", "TD3"):
        with pytest.raises(ValueError, match="support_conti_env"):
            get_rl_model(algo, {}, env=FakeEnv(8), device="cpu")
        masked = FakeContiEnv(8); masked.config["support_rllib_mask"] = True
        with pytest.raises(ValueError, match="support_rllib_mask"):
            get_rl_model(algo, {}, env=masked, device="cpu")
        with pytest.raises(NotImplementedError):
            get_rl_model(algo + "_rawstate", {}, env=conti, device="cpu")
    with pytest.raises(NotImplementedError):
        get_rl_model("DDPG_conti", {}, env=conti, device="cpu")
    with pytest.raises(NotImplementedError):
        get_rl_model("DQN", {}, env=FakeEnv(8))


def test_defaults_and_layout():
    tr = get_rl_model("TD3", {"no_such_key": 1}, env=FakeContiEnv(8), device="cpu")
    c = tr.config
    assert (c["tau"], c["l2_reg"], c["policy_delay"], c["buffer_size"], c["learning_starts"]) == (0.005, 0.0, 2, 10 ** 6, 10 ** 4)
    assert tr.ou["random_timesteps"] == 10000 and tr.n_local == min(8 * 9, 1024) and tr.replay.prio is None
    dd = get_rl_model("DDPG", {}, env=FakeContiEnv(200), device="cpu")
    assert dd.ou is None and dd.n_local == 1024 and dd.replay.prio is not None and dd.config["tau"] == 0.002
    pol = dd.policy
    actor = 256 * 400 + 400 + 400 * 300 + 300 + 300 * D + D
    critic = 288 * 400 + 400 + 400 * 300 + 300 + 300 + 1
    assert pol.n_actor == actor and pol.n_params == actor + critic and tr.policy.n_params == actor + 2 * critic
    from rl4rs_b200 import _capi
    lib = _capi.load_library()
    assert lib.r4_ddpg_num_params(D, 0) == pol.n_params and lib.r4_ddpg_num_params(D, 1) == tr.policy.n_params
    p = pol.params()
    lim = (6.0 / (256 + 400)) ** 0.5
    p = {k: v.detach() for k, v in p.items()}
    assert float(p["a_w1"].abs().max()) <= lim and float(p["a_w1"].abs().max()) > 0.95 * lim
    assert all(bool((p[k] == 0).all()) for k in ("a_b1", "a_b3", "q1_b1", "q1_b3"))
    assert torch.equal(pol.target, pol.flat.detach())


def test_exploration_defaults():
    obs = FakeContiEnv(16).reset()
    dd = get_rl_model("DDPG", {}, env=FakeContiEnv(16), device="cpu")
    assert np.array_equal(dd.compute_actions(obs, explore=True), dd.compute_actions(obs, explore=False))    # the quirk
    ou = get_rl_model("DDPG", {"exploration_config": dict(OU, random_timesteps=0)}, env=FakeContiEnv(16), device="cpu")
    ou.policy_ts = 1
    det = ou.compute_actions(obs, explore=False)
    noise = []
    for _ in range(3):
        x0 = ou.ou_state[ou._ou_slot].clone()
        a = ou.compute_actions(obs, explore=True)
        x1 = ou.ou_state[ou._ou_slot]
        assert not np.allclose(a, det)
        d = a - det                                          # every row carries the same noise vector (no clipping here)
        assert np.allclose(d, d[:1], atol=1e-5)
        # the recurrence x' = x + theta (-x) + sigma N: x' - 0.85 x is sigma times a standard normal draw
        noise.append(((x1 - 0.85 * x0) / 0.2).numpy())
    z = np.concatenate(noise)
    assert abs(z.mean()) < 0.5 and 0.6 < z.std() < 1.5
    td3 = get_rl_model("TD3", {}, env=FakeContiEnv(4000), device="cpu")
    a = td3.compute_actions(torch.zeros(4000, 256), explore=True)
    assert td3.policy_ts <= 10000 and a.min() >= -1 and a.max() < 1
    n = a.size                                               # U(-1, 1): mean 0, variance 1/3
    assert abs(a.mean()) < 5 * (1 / 3 / n) ** 0.5 and abs(a.var() - 1 / 3) < 5 * (4 / 45 / n) ** 0.5
    assert not np.allclose(a, td3.compute_actions(torch.zeros(4000, 256), explore=False))


def _batch(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, 256, generator=g), torch.rand(n, D, generator=g) * 2 - 1, torch.randn(n, generator=g),
            torch.randn(n, 256, generator=g), (torch.rand(n, generator=g) < 0.3).to(torch.uint8))


@pytest.mark.parametrize("twin", [False, True])
def test_losses_equal_the_formulas(twin):
    torch.manual_seed(0)
    pol = DeterministicActorCritic(D, "cpu", seed=2, twin=twin)
    with torch.no_grad():
        pol.target.add_(0.01 * torch.randn(pol.n_params))
    obs, act, rew, nobs, done = _batch(6)
    w = torch.rand(6) + 0.5
    eps = torch.randn(6, D)
    gamma = 0.9
    cl, al, td = pol.losses(obs, act, rew, nobs, done, w, eps if twin else None, gamma)
    p, t = pol.params(), pol.params(pol.target)

    def mlp(q, pre, x):
        return torch.relu(torch.relu(x @ q[pre + "w1"] + q[pre + "b1"]) @ q[pre + "w2"] + q[pre + "b2"]) @ q[pre + "w3"] + q[pre + "b3"]
    a2 = 2 * torch.sigmoid(2 * mlp(t, "a_", nobs)) - 1                            # (high - low) sigmoid(2x) + low
    if twin:
        a2 = (a2 + (0.2 * eps).clamp(-0.5, 0.5)).clamp(-1, 1)
    qt = mlp(t, "q1_", torch.cat([nobs, a2], 1)).squeeze(-1)
    if twin:
        qt = torch.min(qt, mlp(t, "q2_", torch.cat([nobs, a2], 1)).squeeze(-1))
    y = rew + gamma * (1 - done.float()) * qt
    td1 = mlp(p, "q1_", torch.cat([obs, act], 1)).squeeze(-1) - y
    err = 0.5 * td1 ** 2
    if twin:
        err = err + 0.5 * (mlp(p, "q2_", torch.cat([obs, act], 1)).squeeze(-1) - y) ** 2
    assert torch.allclose(cl, (w * err).mean(), rtol=1e-5) and torch.allclose(td, td1.detach(), atol=1e-5)
    api = 2 * torch.sigmoid(2 * mlp(p, "a_", obs)) - 1
    assert torch.allclose(al, -mlp(p, "q1_", torch.cat([obs, api], 1)).mean(), rtol=1e-5, atol=1e-6)
    # the actor loss reaches the actor weights only; the critic loss the critic weights only
    al.backward()
    assert float(pol.flat.grad[pol.n_actor:].abs().max()) == 0 and float(pol.flat.grad[:pol.n_actor].abs().max()) > 0
    pol.flat.grad = None
    cl.backward()
    assert float(pol.flat.grad[:pol.n_actor].abs().max()) == 0
    l2 = pol.l2_loss(1e-6)
    ref = sum(0.5 * 1e-6 * (v ** 2).sum() for k, v in p.items() if v.dim() == 2)
    assert torch.allclose(l2, ref)


# ---- replay against a NumPy float64 oracle ------------------------------------------------------------------------------
class NpReplay(object):
    def __init__(self, C, alpha):
        self.C, self.alpha, self.added, self.max_p = C, alpha, 0, 1.0
        self.obs, self.prio = np.zeros((C, 256)), np.zeros(C)

    def store(self, obs):                       # obs [n, 256], row order
        for r in range(len(obs)):
            s = (self.added + r) % self.C
            self.obs[s] = obs[r]
            self.prio[s] = self.max_p ** self.alpha
        self.added += len(obs)

    def sample(self, u, beta):
        N = min(self.added, self.C)
        p = self.prio[:N]
        idx = []
        for x in u:                             # RLlib find_prefixsum_idx
            mass, acc = x * p.sum(), 0.0
            for i in range(N):
                acc += p[i]
                if acc > mass:
                    break
            idx.append(i)
        idx = np.array(idx)
        pm = p.min() / p.sum()
        return idx, (p[idx] / p.sum() * N) ** -beta / (pm * N) ** -beta

    def update(self, idx, td, eps):
        for i, t in zip(idx, td):               # sequential: the later position wins
            self.prio[i] = (abs(t) + eps) ** self.alpha
            self.max_p = max(self.max_p, abs(t) + eps)


def test_replay_matches_numpy_oracle():
    g = torch.Generator().manual_seed(1)
    C, T, B = 50, 3, 8
    rb, ref = ReplayBuffer(C, D, torch.device("cpu"), True, alpha=0.6), NpReplay(C, 0.6)
    for ep in range(3):                         # 72 transitions into 50 slots: wraps around
        obs = torch.randn(T, B, 256, generator=g)
        fin = torch.randn(B, 256, generator=g)
        rb.store(obs, fin, torch.randn(T, B, D, generator=g), torch.randn(T, B, generator=g), torch.zeros(T, B, dtype=torch.uint8))
        ref.store(obs.reshape(-1, 256).numpy())
        if ep == 0:                             # new_obs: the next step's obs, the final obs on the last step
            assert torch.equal(rb.new_obs[:B], obs[1]) and torch.equal(rb.new_obs[2 * B:3 * B], fin)
        N = rb.size
        assert N == min(ref.added, C) and np.allclose(rb.obs[:N].numpy(), ref.obs[:N])
        assert np.allclose(rb.prio[:N].numpy(), ref.prio[:N], rtol=1e-6)        # max-priority insertion
        u = torch.rand(64, generator=g)
        idx, w = rb.sample(u, 0.4)
        ridx, rw = ref.sample(u.double().numpy(), 0.4)
        np.testing.assert_array_equal(idx.numpy(), ridx)
        assert np.allclose(w.numpy(), rw, rtol=1e-5)
        idx[5] = idx[9] = idx[0]                # duplicate indices: the later position wins
        td = torch.randn(64, generator=g) * (ep + 1)
        rb.update_priorities(idx, td, 1e-6)
        ref.update(idx.numpy(), td.double().numpy(), 1e-6)
        assert np.allclose(rb.prio[:rb.size].numpy(), ref.prio[:rb.size], rtol=1e-5)
        assert abs(float(rb.max_prio) - ref.max_p) <= 1e-6 * ref.max_p
    uni = ReplayBuffer(C, D, torch.device("cpu"), False)
    uni.store(*[torch.randn(T, B, *s) for s in ((256,),)], torch.randn(B, 256), torch.randn(T, B, D), torch.randn(T, B),
              torch.zeros(T, B, dtype=torch.uint8))
    idx, w = uni.sample(torch.tensor([0.0, 0.5, 0.999999]), 0.4)
    assert idx.tolist() == [0, 12, 23] and torch.equal(w, torch.ones(3))


@pytest.mark.parametrize("algo,cfg", [("TD3", {}), ("DDPG", {"exploration_config": OU})])
def test_learning_signal_schedule_and_checkpoint(algo, cfg):
    """On FakeContiEnv with gamma 0 (Q = the reward) and uniform actions, the critic learns the reward's slope in the
    action (positive cosine with -2 (a - target)), and an actor step against the learned critic raises Q(s, pi(s)).
    (End to end, the one SGD step per 576 stored transitions of the RLlib schedule leaves the critic far behind the actor on
    this env: the greedy reward does not improve within a CPU test's budget.)"""
    torch.manual_seed(0)
    B = 8
    cfg = dict(cfg, gamma=0.0, actor_lr=0.0, learning_starts=B * 9 * 4, buffer_size=2000, timesteps_per_iteration=B * 9 * 8,
               train_batch_size=128, exploration_config=dict(cfg.get("exploration_config", OU), random_timesteps=10 ** 6))
    env = FakeContiEnv(B, seed=3)
    tr = get_rl_model(algo, cfg, env=env, device="cpu")
    res = [tr.train() for _ in range(20)]
    assert res[0]["sgd_steps"] == 5 and all(r["sgd_steps"] == 8 for r in res[1:])     # none before learning_starts
    assert res[-1]["timesteps_total"] == 20 * 8 * B * 9 and res[-1]["replay_size"] == 2000
    assert np.isfinite(res[-1]["critic_loss"]) and res[-1]["critic_loss"] < res[0]["critic_loss"]
    pol = tr.policy
    o = env.reset()
    a = pol.actor(o).detach().requires_grad_(True)
    pol.critic(o, a, 1, pol.flat.detach()).sum().backward()
    cos = torch.nn.functional.cosine_similarity(a.grad, -2 * (a.detach() - env.target), dim=1)
    assert float(cos.min()) > 0.2, cos
    tr.config["actor_lr"] = 1e-4
    tr.opt_actor.param_groups[0]["lr"] = 1e-4
    with torch.no_grad():
        q0 = float(pol.critic(o, pol.actor(o)).mean())
    tr.twin_step(*tr.replay.gather(torch.arange(128)), None, None, True)
    with torch.no_grad():
        assert float(pol.critic(o, pol.actor(o)).mean()) > q0
    d = tempfile.mkdtemp()
    path = tr.save(d)
    tr2 = get_rl_model(algo, cfg, env=FakeContiEnv(B, seed=3), device="cpu")
    tr2.restore(path)
    tr2.opt_actor.param_groups[0]["lr"] = 1e-4
    assert torch.equal(tr2.policy.flat, tr.policy.flat) and torch.equal(tr2.policy.target, tr.policy.target)
    assert (tr2.actor_steps, tr2.critic_steps, tr2.policy_ts, tr2.iteration) == (tr.actor_steps, tr.critic_steps, tr.policy_ts, tr.iteration)
    assert torch.equal(tr2.ou_state, tr.ou_state) and tr2.replay.size == 0
    a = tr.compute_actions(o)
    assert a.shape == (B, D) and a.dtype == np.float32 and np.abs(a).max() <= 1.0
    np.testing.assert_array_equal(a, tr2.compute_actions({"obs": o.numpy()}))
    rl = tr.compute_actions({i: o[i].numpy() for i in range(3)})
    assert sorted(rl) == [0, 1, 2] and all(np.array_equal(rl[i], a[i]) for i in range(3))
    # both take one more step identically after the restore (the optimisers' state came back)
    batch = _batch(32, 4)
    for t in (tr, tr2):
        t.twin_step(*batch, None, None, True)
    assert torch.equal(tr2.policy.flat, tr.policy.flat)
    with pytest.raises(AssertionError):
        get_rl_model("TD3" if algo == "DDPG" else "DDPG", cfg, env=FakeContiEnv(B), device="cpu").restore(path)


def test_policy_delay_and_soft_update():
    tr = get_rl_model("TD3", {}, env=FakeContiEnv(8), device="cpu")
    na = tr.policy.n_actor
    batch = _batch(16, 2)
    for step in range(4):
        p0, t0 = tr.policy.flat.detach().clone(), tr.policy.target.clone()
        upd = tr.critic_steps % 2 == 0
        tr.critic_steps += 1
        tr.twin_step(*batch, None, torch.randn(16, D), upd)
        p1 = tr.policy.flat.detach()
        assert bool((p1[:na] != p0[:na]).any()) == upd and bool((p1[na:] != p0[na:]).any())
        assert torch.allclose(tr.policy.target, 0.005 * p1 + 0.995 * t0, atol=1e-7)


def _worker(rank, world, algo, init_file, out_dir):
    dist.init_process_group("gloo", init_method="file://" + init_file, rank=rank, world_size=world)
    tr = get_rl_model(algo, {"l2_reg": 1e-3}, env=FakeContiEnv(8), device="cpu")
    batch = _batch(32, 9)
    per = 32 // world
    half = [x[rank * per:(rank + 1) * per] for x in batch]
    g = torch.Generator().manual_seed(3)
    for _ in range(2):
        noise = torch.randn(32, D, generator=g)[rank * per:(rank + 1) * per]
        tr.twin_step(*half, torch.linspace(0.5, 1.5, 32)[rank * per:(rank + 1) * per], noise, True)
    torch.save({"flat": tr.policy.flat.detach(), "target": tr.policy.target}, os.path.join(out_dir, "r%d.pt" % rank))
    dist.destroy_process_group()


@pytest.mark.parametrize("algo", ["DDPG", "TD3"])
def test_world_size_2_gloo_matches_single_learner(algo):
    """Two ranks with half of a fixed batch each (and their halves of the weights and smoothing draws) end on the
    parameters of one learner given the whole batch."""
    d = tempfile.mkdtemp()
    mp.spawn(_worker, args=(2, algo, os.path.join(d, "init"), d), nprocs=2, join=True)
    r0, r1 = torch.load(os.path.join(d, "r0.pt")), torch.load(os.path.join(d, "r1.pt"))
    assert torch.equal(r0["flat"], r1["flat"]) and torch.equal(r0["target"], r1["target"])
    single = get_rl_model(algo, {"l2_reg": 1e-3}, env=FakeContiEnv(8), device="cpu")
    p0 = single.policy.flat.detach().clone()
    batch = _batch(32, 9)
    g = torch.Generator().manual_seed(3)
    for _ in range(2):
        single.twin_step(*batch, torch.linspace(0.5, 1.5, 32), torch.randn(32, D, generator=g), True)
    p = single.policy.flat.detach()
    assert (p - p0).abs().max() > 1e-4
    assert torch.allclose(r0["flat"], p, atol=2e-6) and torch.allclose(r0["target"], single.policy.target, atol=2e-6)
