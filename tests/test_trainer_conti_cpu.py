"""CPU: the Gaussian policy of the continuous-action env (PPO_conti / A2C_conti) -- the torch twin of csrc/r4_gauss.cuh against
torch.distributions, clipping between policy and env, learning on a fake continuous env, checkpoints, the world-size-2
learner over gloo, one iteration through the product's host layer, and the get_rl_model dispatch."""
import math
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from rl4rs_b200.policy import GaussianPolicy
from rl4rs_b200.trainer import GaussA2CTrainer, GaussPPOTrainer, get_rl_model

D = 32


class FakeContiEnv(object):
    """Torch-format continuous-action env on CPU: every row observes one fixed random vector (plus a little noise), the
    reward per step is -||a - target||^2 for a fixed target in (-1, 1)^D, so a policy whose mean moves to the target earns
    more.  Records the actions it receives."""

    def __init__(self, B, T=9, seed=0):
        self.config = {"max_steps": T, "batch_size": B, "action_size": 284, "action_emb_size": D, "support_conti_env": True}
        self.B, self.T = B, T
        self.g = torch.Generator().manual_seed(seed)
        self.target = torch.linspace(-0.6, 0.6, D)
        self.obs0 = torch.randn(256, generator=self.g)
        self.sim = type("S", (), {"engine": type("E", (), {"device": torch.device("cpu")})()})()
        self.received = []

    def _obs(self):
        return self.obs0 + 0.1 * torch.randn(self.B, 256, generator=self.g)

    def reset(self):
        self.t = 0
        return self._obs()

    def step(self, a):
        a = torch.as_tensor(a).clone()
        self.received.append(a)
        self.t += 1
        r = -((a.to(torch.float64) - self.target.to(torch.float64)) ** 2).sum(-1)
        return self._obs(), r, torch.full((self.B,), int(self.t >= self.T)), {}


def test_gaussian_twin_matches_torch_distributions_and_normc_init():
    from rl4rs_b200 import _capi
    pol = GaussianPolicy(D, "cpu", seed=4)
    assert pol.n_params == 148032 + 131841 == 279873 == _capi.load_library().r4_gauss_num_params(D)
    p = pol.params()
    for name in ("w1", "w2", "vw1", "vw2"):                  # normc_initializer(1.0): every column has unit norm
        assert torch.allclose(p[name].norm(dim=0), torch.ones(p[name].shape[1]), atol=1e-5), name
    for name in ("wo", "vwo"):
        assert torch.allclose(p[name].norm(dim=0), torch.full((p[name].shape[1],), 0.01), atol=1e-7), name
    for name in ("b1", "b2", "bo", "vb1", "vb2", "vbo"):
        assert bool((p[name] == 0).all()), name
    g = torch.Generator().manual_seed(0)
    new, old = torch.randn(50, 2 * D, generator=g) * 0.5, torch.randn(50, 2 * D, generator=g) * 0.5
    a = torch.randn(50, D, generator=g)
    nn = torch.distributions.Normal(new[:, :D], new[:, D:].exp())
    no = torch.distributions.Normal(old[:, :D], old[:, D:].exp())
    assert torch.allclose(GaussianPolicy.logp(new, a), nn.log_prob(a).sum(-1), atol=1e-4)
    assert torch.allclose(GaussianPolicy.entropy(new), nn.entropy().sum(-1), atol=1e-4)
    assert torch.allclose(GaussianPolicy.kl(old, new), torch.distributions.kl_divergence(no, nn).sum(-1), atol=1e-4)
    # the forward is the layer list of the default FullyConnectedNetwork
    obs = torch.randn(7, 256, generator=g)
    d, v = pol.forward(obs)
    h = torch.tanh(torch.tanh(obs @ p["w1"] + p["b1"]) @ p["w2"] + p["b2"])
    assert d.shape == (7, 2 * D) and torch.allclose(d, h @ p["wo"] + p["bo"], atol=1e-6) and v.shape == (7,)
    # greedy action = the mean, logp of the mean = -sum(log_std) - D/2 log(2 pi)
    act, env_act, logp, value, dist_in = pol.act(obs, explore=False)
    assert torch.equal(act, d[:, :D]) and torch.equal(env_act, d[:, :D].clamp(-1, 1))
    assert torch.allclose(logp, -d[:, D:].sum(-1) - 0.5 * D * math.log(2 * math.pi), atol=1e-4)


def test_env_gets_clipped_actions_and_buffer_keeps_the_sample():
    torch.manual_seed(0)
    env = FakeContiEnv(64)
    tr = get_rl_model("PPO_conti", {}, env=env, device="cpu")
    with torch.no_grad():                                    # wide log_std: most samples leave [-1, 1]
        tr.policy.params()["bo"][D:].fill_(1.0)
    buf = tr.rollout(explore=True)
    assert len(env.received) == 9
    got = torch.stack(env.received)
    assert float(got.abs().max()) <= 1.0 and float(buf.action.abs().max()) > 1.5
    assert torch.equal(got, buf.action.clamp(-1.0, 1.0))
    assert torch.allclose(buf.logp, GaussianPolicy.logp(buf.dist, buf.action), atol=1e-4)


@pytest.mark.parametrize("algo", ["PPO_conti", "A2C_conti"])
def test_training_improves_reward_checkpoint_and_compute_actions(algo):
    torch.manual_seed(0)
    env = FakeContiEnv(128, seed=3)
    cfg = {"lr": 1e-3 if algo.startswith("PPO") else 3e-4}
    tr = get_rl_model(algo, cfg, env=env, device="cpu")
    assert isinstance(tr, GaussPPOTrainer if algo.startswith("PPO") else GaussA2CTrainer) and tr.algo == algo
    before = tr.evaluate(1)
    for _ in range(12):
        res = tr.train()
    assert res["timesteps_total"] == 12 * 9 * 128 and np.isfinite(res["total_loss"])
    after = tr.evaluate(1)
    assert after > before + 0.2 * abs(before), (before, after)      # the mean walks towards the target (about +30 %)
    d = tempfile.mkdtemp()
    path = tr.save(d)
    tr2 = get_rl_model(algo, cfg, env=FakeContiEnv(128, seed=3), device="cpu")
    tr2.restore(path)
    assert torch.equal(tr2.policy.flat, tr.policy.flat) and tr2.iteration == tr.iteration
    o = env.reset()
    a = tr.compute_actions(o)
    assert a.shape == (128, D) and a.dtype == np.float32 and np.abs(a).max() <= 1.0
    np.testing.assert_array_equal(a, tr2.compute_actions({"obs": o.numpy()}))
    rl = tr.compute_actions({i: o[i].numpy() for i in range(4)})
    assert sorted(rl) == [0, 1, 2, 3] and all(np.array_equal(rl[i], a[i]) for i in range(4))
    # a conti checkpoint does not restore into the discrete trainer
    from test_trainer_cpu import FakeEnv
    with pytest.raises(AssertionError):
        get_rl_model(algo.split("_")[0], cfg, env=FakeEnv(128), device="cpu").restore(path)


def _fill(tr, seed, lo, hi):
    g = torch.Generator().manual_seed(seed)
    T, Bfull = tr.T, 32
    obs = torch.randn(T, Bfull, 256, generator=g)
    act = torch.randn(T, Bfull, D, generator=g)
    rew = torch.randn(T, Bfull, generator=g)
    buf = tr.buf
    buf.obs.copy_(obs[:, lo:hi]); buf.action.copy_(act[:, lo:hi]); buf.reward.copy_(rew[:, lo:hi])
    with torch.no_grad():
        for t in range(tr.T):
            d, v = tr.policy.forward(buf.obs[t])
            buf.dist[t].copy_(d + 0.1); buf.value[t].copy_(v)
            buf.logp[t].copy_(GaussianPolicy.logp(d + 0.1, buf.action[t]))


def _worker(rank, world, algo, init_file, out_dir):
    dist.init_process_group("gloo", init_method="file://" + init_file, rank=rank, world_size=world)
    per = 32 // world
    tr = get_rl_model(algo, {"sgd_minibatch_size": 288, "shuffle_sequences": False}, env=FakeContiEnv(per), device="cpu")
    _fill(tr, 7, rank * per, (rank + 1) * per)
    st = tr.learn(tr.buf)
    torch.save({"flat": tr.policy.flat.detach(), "grad": tr.policy.flat.grad.detach().clone(), "stats": st},
               os.path.join(out_dir, "r%d.pt" % rank))
    dist.destroy_process_group()


@pytest.mark.parametrize("algo", ["A2C_conti", "PPO_conti"])
def test_world_size_2_gloo_matches_single_learner(algo):
    """Two ranks with half the rows each + one gradient all-reduce per step == one learner on all rows (PPO: one
    minibatch = the whole batch, unshuffled)."""
    d = tempfile.mkdtemp()
    mp.spawn(_worker, args=(2, algo, os.path.join(d, "init"), d), nprocs=2, join=True)
    r0, r1 = torch.load(os.path.join(d, "r0.pt")), torch.load(os.path.join(d, "r1.pt"))
    assert torch.equal(r0["flat"], r1["flat"]) and torch.equal(r0["grad"], r1["grad"])
    single = get_rl_model(algo, {"sgd_minibatch_size": 288, "shuffle_sequences": False}, env=FakeContiEnv(32), device="cpu")
    _fill(single, 7, 0, 32)
    p0 = single.policy.flat.detach().clone()
    st = single.learn(single.buf)
    assert (single.policy.flat.detach() - p0).abs().max() > 1e-5
    g1, g2 = r0["grad"], single.policy.flat.grad.detach()
    assert (g1 - g2).abs().max() <= 1e-5 * g2.abs().max(), ((g1 - g2).abs().max(), g2.abs().max())
    big = g2.abs() > 1e-3 * g2.abs().max()
    assert torch.allclose(r0["flat"][big], single.policy.flat.detach()[big], atol=2e-6)
    assert abs(r0["stats"]["total_loss"] - st["total_loss"]) <= 1e-4 * max(1.0, abs(st["total_loss"]))


@pytest.fixture()
def oracle_engine(monkeypatch):
    from oracle_engine import OracleEngine
    import rl4rs_b200.engine as engine_mod
    monkeypatch.setattr(engine_mod, "Engine", OracleEngine)


def test_ppo_conti_iteration_through_the_host_layer(oracle_engine):
    """One PPO_conti iteration driving SlateRecEnv-v0 (torch format, support_conti_env, no rllib mask) through the product's
    env classes over the oracle-backed engine: the env receives the clipped actions, and the items it places are the
    masked kNN (slate.py:186-191) of those actions replayed on the oracle's state."""
    from oracle.env_np import OracleState
    from test_gpu_parity import _synthetic
    from test_host_layer_cpu import make_env
    torch.manual_seed(0)
    np.random.seed(0)
    cfg, cat, log, w = _synthetic(8, False, support_conti_env=True)
    env = make_env(cfg, False, cat, log, w, output_format="torch")
    sent = []
    step = env.step
    env.step = lambda a: (sent.append(a.clone()), step(a))[1]
    tr = get_rl_model("PPO_conti", {"sgd_minibatch_size": 24}, env=env, device="cpu", seed=0)
    st = tr.train()
    assert np.isfinite(st["total_loss"]) and st["sgd_steps"] == 3 and tr.buf.obs.shape == (9, 8, 256)
    assert torch.equal(torch.stack(sent), tr.buf.action.clamp(-1.0, 1.0))
    ref = OracleState(dict(cfg, support_conti_env=True), log, cat, env.samples.rows, False)
    for a in sent:
        ref.act(a.numpy())
    np.testing.assert_array_equal(np.asarray(env.samples.prev_actions), ref.prev_actions)


def test_dispatch_and_errors():
    from test_trainer_cpu import FakeEnv
    from rl4rs_b200.trainer import A2CTrainer, PPOTrainer
    conti, discrete = FakeContiEnv(8), FakeEnv(8)
    assert type(get_rl_model("PPO", {}, env=conti, device="cpu")) is GaussPPOTrainer
    assert type(get_rl_model("A2C", {}, env=conti, device="cpu")) is GaussA2CTrainer
    assert type(get_rl_model("A2C_conti", {}, env=conti, device="cpu")) is GaussA2CTrainer
    assert type(get_rl_model("PPO", {}, env=discrete, device="cpu")) is PPOTrainer
    assert type(get_rl_model("A2C", {}, env=discrete, device="cpu")) is A2CTrainer
    with pytest.raises(ValueError, match="support_conti_env"):
        get_rl_model("PPO_conti", {}, env=discrete, device="cpu")
    masked = FakeContiEnv(8); masked.config["support_rllib_mask"] = True
    with pytest.raises(ValueError, match="support_rllib_mask"):
        get_rl_model("PPO_conti", {}, env=masked, device="cpu")
    raw = FakeContiEnv(8); raw.config["rawstate_as_obs"] = True
    with pytest.raises(NotImplementedError):
        get_rl_model("A2C_conti", {}, env=raw, device="cpu")
    with pytest.raises(NotImplementedError):
        get_rl_model("DDPG_conti", {}, env=conti, device="cpu")
    with pytest.raises(NotImplementedError):
        get_rl_model("DQN", {}, env=discrete)
