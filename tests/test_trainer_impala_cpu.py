"""CPU: PG and IMPALA -- the trainer's V-trace against a float64 restatement of vtrace.from_importance_weights, RLlib 1.5's
drop-last quirk, PG's gradient against autograd of -mean(logp G), the get_rl_model routes, checkpoints, learning on a fake
env, and the world-size-2 learner over gloo against one learner on the same global batch."""
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from rl4rs_b200.trainer import (GaussIMPALATrainer, GaussPGTrainer, IMPALATrainer, PGTrainer, get_rl_model)
from test_trainer_conti_cpu import FakeContiEnv
from test_trainer_cpu import A, FakeEnv, FakeRawEnv, _fill, _prepare


def from_importance_weights(log_rhos, discounts, rewards, values, bootstrap_value, clip_rho, clip_pg_rho):
    """vtrace.from_importance_weights (RLlib 1.5), time-major [T, B], float64, written as the published scan."""
    rhos = np.exp(log_rhos)
    clipped_rhos = np.minimum(clip_rho, rhos)
    cs = np.minimum(1.0, rhos)
    values_t_plus_1 = np.concatenate([values[1:], bootstrap_value[None]], 0)
    deltas = clipped_rhos * (rewards + discounts * values_t_plus_1 - values)
    acc, out = np.zeros_like(bootstrap_value), []
    for t in reversed(range(len(deltas))):
        acc = deltas[t] + discounts[t] * cs[t] * acc
        out.append(acc)
    vs = np.stack(out[::-1]) + values
    vs_t_plus_1 = np.concatenate([vs[1:], bootstrap_value[None]], 0)
    pg_advantages = np.minimum(clip_pg_rho, rhos) * (rewards + discounts * vs_t_plus_1 - values)
    return vs, pg_advantages


def vtrace_ref(blogp, tlogp, value, reward, gamma, rho_bar, rho_pg_bar, drop_last):
    """RLlib's IMPALA batch of complete [T, B] episodes (done at T - 1): drop_last keeps steps 0..T-2 and bootstraps with
    V(s_{T-1}); otherwise every step, discount 0 at the done step (the bootstrap is then multiplied by 0).  -> (vs, pg_adv)
    over the kept steps."""
    f = lambda x: x.detach().double().numpy()
    lr, v, r = f(tlogp) - f(blogp), f(value), f(reward)
    T = r.shape[0]
    done = np.zeros_like(r)
    done[T - 1] = 1.0
    disc = gamma * (1.0 - done)
    K = T - 1 if drop_last else T
    return from_importance_weights(lr[:K], disc[:K], r[:K], v[:K], v[T - 1], rho_bar, rho_pg_bar)


def _page_rewards(T, B, g):
    """Rewards where the envs put them: the last step of Slate (T = 9), every ninth step of SeqSlate (T = 36)."""
    r = torch.zeros(T, B)
    for t in range(8, T, 9):
        r[t] = torch.rand(B, generator=g) * 10
    return r


@pytest.mark.parametrize("T", [9, 36])
@pytest.mark.parametrize("drop_last", [True, False])
@pytest.mark.parametrize("off_policy", [False, True])
def test_vtrace_matches_from_importance_weights(T, drop_last, off_policy):
    B = 24
    g = torch.Generator().manual_seed(T + 2 * drop_last + 4 * off_policy)
    tr = IMPALATrainer({"vtrace_drop_last_ts": drop_last, "gamma": 0.97, "vtrace_clip_rho_threshold": 1.2,
                        "vtrace_clip_pg_rho_threshold": 0.7}, FakeEnv(B, T), device="cpu")
    blogp = -3 * torch.rand(T, B, generator=g)
    tlogp = blogp + (torch.empty(T, B).uniform_(-1.5, 1.5, generator=g) if off_policy else 0.0)
    value, reward = torch.randn(T, B, generator=g) * 3, _page_rewards(T, B, g)
    vs, pg = tr.vtrace(blogp, tlogp, value, reward)
    K = T - 1 if drop_last else T
    rvs, rpg = vtrace_ref(blogp, tlogp, value, reward, 0.97, 1.2, 0.7, drop_last)
    scale = 1.0 + np.abs(rvs).max()
    np.testing.assert_allclose(vs[:K].double().numpy(), rvs, atol=2e-6 * scale, rtol=0)
    np.testing.assert_allclose(pg[:K].double().numpy(), rpg, atol=2e-6 * scale, rtol=0)
    if drop_last:                             # the dropped step: vs = V, no advantage
        assert torch.equal(vs[T - 1], value[T - 1]) and bool((pg[T - 1] == 0).all())
    rho = (tlogp - blogp).exp()[:K]
    if off_policy:                            # rho lies on both sides of both thresholds
        assert bool((rho > 1.2).any() & (rho < 0.7).any())
    else:                                     # on-policy: vs = the lambda = 1 return, bootstrapped at V(s_{T-1})
        r = reward.double().numpy()
        boot = value[T - 1].double().numpy() if drop_last else np.zeros(B)
        ret = np.zeros((K, B))
        acc = boot
        for t in reversed(range(K)):
            acc = r[t] + 0.97 * acc
            ret[t] = acc
        np.testing.assert_allclose(vs[:K].double().numpy(), ret, atol=2e-6 * scale, rtol=0)


def _impala_grad(tr, reward_last):
    buf = tr.buf
    buf.reward[-1] = reward_last
    tr.policy.flat.grad = None
    total, _ = tr.loss(*buf.columns()[:-3], buf.logp, buf.reward)
    total.backward()
    return tr.policy.flat.grad.detach().clone()


def test_drop_last_leaves_slate_final_reward_out_of_the_gradient():
    """Slate's only reward is at step T - 1: with RLlib 1.5's drop-last it never reaches the loss (bit-identical gradient for
    any final reward); with vtrace_drop_last_ts=False it does."""
    grads = {}
    for drop in (True, False):
        tr = IMPALATrainer({"vtrace_drop_last_ts": drop}, FakeEnv(32), device="cpu")
        _fill(tr.buf, 7, 0, 32)
        _prepare(tr)
        tr.buf.logp.add_(0.3 * torch.randn(tr.buf.logp.shape, generator=torch.Generator().manual_seed(1)))   # off-policy
        grads[drop] = (_impala_grad(tr, 1.0), _impala_grad(tr, 50.0))
    assert torch.equal(*grads[True])
    assert not torch.equal(*grads[False])


def test_pg_gradient_is_autograd_of_mean_logp_return_and_leaves_the_value_head():
    tr = PGTrainer({"gamma": 0.9}, FakeEnv(32), device="cpu")
    _fill(tr.buf, 3, 0, 32)
    buf, pol = tr.buf, tr.policy
    buf.reward.copy_(torch.rand(buf.reward.shape, generator=torch.Generator().manual_seed(2)))
    r = buf.reward.double().numpy()
    G = np.zeros_like(r)
    acc = np.zeros(r.shape[1])
    for t in reversed(range(r.shape[0])):
        acc = r[t] + 0.9 * acc
        G[t] = acc
    ret = tr.returns(buf)
    np.testing.assert_allclose(ret.double().numpy(), G, rtol=1e-6)
    # autograd of -mean(logp(a) G), written from the layers
    flat = pol.flat.detach().clone().requires_grad_(True)
    off, p = 0, {}
    for name, shape in pol._shapes:
        k = int(np.prod(shape))
        p[name] = flat[off:off + k].view(shape)
        off += k
    obs, mask, action = buf.obs.reshape(-1, 256), buf.mask.reshape(-1, A), buf.action.reshape(-1)
    h = torch.tanh(obs @ p["w1"] + p["b1"])
    logits = h @ p["w2"] + p["b2"] + torch.clamp(torch.log(mask.float()), min=torch.finfo(torch.float32).min)
    logp = torch.log_softmax(logits, -1)[torch.arange(len(action)), action]
    (-(logp * torch.as_tensor(G, dtype=torch.float32).reshape(-1)).mean()).backward()
    pol.flat.grad = None
    tr.loss(obs, mask, action, ret.reshape(-1))[0].backward()
    assert torch.allclose(pol.flat.grad, flat.grad, atol=1e-6 * float(flat.grad.abs().max()))
    head = slice(pol.n_params - 65, pol.n_params)                    # wv[64], bv[1]
    assert bool((pol.flat.grad[head] == 0).all()) and bool((pol.flat.grad[:pol.n_params - 65] != 0).any())
    before = pol.flat.detach().clone()
    tr.learn(buf)                                                      # Adam on a zero gradient leaves the head as it was
    assert torch.equal(pol.flat.detach()[head], before[head]) and not torch.equal(pol.flat.detach(), before)


def test_routes():
    plain, raw, conti = FakeEnv(8), FakeRawEnv(8), FakeContiEnv(8)
    for name, env, cls in (("PG", plain, PGTrainer), ("PG_rawstate", raw, PGTrainer), ("PG_conti", conti, GaussPGTrainer),
                           ("PG", conti, GaussPGTrainer), ("IMPALA", plain, IMPALATrainer),
                           ("IMPALA_rawstate", raw, IMPALATrainer), ("IMPALA_conti", conti, GaussIMPALATrainer),
                           ("IMPALA", conti, GaussIMPALATrainer)):
        tr = get_rl_model(name, {}, env=env, device="cpu")
        assert type(tr) is cls, name
        assert tr.rawstate == (env is raw) and tr.conti == (env is conti)
    assert get_rl_model("PG", {}, env=plain, device="cpu").config["lr"] == 4e-4
    c = get_rl_model("IMPALA", {}, env=plain, device="cpu").config
    assert (c["lr"], c["grad_clip"], c["vf_loss_coeff"], c["entropy_coeff"], c["vtrace_drop_last_ts"]) == (1e-4, 10.0, 0.5, 0.01, True)
    for name in ("PG_conti", "IMPALA_conti"):
        with pytest.raises(ValueError):                       # a *_conti name needs the continuous-action env
            get_rl_model(name, {}, env=plain, device="cpu")
        masked = FakeContiEnv(8)
        masked.config["support_rllib_mask"] = True
        with pytest.raises(ValueError):
            get_rl_model(name, {}, env=masked, device="cpu")
        rawc = FakeContiEnv(8)
        rawc.config["rawstate_as_obs"] = True
        with pytest.raises(NotImplementedError):
            get_rl_model(name, {}, env=rawc, device="cpu")
    with pytest.raises(ValueError):                           # drop-last on one-step episodes: nothing left to learn from
        get_rl_model("IMPALA", {}, env=FakeEnv(8, T=1), device="cpu")
    assert get_rl_model("IMPALA", {"vtrace_drop_last_ts": False}, env=FakeEnv(8, T=1), device="cpu").kept(1) == 1
    with pytest.raises(NotImplementedError):
        get_rl_model("IMPALA", {"opt_type": "rmsprop"}, env=plain, device="cpu")
    for name in ("DQN", "A3C", "SLATEQ", "PG_foo_conti"):
        with pytest.raises(NotImplementedError):
            get_rl_model(name, {}, env=plain, device="cpu")


@pytest.mark.parametrize("algo", ["PG", "IMPALA"])
def test_training_improves_reward_and_checkpoint_roundtrip(algo):
    torch.manual_seed(0)
    cfg = {"lr": 3e-3, "vtrace_drop_last_ts": False}       # FakeEnv pays at the last step only
    env = FakeEnv(256, seed=3)
    tr = get_rl_model(algo, cfg, env=env, device="cpu")
    first = np.mean([tr.train()["episode_reward_mean"] for _ in range(3)])
    for _ in range(25):
        res = tr.train()
    assert res["sgd_steps"] == 1 and np.isfinite(res["total_loss"])
    assert tr.evaluate(2) > first + 2.0
    path = tr.save(tempfile.mkdtemp())
    tr2 = get_rl_model(algo, cfg, env=FakeEnv(256, seed=3), device="cpu")
    tr2.restore(path)
    assert torch.equal(tr2.policy.flat, tr.policy.flat) and tr2.iteration == tr.iteration
    o = env.reset()
    np.testing.assert_array_equal(tr.compute_actions(o), tr2.compute_actions(o))
    assert torch.load(path)["algo"] == algo


@pytest.mark.parametrize("algo", ["PG_conti", "IMPALA_conti"])
def test_gauss_checkpoint_is_tagged(algo):
    tr = get_rl_model(algo, {}, env=FakeContiEnv(16), device="cpu")
    tr.train()
    path = tr.save(tempfile.mkdtemp())
    assert torch.load(path)["algo"] == algo
    tr2 = get_rl_model(algo, {}, env=FakeContiEnv(16), device="cpu")
    tr2.restore(path)
    assert torch.equal(tr2.policy.flat, tr.policy.flat)


def test_num_sgd_iter_passes_are_off_policy():
    """The second pass over the same batch sees rho != 1 (the parameters moved) and takes another step."""
    tr = IMPALATrainer({"num_sgd_iter": 2, "lr": 1e-2}, FakeEnv(32), device="cpu")
    _fill(tr.buf, 7, 0, 32)
    _prepare(tr)
    seen = []
    orig = tr.vtrace
    tr.vtrace = lambda b, t, v, r: (seen.append((t - b).abs().max().item()), orig(b, t, v, r))[1]
    assert tr.learn(tr.buf)["sgd_steps"] == 2
    assert seen[0] == 0.0 and seen[1] > 1e-4


CFG = {"PG": {"gamma": 0.9}, "IMPALA": {"vtrace_drop_last_ts": False, "gamma": 0.95, "grad_clip": 5.0}}


def _worker(rank, world, algo, init_file, out_dir):
    dist.init_process_group("gloo", init_method="file://" + init_file, rank=rank, world_size=world)
    per = 32 // world
    tr = get_rl_model(algo, CFG[algo], env=FakeEnv(per), device="cpu")
    _setup(tr, rank * per, (rank + 1) * per)
    st = tr.learn(tr.buf)
    torch.save({"flat": tr.policy.flat.detach(), "grad": tr.policy.flat.grad.detach().clone(), "stats": st},
               os.path.join(out_dir, "r%d.pt" % rank))
    dist.destroy_process_group()


def _setup(tr, lo, hi):
    _fill(tr.buf, 7, lo, hi)
    _prepare(tr)
    g = torch.Generator().manual_seed(5)
    tr.buf.logp.add_(0.5 * torch.randn(tr.T, 32, generator=g)[:, lo:hi])          # off-policy behaviour logp
    tr.buf.reward.add_(torch.rand(tr.T, 32, generator=g)[:, lo:hi])                # a reward at every step


@pytest.mark.parametrize("algo", ["PG", "IMPALA"])
def test_world_size_2_gloo_matches_single_learner(algo):
    """Two ranks with half the episodes each: PG's mean and IMPALA's sum over the global batch, one all-reduce per step, land
    on the parameters of one learner holding every episode (V-trace is per episode: no other collective)."""
    d = tempfile.mkdtemp()
    mp.spawn(_worker, args=(2, algo, os.path.join(d, "init"), d), nprocs=2, join=True)
    r0, r1 = torch.load(os.path.join(d, "r0.pt")), torch.load(os.path.join(d, "r1.pt"))
    assert torch.equal(r0["flat"], r1["flat"]) and torch.equal(r0["grad"], r1["grad"])
    single = get_rl_model(algo, CFG[algo], env=FakeEnv(32), device="cpu")
    _setup(single, 0, 32)
    p0 = single.policy.flat.detach().clone()
    st = single.learn(single.buf)
    assert (single.policy.flat.detach() - p0).abs().max() > 1e-5
    g1, g2 = r0["grad"], single.policy.flat.grad.detach()
    assert (g1 - g2).abs().max() <= 1e-5 * g2.abs().max(), ((g1 - g2).abs().max(), g2.abs().max())
    big = g2.abs() > 1e-3 * g2.abs().max()
    assert torch.allclose(r0["flat"][big], single.policy.flat.detach()[big], atol=2e-6)
    assert abs(r0["stats"]["total_loss"] - st["total_loss"]) <= 1e-4 * max(1.0, abs(st["total_loss"]))
