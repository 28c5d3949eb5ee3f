"""GPU: the Gaussian-policy kernels of the continuous-action env (csrc/r4_gauss.cuh) against the torch twin and autograd, the
epoch driver against the per-step loop, and PPO_conti / A2C_conti end to end on the CUDA env."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

D = 32


def _policy(dev, seed=3):
    import torch
    from rl4rs_b200.policy import GaussianPolicy
    pol = GaussianPolicy(D, dev, seed=seed)
    with torch.no_grad():                      # move off the init: non-trivial output layers and log_std
        g = torch.Generator().manual_seed(seed)
        pol.flat.add_(0.02 * torch.randn(pol.n_params, generator=g).to(dev))
    return pol


def test_act_kernel_matches_the_twin_and_samples_the_gaussian():
    import torch
    from rl4rs_b200.trainer import GaussKernelOps
    dev = torch.device("cuda")
    pol = _policy(dev)
    ops = GaussKernelOps(D, dev, pol.n_params)
    n = 300
    obs = torch.randn(n, 256, generator=torch.Generator().manual_seed(0)).to(dev)
    e = lambda *s: torch.empty(*s, device=dev)
    a, ea, lp, v, d = e(n, D), e(n, D), e(n), e(n), e(n, 2 * D)
    ops.act(pol.flat, obs, False, 1, a, ea, lp, v, d)
    td, tv = pol.forward(obs)
    assert float((d - td).abs().max()) < 1e-4 and float((v - tv).abs().max()) < 1e-4
    assert torch.equal(a, d[:, :D]) and torch.equal(ea, a.clamp(-1.0, 1.0))             # greedy action = clip(mean)
    assert torch.allclose(lp, pol.logp(d, a), atol=1e-4)
    # 4000 samples of one row: z = (a - mean) / std is N(0, 1) per dimension.  The mean of 4000 draws has std 1/63 and the
    # sample std has std ~ 1/89; 5 sigma bounds on both (32 dimensions: a false alarm is < 1e-5)
    reps = 4000
    o1 = obs[:1].repeat(reps, 1).contiguous()
    a1, ea1, lp1, v1 = e(reps, D), e(reps, D), e(reps), e(reps)
    c0 = ops.counter
    ops.act(pol.flat, o1, True, 7, a1, ea1, lp1, v1, None)
    z = (a1 - d[:1, :D]) / d[:1, D:].exp()
    assert float(z.mean(0).abs().max()) < 5 / reps ** 0.5, float(z.mean(0).abs().max())
    assert float((z.std(0) - 1).abs().max()) < 5 / (2 * reps) ** 0.5, float((z.std(0) - 1).abs().max())
    assert float(ea1.abs().max()) <= 1.0 and torch.allclose(lp1, pol.logp(d[:1].expand(reps, -1), a1), atol=1e-3)
    # the same seed and counter give the same actions; another counter gives others
    a2 = e(reps, D)
    ops.counter = c0
    ops.act(pol.flat, o1, True, 7, a2, e(reps, D), e(reps), e(reps), None)
    assert torch.equal(a1, a2)
    ops.act(pol.flat, o1, True, 7, a2, e(reps, D), e(reps), e(reps), None)
    assert not torch.equal(a1, a2)


def _batch(pol, n, dev, seed=5):
    import torch
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(n, 256, generator=g).to(dev)
    with torch.no_grad():
        d, v = pol.forward(obs)
    old_d = (d + 0.2 * torch.randn(n, 2 * D, generator=g).to(dev)).contiguous()
    act = (old_d[:, :D] + old_d[:, D:].exp() * torch.randn(n, D, generator=g).to(dev)).contiguous()
    old_lp = pol.logp(old_d, act).contiguous()
    old_v = (v + torch.randn(n, generator=g).to(dev)).contiguous()
    adv = torch.randn(n, generator=g).to(dev)
    tgt = (old_v + 600 * torch.randn(n, generator=g).to(dev)).contiguous()     # exercises the vf clip (500)
    return obs, act, old_lp, old_d, old_v, adv, tgt


class _E(object):
    config = {"max_steps": 3, "batch_size": 100, "action_size": 284, "action_emb_size": D, "support_conti_env": True}


@pytest.mark.parametrize("mode,n", [(0, 300), (1, 300), (1, 2500)])
def test_gradient_kernel_matches_autograd(mode, n):
    """PPO (mode 0, mean) and A2C (mode 1, sums; n = 2500 spans two 2048-sample chunks) against autograd.  Bound: 2e-5 of
    the largest gradient element, as for the mask policy."""
    import torch
    from rl4rs_b200.trainer import GaussA2CTrainer, GaussKernelOps, GaussPPOTrainer
    dev = torch.device("cuda")
    pol = _policy(dev)
    ops = GaussKernelOps(D, dev, pol.n_params)
    obs, act, old_lp, old_d, old_v, adv, tgt = _batch(pol, n, dev)
    env = _E()
    env.sim = type("S", (), {"engine": type("X", (), {"device": dev})()})()
    tr = (GaussPPOTrainer if mode == 0 else GaussA2CTrainer)({"entropy_coeff": 0.01, "use_kernels": False}, env, device=dev)
    tr.policy = pol
    if mode == 0:
        tr.kl_coeff = 0.2
        total, st = tr.loss(obs, act, old_lp, old_d, old_v, adv, tgt)
        hp = {"clip": 0.3, "vf_clip": 500.0, "vf_coeff": 0.5, "kl_coeff": 0.2, "ent_coeff": 0.01}
        inv_n = 1.0 / n
        data = (obs, act, old_lp, old_d, old_v, adv, tgt)
    else:
        total, st = tr.loss(obs, act, adv, tgt)
        hp = {"clip": 0.0, "vf_clip": 0.0, "vf_coeff": 0.5, "kl_coeff": 0.0, "ent_coeff": 0.01}
        inv_n = 1.0
        data = (obs, act, None, None, None, adv, tgt)
    total.backward()
    ref = pol.flat.grad.detach().clone()
    ops.stats.zero_()
    ops.policy_grad(mode, pol.flat, data, None, 0, n, hp, inv_n, inv_n)
    err = float((ops.grad - ref).abs().max() / ref.abs().max())
    assert err < 2e-5, err
    assert abs(float(ops.stats[4]) - float(total)) <= 1e-4 * abs(float(total)), (float(ops.stats[4]), float(total))
    # an index list gives the gradient of the gathered rows, bit for bit
    m = 128
    idx = torch.randperm(n, generator=torch.Generator().manual_seed(9))[:m].to(dev)
    ops.policy_grad(mode, pol.flat, data, idx, 0, m, hp, 1.0 / m, 1.0)
    g_idx = ops.grad.clone()
    sel = tuple(x[idx].contiguous() if x is not None else None for x in data)
    ops.policy_grad(mode, pol.flat, sel, None, 0, m, hp, 1.0 / m, 1.0)
    assert torch.equal(g_idx, ops.grad)


def test_epoch_driver_matches_the_per_step_loop_bitwise():
    import torch
    from rl4rs_b200.trainer import GaussKernelOps
    dev = torch.device("cuda")
    pol = _policy(dev)
    n = 300
    data = _batch(pol, n, dev)
    hp = {"clip": 0.3, "vf_clip": 500.0, "vf_coeff": 0.5, "kl_coeff": 0.2, "ent_coeff": 0.0}
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(2)).to(dev)
    for clip in (None, 0.5):
        pa, pb = pol.flat.detach().clone(), pol.flat.detach().clone()
        oa, ob = GaussKernelOps(D, dev, pol.n_params), GaussKernelOps(D, dev, pol.n_params)
        assert oa.ppo_epoch(pa, data, perm, n, 64, hp, 1e-3, clip) == n // 64 and oa.step == n // 64
        for s in range(0, n - 64 + 1, 64):
            ob.policy_grad(0, pb, data, perm, s, 64, hp, 1.0 / 64, 1.0 / 64)
            ob.adam(pb, 1e-3, 1.0, clip)
        assert float((pa - pol.flat).abs().max()) > 1e-4
        # the gradient, the clip's global norm (one CTA, fixed order) and Adam are deterministic, clipped or not
        assert torch.equal(pa, pb) and torch.equal(oa.stats, ob.stats)
        assert torch.equal(oa.m, ob.m) and torch.equal(oa.v, ob.v)


@pytest.mark.parametrize("algo", ["PPO_conti", "A2C_conti"])
@pytest.mark.parametrize("seq", [False, True])
def test_conti_trainer_end_to_end_on_cuda_env(algo, seq):
    """Two iterations on the CUDA env (Slate, SeqSlate-27) at B = 64: finite losses, and the items the env placed are the
    oracle's masked kNN of the clipped actions the policy sent."""
    import torch
    from oracle.env_np import OracleState
    from test_gpu_parity import _synthetic, make_env
    from rl4rs_b200.trainer import get_rl_model
    B = 64
    cfg, cat, log, w = _synthetic(B, seq, support_conti_env=True, is_eval=False, cache_size=4 * B)
    env = make_env(cfg, seq, cat, log, w, output_format="torch")
    sent = []
    step = env.step
    env.step = lambda a: (sent.append(a.detach().cpu().clone()), step(a))[1]
    tr = get_rl_model(algo, {}, env=env)
    assert tr.use_kernels and tr.algo == algo
    r = [tr.train() for _ in range(2)]
    assert all(np.isfinite(x["total_loss"]) and np.isfinite(x["episode_reward_mean"]) for x in r)
    assert r[-1]["timesteps_total"] == 2 * B * cfg["max_steps"]
    assert torch.isfinite(tr.policy.flat).all()
    T = cfg["max_steps"]
    last = sent[-T:]
    assert torch.equal(torch.stack(last), tr.buf.action.cpu().clamp(-1.0, 1.0))
    ref = OracleState(dict(cfg), log, cat, env.samples.rows, seq)
    for a in last:
        ref.act(a.numpy())
    np.testing.assert_array_equal(np.asarray(env.samples.prev_actions), ref.prev_actions)
    assert np.isfinite(tr.evaluate(1))
