"""GPU: the DDPG / TD3 kernels (csrc/r4_ddpg.cuh) against the torch twin and autograd -- act in its three modes, the replay
kernels against the torch replay, the gradients, the whole SGD step -- and both trainers end to end on the CUDA env."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

D = 32


def _pair(algo, B=8, **cfg):
    """A kernel trainer and a torch-twin trainer on the same device with the same init."""
    import torch
    from test_trainer_conti_cpu import FakeContiEnv
    from rl4rs_b200.trainer import get_rl_model
    class HostEnv(FakeContiEnv):             # the fake env computes on the host
        def step(self, a):
            return super().step(a.cpu())
    cfg = dict({"buffer_size": 500}, **cfg)
    tk = get_rl_model(algo, cfg, env=HostEnv(B), device="cuda")
    tt = get_rl_model(algo, dict(cfg, use_kernels=False), env=HostEnv(B), device="cuda")
    assert tk.use_kernels and not tt.use_kernels
    with torch.no_grad():                      # move the targets off the online weights
        g = torch.Generator().manual_seed(1)
        tk.policy.target.add_(0.01 * torch.randn(tk.policy.n_params, generator=g).cuda())
        tt.policy.target.copy_(tk.policy.target)
    return tk, tt


def _fill(trs, T=9, B=40, seed=0):
    import torch
    g = torch.Generator().manual_seed(seed)
    obs, fin = torch.randn(T, B, 256, generator=g).cuda(), torch.randn(B, 256, generator=g).cuda()
    act = (torch.rand(T, B, D, generator=g) * 2 - 1).cuda()
    rew = torch.randn(T, B, generator=g).cuda()
    done = torch.zeros(T, B, dtype=torch.uint8).cuda()
    done[-1] = 1
    for tr in trs:
        tr.replay.store(obs, fin, act, rew, done)


def test_act_kernel_matches_the_twin():
    import torch
    from rl4rs_b200.policy import counter_draws
    tk, tt = _pair("DDPG", exploration_config={"type": "OrnsteinUhlenbeckNoise", "random_timesteps": 100})
    obs = torch.randn(300, 256, generator=torch.Generator().manual_seed(0)).cuda()
    a = torch.empty(300, D, device="cuda")
    tk._act(obs, False, a)
    assert float((a - tt.policy.actor(obs).detach()).abs().max()) < 1e-4
    # random phase: U(-1, 1), reproducible from (seed, counter), equal to the counter-based draws
    big = torch.randn(4000, 256).cuda()
    r = torch.empty(4000, D, device="cuda")
    c0 = tk.counter
    tk._act(big, True, r)
    n = r.numel()
    assert abs(float(r.mean())) < 5 * (1 / 3 / n) ** 0.5 and abs(float(r.var()) - 1 / 3) < 5 * (4 / 45 / n) ** 0.5
    assert np.allclose(r.cpu().numpy(), counter_draws(tk._seed, c0, 4000, D)[0], atol=1e-6)
    tk.counter, tk.policy_ts = c0, 0
    r2 = torch.empty_like(r)
    tk._act(big, True, r2)
    assert torch.equal(r, r2)
    # OU: the state recurrence over several calls equals the twin's; one noise vector for every row
    tk.policy_ts = tt.policy_ts = 101
    tt.counter, tt._seed = tk.counter, tk._seed
    for _ in range(4):
        ak, at = torch.empty(300, D, device="cuda"), torch.empty(300, D, device="cuda")
        tk._act(obs, True, ak)
        tt._act(obs, True, at)
        assert float((tk.ou_state[tk._ou_slot] - tt.ou_state[tt._ou_slot]).abs().max()) < 1e-5
        assert float((ak - at).abs().max()) < 1e-4
    det = tt.policy.actor(obs).detach()
    d = ak - det
    inside = (ak.abs() < 0.999).all(1)
    assert float((d[inside] - d[inside][:1]).abs().max()) < 1e-4 and float(d.abs().max()) > 1e-3


def test_replay_kernels_match_the_torch_replay():
    import torch
    tk, tt = _pair("DDPG")
    for ep in range(2):                       # 720 rows into 500 slots: wraps around
        _fill((tk, tt), seed=ep)
        N = tk.replay.size
        for name in ("obs", "action", "reward", "new_obs", "done"):
            assert torch.equal(getattr(tk.replay, name)[:N], getattr(tt.replay, name)[:N]), name
        assert torch.allclose(tk.replay.prio[:N], tt.replay.prio[:N], rtol=1e-6)
        u = torch.rand(256, generator=torch.Generator(device="cuda").manual_seed(ep), device="cuda")
        (ik, wk), (it, wt) = tk.replay.sample(u, 0.4), tt.replay.sample(u, 0.4)
        assert torch.equal(ik, it) and torch.allclose(wk, wt, rtol=1e-5)
        ik[7] = ik[3] = ik[0]
        td = torch.randn(256, device="cuda") * 3
        tk.replay.update_priorities(ik, td, 1e-6)
        tt.replay.update_priorities(ik, td, 1e-6)
        assert torch.allclose(tk.replay.prio[:N], tt.replay.prio[:N], rtol=1e-6)
        assert torch.allclose(tk.replay.max_prio, tt.replay.max_prio)
    u = torch.tensor([0.0, 0.5, 0.999999], device="cuda")
    un = _pair("TD3")[0]
    _fill((un,))
    assert un.replay.sample(u, 0.4)[0].tolist() == [0, 180, 359]


@pytest.mark.parametrize("algo", ["DDPG", "TD3"])
def test_gradient_matches_autograd(algo):
    import torch
    tk, tt = _pair(algo, l2_reg=1e-6)
    _fill((tk,))
    n = 200
    g = torch.Generator(device="cuda").manual_seed(2)
    idx = torch.randint(0, tk.replay.size, (n,), generator=g, device="cuda")
    w = torch.rand(n, generator=g, device="cuda") + 0.5 if algo == "DDPG" else None
    noise = torch.randn(n, D, generator=g, device="cuda") if algo == "TD3" else None
    ops = tk.ops
    ops.td = torch.zeros(n, device="cuda")
    ops.scratch = torch.zeros(ops.lib.r4_ddpg_scratch_size(D, ops.twin, n), device="cuda")
    ops.grad_(tk.policy, tk.replay, idx, w, noise, tk._hp(), 1.0 / n)
    pol = tk.policy
    cl, al, td = pol.losses(*tk.replay.gather(idx), w, noise, 1.0, 0.2, 0.5, 1.0 / n)
    pol.flat.grad = None
    (cl + al).backward()
    ref = pol.flat.grad
    err = (ops.grad - ref).abs().max()
    assert float(err) <= 2e-5 * float(ref.abs().max()), (float(err), float(ref.abs().max()))
    na = pol.n_actor
    for part in (ref[:na], ref[na:]):
        assert float(part.abs().max()) > 0
    assert float((ops.td - td).abs().max()) < 1e-4
    assert abs(float(ops.stats[0]) - float(cl)) <= 1e-4 * max(1.0, abs(float(cl)))
    assert abs(float(ops.stats[1]) - float(al)) <= 1e-4 * max(1.0, abs(float(al)))


@pytest.mark.parametrize("algo", ["DDPG", "TD3"])
def test_whole_sgd_step_matches_the_twin(algo):
    import torch
    tk, tt = _pair(algo, l2_reg=1e-6, train_batch_size=128)
    _fill((tk, tt))
    na = tk.policy.n_actor
    for step in range(3):
        u, noise = tk.draws()
        a0, t0 = tk.policy.flat.detach().clone(), tk.policy.target.clone()
        tk.sgd_step(u, noise)
        tt.sgd_step(u, noise)
        if step == 0:        # one step from the same state; later states differ by Adam's amplification of fp32 noise
            g = tt.policy.flat.grad      # Adam moves a parameter by about lr * sign(g): compare where g is clearly non-zero
            big = g.abs() > 1e-3 * g.abs().max()
            for x, y in ((tk.policy.flat.detach(), tt.policy.flat.detach()), (tk.policy.target, tt.policy.target)):
                err = float((x - y)[big].abs().max())
                assert err <= 1e-5 * float(y.abs().max()), err
        moved = bool((tk.policy.flat.detach()[:na] != a0[:na]).any())
        assert moved == (algo == "DDPG" or step % 2 == 0)               # policy_delay 2: the actor waits on odd steps
        assert bool((tk.policy.target[:na] != t0[:na]).any())           # the targets move every step
        if tk.replay.prio is not None and step == 0:
            assert torch.allclose(tk.replay.prio[:tk.replay.size], tt.replay.prio[:tt.replay.size], rtol=1e-4)


def test_seeded_runs_are_bit_identical():
    import torch
    out = []
    for _ in range(2):
        tk, _ = _pair("TD3", learning_starts=72, timesteps_per_iteration=150, train_batch_size=64,
                      exploration_config={"type": "OrnsteinUhlenbeckNoise", "random_timesteps": 100})
        for _ in range(3):
            tk.train()
        torch.cuda.synchronize()
        out.append(tk.policy.flat.detach().clone())
    assert torch.equal(out[0], out[1])


@pytest.mark.parametrize("algo", ["DDPG", "TD3"])
@pytest.mark.parametrize("seq", [False, True])
def test_ddpg_trainers_end_to_end_on_cuda_env(algo, seq, tmp_path):
    import torch
    from test_gpu_parity import _synthetic, make_env
    from rl4rs_b200.trainer import get_rl_model
    B = 64
    cfg, cat, log, w = _synthetic(B, seq, support_conti_env=True, is_eval=False, cache_size=4 * B)
    env = make_env(cfg, seq, cat, log, w, output_format="torch")
    T = cfg["max_steps"]
    ls = 3 * B * T
    tr = get_rl_model(algo, {"learning_starts": ls, "buffer_size": 4 * B * T,
                             "exploration_config": {"type": "OrnsteinUhlenbeckNoise", "random_timesteps": B * T}}, env=env)
    assert tr.use_kernels and tr.algo == algo
    per_it = -(-1000 // (B * T))
    res = [tr.train() for _ in range(3)]
    added = 3 * per_it * B * T
    assert res[-1]["timesteps_total"] == added and tr.replay.size == min(added, 4 * B * T)
    episodes = 3 * per_it
    assert sum(r["sgd_steps"] for r in res) == episodes - 2          # no step before learning_starts
    assert np.isfinite(res[-1]["critic_loss"]) and np.isfinite(res[-1]["actor_loss"])
    assert torch.isfinite(tr.policy.flat).all() and tr.evaluate(1) >= 0
    a = tr.compute_actions(env.reset())
    assert a.shape == (B, D) and a.dtype == np.float32 and np.abs(a).max() <= 1.0
    path = tr.save(str(tmp_path))
    tr2 = get_rl_model(algo, {}, env=env)
    tr2.restore(path)
    assert torch.equal(tr2.policy.flat, tr.policy.flat) and torch.equal(tr2.ops.m, tr.ops.m)
