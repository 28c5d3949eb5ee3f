"""GPU: the RAINBOW kernels (csrc/r4_rainbow.cuh) against the torch twin and autograd -- act (argmax and SoftQ), the n-step
store against the torch store, the gradient, the whole SGD step -- and the trainer end to end on the CUDA env."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

A, Z = 284, 8


def _pair(B=8, **cfg):
    """A kernel trainer and a torch-twin trainer on the same device with the same init, the targets moved off the online
    weights."""
    import torch
    from test_trainer_rainbow_cpu import FakeEnv
    from rl4rs_b200.trainer import get_rl_model

    class HostEnv(FakeEnv):                  # the fake env computes on the host
        def step(self, a):
            return super().step(a.cpu())
    cfg = dict({"buffer_size": 500}, **cfg)
    tk = get_rl_model("RAINBOW", cfg, env=HostEnv(B), device="cuda")
    tt = get_rl_model("RAINBOW", dict(cfg, use_kernels=False), env=HostEnv(B), device="cuda")
    assert tk.use_kernels and not tt.use_kernels
    with torch.no_grad():
        g = torch.Generator().manual_seed(1)
        tk.policy.target.add_(0.3 * torch.randn(tk.policy.n_params, generator=g).cuda())
        tt.policy.target.copy_(tk.policy.target)
    return tk, tt


def _fill(trs, T=9, B=40, seed=0):
    import torch
    g = torch.Generator().manual_seed(seed)
    obs, fin = torch.randn(T, B, 256, generator=g).cuda(), torch.randn(B, 256, generator=g).cuda()
    act = torch.randint(0, A, (T, B), generator=g, dtype=torch.int32).cuda()
    rew = (torch.rand(T, B, generator=g) * 3).cuda()
    done = torch.zeros(T, B, dtype=torch.uint8).cuda()
    done[-1] = 1
    for tr in trs:
        tr.replay.store(obs, fin, act, rew, done)


def test_act_kernel_matches_the_twin():
    import torch
    from rl4rs_b200.policy import DistributionalQNetwork
    tk, tt = _pair()
    obs = torch.randn(300, 256, generator=torch.Generator().manual_seed(0)).cuda()
    a = torch.empty(300, dtype=torch.int32, device="cuda")
    q = torch.empty(300, A, device="cuda")
    tk.ops.act(tk.policy, obs, False, 5, 0, a, q)
    qt = tt.policy.forward(obs)[1].detach()
    assert float((q - qt).abs().max()) <= 1e-4 * float(qt.abs().max())
    top2 = qt.topk(2, 1).values
    clear = (top2[:, 0] - top2[:, 1]) > 1e-4 * float(qt.abs().max())
    assert int(clear.sum()) > 150 and torch.equal(a.long()[clear], qt.argmax(1)[clear])
    # SoftQ: reproducible from (seed, counter); the twin's sampler with the same draws agrees
    s1, s2, s3 = (torch.empty(300, dtype=torch.int32, device="cuda") for _ in range(3))
    tk.ops.act(tk.policy, obs, True, 5, 100, s1)
    tk.ops.act(tk.policy, obs, True, 5, 100, s2)
    tk.ops.act(tk.policy, obs, True, 5, 400, s3)
    assert torch.equal(s1, s2) and not torch.equal(s1, s3)
    st = tt.policy.act(obs, True, 5, 100)[0]
    assert float((st == s1).float().mean()) > 0.95
    # with small Q (v_max = 3) the draws follow softmax(Q)
    pol = DistributionalQNetwork(A, "cuda", seed=1, v_max=3.0)
    one = torch.randn(1, 256, generator=torch.Generator().manual_seed(2)).cuda().repeat(40000, 1)
    s = torch.empty(40000, dtype=torch.int32, device="cuda")
    qs = torch.empty(40000, A, device="cuda")
    tk.ops.act(pol, one, True, 9, 0, s, qs)
    p = torch.softmax(qs[0].double(), 0).cpu().numpy()
    freq = np.bincount(s.cpu().numpy(), minlength=A) / 40000
    assert p.max() < 0.05 and np.abs(freq - p).max() < 5 * np.sqrt(p.max() / 40000)


@pytest.mark.parametrize("T,B", [(9, 40), (36, 10)])
def test_nstep_store_kernel_is_bit_exact(T, B):
    import torch
    tk, tt = _pair(gamma=0.9)
    for ep in range(2):                       # 720 rows into 500 slots: wraps around
        _fill((tk, tt), T=T, B=B, seed=ep)
        N = tk.replay.size
        for name in ("obs", "action", "reward", "new_obs", "done"):
            assert torch.equal(getattr(tk.replay, name)[:N], getattr(tt.replay, name)[:N]), name
        assert torch.equal(tk.replay.prio[:N], tt.replay.prio[:N])


def test_gradient_matches_autograd():
    import torch
    tk, _ = _pair(v_max=10.0, grad_clip=None)
    _fill((tk,))
    n = 200
    g = torch.Generator(device="cuda").manual_seed(2)
    idx = torch.randint(0, tk.replay.size, (n,), generator=g, device="cuda")
    w = torch.rand(n, generator=g, device="cuda") + 0.5
    ops, pol = tk.ops, tk.policy
    ops.td = torch.zeros(n, device="cuda")
    ops.scratch = torch.zeros(ops.lib.r4_rainbow_scratch_size(A, Z, n), device="cuda")
    ops.grad_(pol, tk.replay, idx, w, 1.0, 1.0 / n)
    obs, act, rew, nobs, done = tk.replay.gather(idx)
    assert (pol.forward(nobs)[1].argmax(1) != pol.forward(nobs, pol.target)[1].argmax(1)).any()   # double Q matters
    loss, td = pol.loss(obs, act, rew, nobs, done, w, 1.0, 1.0 / n)
    pol.flat.grad = None
    loss.backward()
    ref = pol.flat.grad
    err = (ops.grad - ref).abs().max()
    assert float(err) <= 2e-5 * float(ref.abs().max()), (float(err), float(ref.abs().max()))
    for lo, hi in pol.slices:                 # every tensor gets a gradient
        assert float(ref[lo:hi].abs().max()) > 0
    assert float((ops.td - td).abs().max()) < 1e-4 * max(1.0, float(td.abs().max()))
    q = pol.forward(obs)[1].gather(1, act.long().unsqueeze(1)).mean()
    for got, want in ((ops.stats[0], loss.detach()), (ops.stats[1], td.mean()), (ops.stats[2], q.detach())):
        assert abs(float(got) - float(want)) <= 1e-4 * max(1.0, abs(float(want)))


def test_whole_sgd_step_matches_the_twin():
    import torch
    tk, tt = _pair(v_max=10.0, train_batch_size=128)
    _fill((tk, tt))
    tk.policy_ts = tt.policy_ts = 1000          # the first step copies the target
    u, = tk.draws()
    tk.sgd_step(u)
    tt.sgd_step(u)
    g = tt.policy.flat.grad      # Adam moves a parameter by about lr * sign(g): compare where g is clearly non-zero
    big = g.abs() > 1e-3 * g.abs().max()
    for x, y in ((tk.policy.flat.detach(), tt.policy.flat.detach()), (tk.policy.target, tt.policy.target)):
        err = float((x - y)[big].abs().max())
        assert err <= 1e-5 * float(y.abs().max()), err
    assert torch.equal(tk.policy.target, tk.policy.flat.detach())
    N = tk.replay.size
    assert torch.allclose(tk.replay.prio[:N], tt.replay.prio[:N], rtol=1e-4)
    assert torch.allclose(tk.replay.max_prio, tt.replay.max_prio, rtol=1e-4)
    t0 = tk.policy.target.clone()
    tk.sgd_step(*tk.draws())                    # no sampling since the copy: the target stays
    assert torch.equal(tk.policy.target, t0) and not torch.equal(tk.policy.flat.detach(), t0)


def test_seeded_runs_are_bit_identical():
    import torch
    out = []
    for _ in range(2):
        tk, _ = _pair(learning_starts=72, timesteps_per_iteration=150, train_batch_size=64)
        for _ in range(3):
            tk.train()
        torch.cuda.synchronize()
        out.append((tk.policy.flat.detach().clone(), tk.policy.target.clone(), tk.replay.prio.clone()))
    for a, b in zip(*out):
        assert torch.equal(a, b)


@pytest.mark.parametrize("seq", [False, True])
def test_rainbow_end_to_end_on_cuda_env(seq, tmp_path):
    import torch
    from test_gpu_parity import _synthetic, make_env
    from rl4rs_b200.trainer import get_rl_model
    B = 64
    cfg, cat, log, w = _synthetic(B, seq, support_rllib_mask=False, is_eval=False, cache_size=4 * B)
    env = make_env(cfg, seq, cat, log, w, output_format="torch")
    T = cfg["max_steps"]
    tr = get_rl_model("RAINBOW", {"learning_starts": 2 * B * T, "buffer_size": 4 * B * T}, env=env)
    assert tr.use_kernels and tr.algo == "RAINBOW"
    per_it = -(-1000 // (B * T))
    res = [tr.train() for _ in range(3)]
    added = 3 * per_it * B * T
    assert res[-1]["timesteps_total"] == added and tr.replay.size == min(added, 4 * B * T)
    assert sum(r["sgd_steps"] for r in res) == 3 * per_it - 1          # no step before learning_starts
    assert all(np.isfinite(r["loss"]) for r in res[1:]) and np.isfinite(res[-1]["mean_q"])
    assert torch.isfinite(tr.policy.flat).all() and np.isfinite(tr.evaluate(1))
    a = tr.compute_actions(env.reset())
    assert a.shape == (B,) and a.dtype == np.int32 and a.min() >= 0 and a.max() < A
    path = tr.save(str(tmp_path))
    tr2 = get_rl_model("RAINBOW", {}, env=env)
    tr2.restore(path)
    assert torch.equal(tr2.policy.flat, tr.policy.flat) and torch.equal(tr2.policy.target, tr.policy.target)
    assert torch.equal(tr2.ops.m, tr.ops.m) and tr2.critic_steps == tr.critic_steps
    np.testing.assert_array_equal(tr2.compute_actions(env.reset()).shape, (B,))
