"""GPU: the PA-DQN kernels (csrc/r4_padqn.cuh) against float64 and the torch twin -- the pair scorer over every (row, item)
pair at n from 1 to 8192, A at 284 and the ends r4_create accepts, dense and one-hot item vectors and three mask regimes;
argmax and SoftQ; the next-mask store; the gradient and a whole r4_padqn_train_step; determinism, launch counts, peak
memory -- and the trainer end to end on the CUDA env, with ope_eval over it."""
import numpy as np
import pytest

import padqn_ref64 as ref

pytestmark = pytest.mark.gpu

NS = (1, 7, 128, 1000, 4096, 8192)


def _qm64(flat, obs, mask, emb, D):
    """Qm in float64 on the device (torch), in row chunks: the reference of the pair scorer at every size."""
    import torch
    p = {k: torch.as_tensor(v, device="cuda") for k, v in ref.params(flat.detach().double().cpu().numpy(), D).items()}
    P = emb.double() @ p["w1"][256:]
    out = []
    for i in range(0, obs.shape[0], 128):
        S = obs[i:i + 128].double() @ p["w1"][:256] + p["b1"]
        h = torch.tanh(torch.tanh(S[:, None, :] + P[None]) @ p["w2"] + p["b2"])
        out.append((h @ p["w3"])[..., 0] + p["b3"][0])
    q = torch.cat(out)
    return torch.where(mask.bool(), q, torch.full_like(q, ref.FLOAT_MIN))


def _net(A, onehot, seed=0):
    import torch
    from rl4rs_b200.policy import ParametricQNetwork
    from rl4rs_b200.trainer import PADQNKernelOps
    emb = ref.item_vectors(A, 32, seed=seed, onehot=onehot)
    pol = ParametricQNetwork(emb, "cuda", seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        pol.flat.add_(0.05 * torch.randn(pol.n_params, generator=g).cuda())
        pol.flat[pol.slices[4][0]:pol.slices[4][1]] *= 20.0                # Q of order 1
        pol.target.copy_(pol.flat.detach() + 0.05 * torch.randn(pol.n_params, generator=g).cuda())
    ops = PADQNKernelOps(pol.emb, "cuda", pol.n_params, 64)
    ops.refresh(pol)
    return pol, ops


def _masks(regime, n, A, seed):
    import torch
    m = {"ones": lambda: np.ones((n, A), np.uint8), "env": lambda: ref.env_like_masks(n, A, seed),
         "planted": lambda: ref.planted_masks(n, A, seed)}[regime]()
    return torch.as_tensor(m).cuda()


@pytest.mark.parametrize("A", [149, 284, 512])
@pytest.mark.parametrize("onehot", [False, True])
@pytest.mark.parametrize("regime", ["ones", "env", "planted"])
def test_pair_scorer_grid(A, onehot, regime, record_property):
    import torch
    pol, ops = _net(A, onehot, seed=A)
    D = pol.D
    worst = 0.0
    for n in NS:
        g = torch.Generator().manual_seed(n)
        obs = torch.randn(n, 256, generator=g).cuda()
        mask = _masks(regime, n, A, n)
        q = torch.empty(n, A, device="cuda")
        a = torch.empty(n, dtype=torch.int32, device="cuda")
        ops.act(pol, obs, mask, False, 3, 0, a, q)
        q64 = _qm64(pol.flat, obs, mask, pol.emb, D)
        live = mask.bool()
        assert torch.equal(q == ref.FLOAT_MIN, ~live), n
        bar = 1e-4 * float(q64[live].abs().max()) if bool(live.any()) else 1e-4
        err = float((q.double() - q64)[live].abs().max()) if bool(live.any()) else 0.0
        assert err <= bar, (n, err, bar)
        worst = max(worst, err / bar)
        # argmax: equal wherever the f64 top-two margin exceeds twice the bar; an all-masked row takes item 0
        top2 = q64.topk(min(2, A), 1).values
        clear = (top2[:, 0] - top2[:, 1]) > 2 * bar
        assert torch.equal(a.long()[clear], q64.argmax(1)[clear]), n
        dead = ~live.any(1)
        assert bool((a[dead] == 0).all())
        # SoftQ on the kernel's own uniforms: equal to the f64 rule wherever u is not within the bar of a CDF step
        s1, s2 = (torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2))
        ops.act(pol, obs, mask, True, 5, 1000, s1)
        ops.act(pol, obs, mask, True, 5, 1000, s2)
        assert torch.equal(s1, s2)
        u = ref.uniforms(5, 1000, n)
        qh = q64.cpu().numpy()
        e = np.exp(qh - qh.max(1, keepdims=True))
        cdf = np.cumsum(e, 1) / e.sum(1, keepdims=True)
        margin = np.abs(cdf - u[:, None]).min(1) > 1e-3
        want = ref.act(qh, u)
        got = s1.cpu().numpy()
        assert np.array_equal(got[margin], want[margin]), n
        assert bool(live[torch.arange(n, device="cuda")[~dead], s1.long()[~dead]].all())
    record_property("worst_err_over_bar", worst)


def test_peak_memory_at_8192_rows_holds_no_pair_plane():
    import torch
    pol, ops = _net(284, False)
    n = 8192
    obs = torch.randn(n, 256, device="cuda")
    mask = torch.ones(n, 284, dtype=torch.uint8, device="cuda")
    a, q = torch.empty(n, dtype=torch.int32, device="cuda"), torch.empty(n, 284, device="cuda")
    ops.act(pol, obs, mask, False, 0, 0, a, q)                      # sizes the act scratch
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ops.act(pol, obs, mask, False, 0, 0, a, q)
    torch.cuda.synchronize()
    plane = n * 284 * 256 * 4                                       # one f32 hidden plane of every pair: 2.4 GB
    assert torch.cuda.max_memory_allocated() - base < 1 << 20
    assert ops.act_scratch.numel() * 4 < plane / 20


def _pair(B=8, **cfg):
    import torch
    from test_trainer_padqn_cpu import FakeEnv
    from rl4rs_b200.trainer import get_rl_model

    class HostEnv(FakeEnv):
        def step(self, a):
            return super().step(a.cpu())
    cfg = dict({"buffer_size": 500}, **cfg)
    tk = get_rl_model("PADQN", cfg, env=HostEnv(B, A=284, D=32), device="cuda")
    tt = get_rl_model("PADQN", dict(cfg, use_kernels=False), env=HostEnv(B, A=284, D=32), device="cuda")
    assert tk.use_kernels and not tt.use_kernels
    with torch.no_grad():
        g = torch.Generator().manual_seed(1)
        tk.policy.flat.add_(0.05 * torch.randn(tk.policy.n_params, generator=g).cuda())
        tk.policy.flat[tk.policy.slices[4][0]:tk.policy.slices[4][1]] *= 30.0
        tk.policy.target.copy_(tk.policy.flat.detach() + 0.05 * torch.randn(tk.policy.n_params, generator=g).cuda())
        tt.policy.flat.copy_(tk.policy.flat)
        tt.policy.target.copy_(tk.policy.target)
    tk.ops.refresh(tk.policy)
    return tk, tt


def _fill(trs, T=9, B=40, seed=0):
    import torch
    g = torch.Generator().manual_seed(seed)
    obs, fin = torch.randn(T, B, 256, generator=g).cuda(), torch.randn(B, 256, generator=g).cuda()
    mask = torch.as_tensor(ref.planted_masks(T * B, 284, seed)).view(T, B, 284).cuda()
    mask[:, :, 1] = 1                          # mid-episode states keep an item; the sparse rest is planted
    fmask = torch.as_tensor(ref.env_like_masks(B, 284, seed)).cuda()
    fmask[::6] = 0                                                                    # all-masked final states
    act = torch.randint(0, 284, (T, B), generator=g, dtype=torch.int32).cuda()
    rew = torch.randn(T, B, generator=g).cuda()
    done = torch.zeros(T, B, dtype=torch.uint8).cuda()
    done[-1] = 1
    for tr in trs:
        tr.replay.store(obs, fin, act, rew, done, mask, fmask)


@pytest.mark.parametrize("T,B", [(9, 40), (36, 10)])
def test_store_kernel_is_bit_exact(T, B):
    tk, tt = _pair()
    for ep in range(2):                        # 720 rows into 500 slots: wraps around
        _fill([tk, tt], T, B, seed=ep)
    n = tk.replay.size
    for name in ("obs", "action", "reward", "new_obs", "done", "next_mask", "prio"):
        import torch
        assert torch.equal(getattr(tk.replay, name)[:n], getattr(tt.replay, name)[:n]), name


def test_gradient_matches_float64_and_autograd():
    import torch
    tk, tt = _pair(train_batch_size=256)
    _fill([tk, tt])
    n = 200
    idx = torch.randperm(tk.replay.size, generator=torch.Generator().manual_seed(3))[:n].cuda()
    w = (torch.rand(n, generator=torch.Generator().manual_seed(4)) + 0.5).cuda()
    batch = tk.replay.gather(idx)
    done = batch[4]
    tk.ops.grad_(tk.policy, tk.replay, idx, w, 0.9, 1.0 / n)
    pol = tt.policy
    loss, td, q = pol.loss(*batch, weights=w, gamma=0.9)
    pol.flat.grad = None
    loss.backward()
    live_next = batch[5].bool().any(1) | (done == 1)
    assert bool(live_next.all())                     # every all-masked next state of _fill ends its episode
    b64 = [x.double().cpu().numpy() if x.is_floating_point() else x.cpu().numpy() for x in batch]
    P, PT = ref.params(pol.flat.detach().double().cpu().numpy(), 32), ref.params(pol.target.double().cpu().numpy(), 32)
    l64, td64, q64, g64 = ref.loss_and_grads(P, PT, pol.emb.double().cpu().numpy(), b64[0], b64[1], b64[2], b64[3],
                                             b64[4].astype(np.float64), b64[5], w.double().cpu().numpy(), gamma=0.9)
    assert float((tk.ops.td[:n].double().cpu() - torch.as_tensor(td64)).abs().max()) <= 1e-4 * np.abs(td64).max()
    st = tk.ops.stats.double().cpu().numpy()
    assert abs(st[0] - l64) <= 1e-4 * abs(l64) and abs(st[2] - q64.mean()) <= 1e-4 * np.abs(q64).max()
    gk = tk.ops.grad.double().cpu().numpy()
    gt = pol.flat.grad.double().cpu().numpy()
    for (lo, hi), name in zip(pol.slices, ref.NAMES):
        g = g64[name].reshape(-1)
        bar = 1e-4 * np.abs(g).max()
        assert np.abs(gk[lo:hi] - g).max() <= bar, name
        assert np.abs(gt[lo:hi] - g).max() <= bar, name


def test_whole_sgd_step_matches_float64_and_the_twin():
    import torch
    tk, tt = _pair(grad_clip=0.5, train_batch_size=64)
    _fill([tk, tt])
    u = torch.rand(64, generator=torch.Generator().manual_seed(7)).cuda()
    f0, t0 = tk.policy.flat.detach().double().cpu().numpy(), tk.policy.target.double().cpu().numpy()
    idx, w = tk.replay.sample(u, 0.4)
    l0 = tk.ops.launches
    tk.ops.train_step(tk.policy, tk.replay, u, 1, True, tk._hp())
    torch.cuda.synchronize()
    launches = tk.ops.launches - l0
    assert launches == 11
    batch = tt.replay.gather(idx)
    td, stats = tt.twin_step(*batch, w, True)
    b64 = [x.double().cpu().numpy() if x.is_floating_point() else x.cpu().numpy() for x in batch]
    P, PT = ref.params(f0, 32), ref.params(t0, 32)
    _, _, _, g64 = ref.loss_and_grads(P, PT, tk.policy.emb.double().cpu().numpy(), b64[0], b64[1], b64[2], b64[3],
                                      b64[4].astype(np.float64), b64[5], w.double().cpu().numpy())
    # the step's gradient (the scratch's last plane) against float64, tensor by tensor; then the optimiser on that gradient.
    # (Adam's first step is g / |g| elementwise, so elements whose |g| is below the gradient's rounding are compared through
    # the gradient, not through the step.)
    np_ = tk.policy.n_params
    gk = tk.ops.scratch[-((np_ + 3) // 4 * 4):][:np_].double().cpu().numpy()
    g = ref.flat_grad(g64, 32)
    for (lo, hi), name in zip(tk.policy.slices, ref.NAMES):
        assert np.abs(gk[lo:hi] - g[lo:hi]).max() <= 1e-4 * np.abs(g[lo:hi]).max(), name
    f1, t1, _, _ = ref.apply(f0, t0, gk, np.zeros_like(f0), np.zeros_like(f0), 1, 32, clip=0.5, copy_target=True)
    fk = tk.policy.flat.detach().double().cpu().numpy()
    assert np.abs(fk - f1).max() < 1e-6
    sk, st = tk.ops.stats.double().cpu().numpy(), stats.double().cpu().numpy()
    assert np.abs(sk - st).max() <= 1e-4 * np.abs(st).max()
    assert torch.equal(tk.policy.target, tk.policy.flat.detach())
    # the caches follow: acting after the step equals a fresh refresh
    obs = torch.randn(50, 256, device="cuda")
    mask = torch.ones(50, 284, dtype=torch.uint8, device="cuda")
    q1, q2 = torch.empty(50, 284, device="cuda"), torch.empty(50, 284, device="cuda")
    a = torch.empty(50, dtype=torch.int32, device="cuda")
    tk.ops.act(tk.policy, obs, mask, False, 0, 0, a, q1)
    tk.ops.refresh(tk.policy)
    tk.ops.act(tk.policy, obs, mask, False, 0, 0, a, q2)
    assert torch.equal(q1, q2)
    # prioritized: the new priorities are (|td| + eps)^alpha at the sampled slots
    p = tk.replay.prio[idx.unique()]
    assert bool(torch.isfinite(p).all())


def test_seeded_runs_are_bit_identical_and_launches_constant(record_property):
    import torch
    out, per_step = [], set()
    for _ in range(2):
        tk, _ = _pair(learning_starts=72, timesteps_per_iteration=150, train_batch_size=64, target_network_update_freq=100)
        for _ in range(3):
            tk.train()
        torch.cuda.synchronize()
        u = tk.draws()[0]
        for copy in (False, True):
            l0 = tk.ops.launches
            tk.ops.train_step(tk.policy, tk.replay, u, tk.critic_steps + 1, copy, tk._hp())
            per_step.add(tk.ops.launches - l0)
        # the ring's stored slots only: 15 episodes of 32 transitions leave 20 of its 500 slots unwritten (torch.empty, never
        # read by the sampler, whose prefix sums stop at the replay's size)
        n = tk.replay.size
        assert n == 480 < tk.replay.C
        out.append({"flat": tk.policy.flat.detach().clone(), "target": tk.policy.target.clone(),
                    "prio": tk.replay.prio[:n].clone(), "next_mask": tk.replay.next_mask[:n].clone(),
                    "cache": tk.ops.cache.clone(), "target_cache": tk.ops.target_cache.clone(), "stats": tk.ops.stats.clone()})
    for k in out[0]:
        assert torch.equal(out[0][k], out[1][k]), k
    assert per_step == {11}
    record_property("launches_per_sgd_step", 11)


@pytest.mark.parametrize("seq", [False, True])
def test_padqn_end_to_end_on_cuda_env(seq, tmp_path):
    import torch
    from test_gpu_parity import _synthetic, make_env
    from rl4rs_b200.trainer import get_rl_model
    B = 64
    cfg, cat, log, w = _synthetic(B, seq, support_rllib_mask=True, is_eval=False, cache_size=4 * B)
    env = make_env(cfg, seq, cat, log, w, output_format="torch")
    T = cfg["max_steps"]
    tr = get_rl_model("PADQN", {"learning_starts": 2 * B * T, "buffer_size": 4 * B * T}, env=env)
    assert tr.use_kernels and tr.algo == "PADQN" and tr.policy.D == env.sim.engine.emb_dim
    per_it = -(-1000 // (B * T))
    res = [tr.train() for _ in range(3)]
    added = 3 * per_it * B * T
    assert res[-1]["timesteps_total"] == added and tr.replay.size == min(added, 4 * B * T)
    assert sum(r["sgd_steps"] for r in res) == 3 * per_it - 1
    assert all(np.isfinite(r["loss"]) for r in res[1:]) and np.isfinite(res[-1]["mean_q"])
    assert torch.isfinite(tr.policy.flat).all() and np.isfinite(tr.evaluate(1))
    obs = env.reset()
    a = tr.compute_actions(obs)
    assert a.shape == (B,) and a.dtype == np.int32 and a.min() >= 0 and a.max() < 284
    m = obs["action_mask"].cpu().numpy()
    assert m[np.arange(B), a].all()
    _, _, infos = tr.compute_actions(obs, full_fetch=True)
    assert infos["q_values"].shape == (B, 284) and np.array_equal(infos["q_values"] == ref.FLOAT_MIN, m == 0)
    path = tr.save(str(tmp_path))
    tr2 = get_rl_model("PADQN", {}, env=env)
    tr2.restore(path)
    assert torch.equal(tr2.policy.flat, tr.policy.flat) and torch.equal(tr2.policy.target, tr.policy.target)
    assert torch.equal(tr2.ops.m, tr.ops.m) and tr2.critic_steps == tr.critic_steps
    assert torch.equal(tr2.ops.cache, tr.ops.cache) and torch.equal(tr2.ops.target_cache, tr.ops.target_cache)
    np.testing.assert_array_equal(tr2.compute_actions(obs), tr.compute_actions(obs))


def test_ope_eval_over_a_padqn_trainer(tmp_path):
    import io
    from contextlib import redirect_stdout
    from test_gpu_ope import _env, _weights
    from rl4rs_b200 import offline_evaluation as oe, trainer
    B = 64
    p = str(tmp_path / "w.npz")
    np.savez(p, **dict(_weights(100000, 284, 1)))
    cfg, cat, env = _env(False, B, True, False)
    cfg = dict(cfg, catalog=cat)
    model = trainer.get_rl_model("PADQN", {}, env, seed=3)
    bm = oe.behavior_model(dict(cfg), p, device="cuda", use_kernels=True)
    with redirect_stdout(io.StringIO()):
        m = oe.ope_eval(dict(cfg, epoch=1), env, model, sample_model=bm, use_kernels=True)
    assert m.shape == (1, 4, 2) and np.all(np.isfinite(m[:, :, 0]))
