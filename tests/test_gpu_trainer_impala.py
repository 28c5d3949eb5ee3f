"""GPU: the IMPALA kernels (r4_policy_eval / r4_gauss_eval, r4_vtrace, r4_impala_step / r4_gauss_impala_step) against a
float64 autograd reference of the torch twins, tensor by tensor, on off-policy batches whose behaviour policy is a perturbed
copy of the learner's (rho on both sides of the thresholds); the fused step against the same kernels run one by one, run to
run, and over a second pass; its launch count; rejected arguments; PG through the kernels against the torch path; and short
PG / IMPALA runs on the synthetic env.  Bounds are test_gpu_learner_shapes.py's for the A2C gradient."""
import math

import numpy as np
import pytest
import torch

import learner_ref64 as R
from test_gpu_learner_launches import _launched, _rejected
from test_gpu_learner_shapes import TOL, _check_grad, _check_rows, _check_stats, _cmp

pytestmark = pytest.mark.gpu

D = 32
HP = {"gamma": 1.0, "rho": 1.0, "rho_pg": 1.0, "vf": 0.5, "ent": 0.01}
# (A, T, B): every A, T and B of the grid, the largest batch (T = 81, B = 4096) included
MASK_CASES = [(149, 2, 4096), (284, 9, 7), (512, 36, 1), (284, 81, 4096), (149, 36, 7), (512, 2, 1), (284, 9, 4096)]
GAUSS_CASES = [(2, 7), (9, 4096), (36, 1), (81, 7)]


def vtrace64(blogp, tlogp, value, reward, gamma, rho_bar, rho_pg_bar, drop_last):
    """from_importance_weights in float64 over [T, B] episodes (done at T - 1) -> vs, pg_adv over the kept steps."""
    T = reward.shape[0]
    K = T - 1 if drop_last else T
    rho = (tlogp - blogp).exp()[:K]
    disc = torch.full((K, reward.shape[1]), float(gamma), dtype=torch.float64, device=reward.device)
    if not drop_last:
        disc[T - 1] = 0.0
    boot = value[T - 1]
    delta = rho.clamp(max=rho_bar) * (reward[:K] + disc * torch.cat([value[1:K], boot[None]]) - value[:K])
    acc, out = torch.zeros_like(boot), []
    for t in reversed(range(K)):
        acc = delta[t] + disc[t] * rho[t].clamp(max=1.0) * acc
        out.append(acc)
    vs = torch.stack(out[::-1]) + value[:K]
    pg = rho.clamp(max=rho_pg_bar) * (reward[:K] + disc * torch.cat([vs[1:], boot[None]]) - value[:K])
    return vs, pg


def impala_ref(twin, flat, inputs, action, blogp, reward, T, B, hp, drop_last):
    """The VTraceLoss of the twin at float64 `flat` -> dict of logp, value, vs, pg_adv ([T*B] / [K*B]), grad and stats."""
    pol = R._f64(twin, flat)
    d, value = pol.forward(*[R._d(x) if x.is_floating_point() else x for x in inputs])
    logp, _, ent = pol.terms(d, action)
    with torch.no_grad():
        vs, pg = vtrace64(blogp.double(), logp.detach().view(T, B), value.detach().view(T, B), reward.double(), hp["gamma"],
                          hp["rho"], hp["rho_pg"], drop_last)
    k = vs.numel()
    pi = -(logp[:k] * pg.reshape(-1))
    vf = 0.5 * (value[:k] - vs.reshape(-1)) ** 2
    total = pi + hp["vf"] * vf - hp["ent"] * ent[:k]
    total.sum().backward()
    stats = torch.tensor([float(pi.sum()), float(vf.sum()), 0.0, float(ent[:k].sum()), float(total.sum())], dtype=torch.float64)
    return {"logp": logp.detach(), "value": value.detach(), "vs": vs.reshape(-1), "pg": pg.reshape(-1),
            "grad": pol.flat.grad.detach(), "stats": stats}


def _hp_tuple(hp, drop_last):
    return (hp["gamma"], hp["rho"], hp["rho_pg"], int(drop_last), hp["vf"], hp["ent"])


def _setup(conti, size, T, B, seed):
    """-> (policy, ops, rollout buffer filled by the act kernel of a perturbed copy of the policy, inputs, action)."""
    from rl4rs_b200.policy import GaussianPolicy, MaskedPolicy
    from rl4rs_b200.trainer import GaussKernelOps, GaussRolloutBuffer, KernelOps, RolloutBuffer
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(seed)
    pol = (GaussianPolicy if conti else MaskedPolicy)(size, dev, seed=3)
    with torch.no_grad():
        pol.flat.add_((0.02 if conti else 0.05) * torch.randn(pol.n_params, generator=g).to(dev))
    ops = (GaussKernelOps if conti else KernelOps)(size, dev, pol.n_params)
    behaviour = pol.flat.detach() + (0.05 if conti else 0.3) * torch.randn(pol.n_params, generator=g).to(dev)
    buf = (GaussRolloutBuffer if conti else RolloutBuffer)(T, B, size, dev)
    buf.obs.copy_(torch.randn(T, B, 256, generator=g))
    if not conti:
        m = torch.rand(T, B, size, generator=g) < 0.5
        m[..., 0] |= ~m.any(-1)
        buf.mask.copy_(m.to(torch.uint8))
    for t in range(T):
        if conti:
            ops.act(behaviour, buf.obs[t], True, 5, buf.action[t], torch.empty(B, size, device=dev), buf.logp[t], buf.value[t],
                    buf.dist[t])
        else:
            a = torch.empty(B, dtype=torch.int32, device=dev)
            ops.act(behaviour, buf.obs[t], buf.mask[t], True, 5, a, buf.logp[t], buf.value[t], buf.logits[t])
            buf.action[t].copy_(a)
    for t in range(8, T, 9):
        buf.reward[t].copy_(torch.rand(B, generator=g) * 5)
    buf.reward[T - 1].add_(torch.rand(B, generator=g).to(dev))
    n = T * B
    inputs = (buf.obs.reshape(n, 256),) if conti else (buf.obs.reshape(n, 256), buf.mask.reshape(n, size))
    action = buf.action.reshape(n, size) if conti else buf.action.reshape(n)
    return pol, ops, buf, inputs, action


def _work(T, B):
    return tuple(torch.zeros(T, B, device="cuda") for _ in range(4))


def _adam64(p, g, m, v, step, lr, clip):
    gn = float(g.norm())
    if clip > 0 and clip / (gn + 1e-6) < 1:
        g = g * (clip / (gn + 1e-6))
    m2, v2 = 0.9 * m + 0.1 * g, 0.999 * v + 0.001 * g * g
    return p - lr / (1 - 0.9 ** step) * m2 / ((v2 / (1 - 0.999 ** step)).sqrt() + 1e-8)


def _check_step(what, pol, ops, buf, inputs, action, T, B, hp, drop_last, twin):
    """One fused step against the float64 reference: every output, the gradient, the statistics, and the clipped Adam
    update (moments from an earlier step, the clip active at half the reference norm)."""
    flat0, m0, v0 = pol.flat.detach().clone(), ops.m.clone(), ops.v.clone()
    ref = impala_ref(twin, flat0, inputs, action, buf.logp, buf.reward, T, B, hp, drop_last)
    K = (T - 1 if drop_last else T)
    rho = (ref["logp"].view(T, B)[:K] - buf.logp[:K].double()).exp()
    clip = 0.5 * float(ref["grad"].norm())
    work = _work(T, B)
    ops.stats.zero_()
    ops.impala_step(None, pol.flat, buf, _hp_tuple(hp, drop_last), 1e-3, clip, work)
    logp, value, vs, pg = (w.reshape(-1) for w in work)
    k = K * B
    _check_rows(what + " logp", logp, ref["logp"])
    _check_rows(what + " value", value, ref["value"])
    vscale = max(1.0, float(ref["vs"].abs().max()))
    assert _cmp(what + " vs", vs[:k], ref["vs"], TOL * vscale) <= 1
    assert _cmp(what + " pg_adv", pg[:k], ref["pg"], TOL * vscale) <= 1
    if drop_last:
        assert torch.equal(vs[k:], value[k:]) and bool((pg[k:] == 0).all())
    _check_grad(what, ops.grad, ref["grad"], twin)
    _check_stats(what, ops.stats.double().cpu(), ref["stats"], keep=[0, 1, 3, 4])
    want = _adam64(flat0.double(), ref["grad"], m0.double(), v0.double(), ops.step, 1e-3, clip)
    dref, dgot = want - flat0.double(), pol.flat.detach().double() - flat0.double()
    assert _cmp(what + " adam", dgot, dref, 1e-3 * float(dref.abs().max())) <= 1
    return rho


def _warm(ops, pol):
    """Adam moments of a few earlier steps, so the update depends on the gradient's values and not only on its signs."""
    g = torch.Generator().manual_seed(9)
    ops.m.copy_(1e-2 * torch.randn(pol.n_params, generator=g))
    ops.v.copy_(1e-3 * (0.5 + torch.rand(pol.n_params, generator=g)))
    ops.step = 4


@pytest.mark.parametrize("A,T,B", MASK_CASES)
def test_mask_impala_step_against_float64(A, T, B):
    pol, ops, buf, inputs, action = _setup(False, A, T, B, seed=A + T + B)
    _warm(ops, pol)
    hp = dict(HP, rho=1.5, rho_pg=0.8) if T == 36 else HP
    rho = _check_step("policy impala A%d T%d B%d" % (A, T, B), pol, ops, buf, inputs, action, T, B, hp, True, pol)
    if T * B > 100:
        assert bool((rho > hp["rho"]).any() & (rho < hp["rho_pg"]).any())


@pytest.mark.parametrize("T,B", GAUSS_CASES)
def test_gauss_impala_step_against_float64(T, B):
    pol, ops, buf, inputs, action = _setup(True, D, T, B, seed=T + B)
    _warm(ops, pol)
    rho = _check_step("gauss impala T%d B%d" % (T, B), pol, ops, buf, inputs, action, T, B, HP, T != 2, pol)
    if T * B > 100:
        assert bool((rho > 1).any() & (rho < 1).any())


def test_second_pass_is_off_policy_and_matches_the_reference():
    """num_sgd_iter = 2: the second step over the same batch (behaviour logp unchanged) has rho != 1 and still matches."""
    pol, ops, buf, inputs, action = _setup(False, 284, 9, 512, seed=1)
    with torch.no_grad():                          # on-policy first pass: the stored logp is the learner's own
        work = _work(9, 512)
        ops.eval(pol.flat, inputs, action, work[0].reshape(-1), work[1].reshape(-1))
        buf.logp.copy_(work[0])
    rho = _check_step("policy impala pass 1", pol, ops, buf, inputs, action, 9, 512, HP, True, pol)
    assert float((rho - 1).abs().max()) < 1e-5                  # 1 up to the float32 logp the reference is compared with
    rho = _check_step("policy impala pass 2", pol, ops, buf, inputs, action, 9, 512, HP, True, pol)
    assert float((rho - 1).abs().max()) > 1e-3


@pytest.mark.parametrize("conti", [False, True])
def test_fused_step_is_the_kernels_run_one_by_one_and_reproducible(conti):
    T, B = 9, 600
    pol, ops, buf, inputs, action = _setup(conti, D if conti else 284, T, B, seed=2)
    hp = _hp_tuple(HP, True)
    n, k = T * B, (T - 1) * B
    flat0 = pol.flat.detach().clone()
    runs = []
    for clip in (0.0, 0.0, 3.0, 3.0):               # clip 0: off; 3: active (the summed gradient's norm is far above)
        with torch.no_grad():
            pol.flat.copy_(flat0)
        ops.m.zero_(); ops.v.zero_(); ops.step = 0; ops.stats.zero_()
        work = _work(T, B)
        ops.impala_step(None, pol.flat, buf, hp, 1e-3, clip, work)
        runs.append((pol.flat.detach().clone(), ops.grad.clone(), ops.stats.clone(), ops.m.clone(), ops.v.clone()) + work)
    for a, b in ((0, 1), (2, 3)):
        assert all(torch.equal(x, y) for x, y in zip(runs[a], runs[b]))
    assert not torch.equal(runs[0][0], runs[2][0])
    # forward, V-trace, gradient and Adam as four calls
    with torch.no_grad():
        pol.flat.copy_(flat0)
    ops.m.zero_(); ops.v.zero_(); ops.step = 0; ops.stats.zero_()
    logp, value, vs, pg = _work(T, B)
    ops.eval(pol.flat, inputs, action, logp, value)
    ops.vtrace(buf.logp, logp, value, buf.reward, hp, vs, pg)
    cols = buf.a2c_columns()
    gh = {"clip": 0.0, "vf_clip": 0.0, "vf_coeff": HP["vf"], "kl_coeff": 0.0, "ent_coeff": HP["ent"]}
    ops.policy_grad(1, pol.flat, cols + (pg.reshape(n), vs.reshape(n)), None, 0, k, gh, 1.0, 1.0)
    ops.adam(pol.flat, 1e-3, 1.0, None)
    sep = (pol.flat.detach(), ops.grad, ops.stats, ops.m, ops.v, logp, value, vs, pg)
    assert all(torch.equal(x, y) for x, y in zip(runs[0], sep))


def test_launches_per_step():
    """DESIGN.md: r4_impala_step launches 6 kernels per step (5 without the clip); r4_gauss_impala_step 4 + 2 per chunk of
    2048 kept rows (3 + 2 per chunk without the clip)."""
    for conti, T, B in ((False, 9, 64), (True, 9, 512)):
        pol, ops, buf, inputs, action = _setup(conti, D if conti else 284, T, B, seed=4)
        hp = _hp_tuple(HP, True)
        chunks = -(-(T - 1) * B // 2048)
        for clip in (10.0, 0.0):
            want = (4 + 2 * chunks if conti else 6) - (clip == 0.0)
            assert _launched(lambda: ops.impala_step(None, pol.flat, buf, hp, 1e-3, clip, _work(T, B))) == want, (conti, clip)
        work = _work(T, B)
        for bad in ((1.0, 1.0, 1.0, 1, 0.5, 0.01, 82), (1.5, 1.0, 1.0, 1, 0.5, 0.01, T), (1.0, 0.0, 1.0, 1, 0.5, 0.01, T)):
            buf.T = bad[-1]
            _rejected(lambda: ops.impala_step(None, pol.flat, buf, bad[:-1], 1e-3, 10.0, work))
        buf.T = T
        one = type(buf).__new__(type(buf))
        one.__dict__.update(buf.__dict__, T=1)
        _rejected(lambda: ops.impala_step(None, pol.flat, one, hp, 1e-3, 10.0, work))      # drop-last on one step
        _rejected(lambda: ops.vtrace(buf.logp, work[0], work[1], buf.reward, (1.0, 1.0, -1.0, 1), work[2], work[3]))
        n = T * B
        assert _launched(lambda: ops.eval(pol.flat, inputs, action, work[0].reshape(n), work[1].reshape(n))) == 1
        assert _launched(lambda: ops.vtrace(buf.logp, work[0], work[1], buf.reward, hp, work[2], work[3])) == 1
        torch.cuda.synchronize()


def _fake_rollout(tr, seed):
    """A rollout of random observations and masks whose actions, logp and values come from the trainer's act kernel."""
    buf = tr.buf
    g = torch.Generator().manual_seed(seed)
    buf.obs.copy_(torch.randn(buf.obs.shape, generator=g))
    m = torch.rand(buf.mask.shape, generator=g) < 0.3
    m[..., 1] = True
    buf.mask.copy_(m.to(torch.uint8))
    a = torch.empty(tr.B, dtype=torch.int32, device="cuda")
    for t in range(tr.T):
        tr.ops.act(tr.policy.flat, buf.obs[t], buf.mask[t], True, 3, a, buf.logp[t], buf.value[t], buf.logits[t])
        buf.action[t].copy_(a)
    buf.reward.copy_(torch.rand(buf.reward.shape, generator=g))


def test_pg_kernels_equal_the_torch_path():
    from rl4rs_b200.trainer import PGTrainer
    from test_trainer_cpu import FakeEnv
    env = FakeEnv(256)
    tk = PGTrainer({"gamma": 0.9}, env, device="cuda")
    tt = PGTrainer({"gamma": 0.9, "use_kernels": False}, env, device="cuda")
    assert tk.use_kernels and not tt.use_kernels
    _fake_rollout(tk, 1)
    for name in ("obs", "mask", "action", "logp", "value", "logits", "reward"):
        getattr(tt.buf, name).copy_(getattr(tk.buf, name))
    assert torch.equal(tk.returns(tk.buf), tt.returns(tt.buf))          # r4_gae over zero values = the torch loop
    p0 = tk.policy.flat.detach().clone()
    n0 = tk.ops.launches
    sk, st = tk.learn(tk.buf), tt.learn(tt.buf)
    assert tk.ops.launches - n0 == 4                                    # gae, gradient, reduction, Adam (DESIGN.md)
    assert abs(sk["policy_loss"] - st["policy_loss"]) <= 1e-5 * max(1.0, abs(st["policy_loss"]))
    g = tt.policy.flat.grad.detach()
    big = g.abs() > 1e-3 * g.abs().max()
    assert torch.allclose(tk.policy.flat.detach()[big], tt.policy.flat.detach()[big], atol=1e-6)
    head = slice(tk.policy.n_params - 65, None)                         # the value head gets no gradient
    assert torch.equal(tk.policy.flat.detach()[head], p0[head]) and torch.equal(tk.ops.grad[head], torch.zeros(65, device="cuda"))


@pytest.mark.parametrize("algo", ["PG", "IMPALA"])
def test_short_run_on_the_synthetic_env_raises_reward(algo):
    from rl4rs_b200.trainer import get_rl_model
    from test_gpu_trainer import _env
    env = _env(False, B=256)
    tr = get_rl_model(algo, {"lr": 3e-3, "vtrace_drop_last_ts": False}, env=env, seed=1)
    assert tr.use_kernels
    r = [tr.train()["episode_reward_mean"] for _ in range(16)]
    assert all(math.isfinite(x) for x in r)
    assert np.mean(r[-4:]) > np.mean(r[:3]), r
