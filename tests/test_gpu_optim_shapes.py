"""GPU: every optimiser entry point against the float64 rules of tests/optim_ref64.py, tensor by tensor, from carried
moments, and the clipped PPO / A2C steps bit-reproducible.

Every case starts from m and v carried from earlier random gradients (optim_ref64.carried: magnitudes over six decades,
exact zeros, elements with sqrt(v_hat) near eps) at steps 1, 2, 10 and 10^4.  params, m, v and the target are compared
with the bounds derived in optim_ref64's docstring (relative to |b m0| + |(1 - b) g| for the moments, to the step plus
one ulp of p for the parameters), and every buffer the kernel writes is padded on both sides with a NaN sentinel that must
come back unchanged.  Each comparison is recorded as an `optim ...` row of the session's margin table.

Measured on an H100 80GB HBM3 at a 700 W power limit, worst err/bound over the whole grid (params / m / v / target):
r4_adam_step 0.50 / 0.48 / 0.50, r4_ddpg_apply 0.50 / 0.48 / 0.49 / 0.66, r4_rainbow_apply 0.50 / 0.27 / 0.25,
r4_batchrl_apply 0.50 / 0.32 / 0.31, r4_cqlc_epoch 0.49 / 0.32 / 0.31 / 0.65, r4_bcqc_epoch 0.50 / 0.32 / 0.31 / 0.66.  A
parameter at 0.50 is the final rounding of p - step (half an ulp of a bound of one).  The epoch split, the copy schedule,
copy_target, actor_step 0 and the clipped PPO / A2C reruns are bit-exact.  Arithmetic mutants of the kernels each failed
these tests: l2 on the biases (test_ddpg_apply, err/bound up to 1.6e6), the actor and critic learning rates swapped
(test_ddpg_apply, 3.8e4), tau and 1 - tau swapped in k_cqlc_adam (every test_conti_epoch_one_group_at_a_time case,
1.1e9), the target copy one float short (test_batchrl_apply BCQ and CQL), step - 1 in adam_update's bias correction
(every adam_step, ddpg, rainbow and batchrl_apply case) and grad_scale dropped from the clip's norm (test_adam_step at
grad_scale 0.5, 5.4e5).
"""
import ctypes as C
import math

import numpy as np
import pytest

import golden_util
import learner_ref64 as R
import optim_ref64 as O

pytestmark = pytest.mark.gpu

STEPS = (1, 2, 10, 10000)
PAD = 64


def _lib():
    from rl4rs_b200 import _capi
    return _capi.load_library()


def _ok(rc, what):
    if rc != 0:
        raise AssertionError("%s failed (%d): %s" % (what, rc, (_lib().r4_last_error(None) or b"?").decode()))


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Padded(object):
    """A float32 device buffer of n elements between two PAD-element NaN sentinels."""

    def __init__(self, x):
        import torch
        x = np.asarray(x, dtype=np.float32).reshape(-1)
        self.n = x.size
        self.full = torch.full((self.n + 2 * PAD,), float("nan"), dtype=torch.float32, device="cuda")
        self.full[PAD:PAD + self.n] = torch.from_numpy(x).cuda()
        self.t = self.full[PAD:PAD + self.n]

    @property
    def ptr(self):
        return C.c_void_p(self.full.data_ptr() + 4 * PAD)

    def host(self):
        return self.t.double().cpu().numpy()

    def sentinel_ok(self):
        import torch
        return bool(torch.isnan(self.full[:PAD]).all()) and bool(torch.isnan(self.full[PAD + self.n:]).all())


def _cmp(what, got, ref, bound):
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    err = np.abs(got - ref)
    bound = np.broadcast_to(np.asarray(bound, dtype=np.float64), err.shape)
    golden_util.record_margin("optim " + what, err, bound, ref)
    q = float((err / bound).max()) if err.size else 0.0
    assert q <= 1, "%s: err/bound %.3g" % (what, q)
    return q


def _check_step(what, st, p, m, v, lo=0, hi=None):
    """params, m and v [lo, hi) of the kernel against a Step over the same range."""
    sl = slice(lo, hi)
    _cmp(what + " p", p.host()[sl], st.p, st.bp)
    _cmp(what + " m", m.host()[sl], st.m, st.bm)
    _cmp(what + " v", v.host()[sl], st.v, st.bv)


def _state(n, seed, scale=0.1):
    """float32 (params, grad, m, v): params of either sign at `scale`, the biases included."""
    g, m, v = O.carried(n, seed)
    p = (np.random.RandomState(seed + 1).randn(n) * scale).astype(np.float32)
    return p, g, m, v


# ---- r4_adam_step: k_adam with the global-norm clip ---------------------------------------------------------------------
def _adam_sizes():
    lib = _lib()
    return (1, 255, 256, 257, lib.r4_policy_num_params(284), lib.r4_gauss_num_params(32))


@pytest.mark.parametrize("grad_scale", [1.0, 0.5])
@pytest.mark.parametrize("which", range(6))
def test_adam_step(which, grad_scale):
    """r4_adam_step over n at and around one 256-thread block and at the policy and Gaussian sizes; clip off, engaged
    (half the scaled norm) and set above the norm (twice it)."""
    n = _adam_sizes()[which]
    lib = _lib()
    for ci, clip_kind in enumerate(("off", "on", "above")):
        for step in STEPS:
            p0, g, m0, v0 = _state(n, 1000 * which + 10 * step + ci)
            if n == 1:
                g[0] = np.float32(0.3)
            norm = math.sqrt(float((g.astype(np.float64) ** 2).sum())) * O.f32(grad_scale)
            clip = {"off": 0.0, "on": 0.5 * norm, "above": 2.0 * norm}[clip_kind]
            P, G, M, V, N = Padded(p0), Padded(g), Padded(m0), Padded(v0), Padded(np.zeros(1))
            _ok(lib.r4_adam_step(P.ptr, G.ptr, M.ptr, V.ptr, n, step, 1e-3, 0.9, 0.999, 1e-8, grad_scale, clip, N.ptr,
                                 _stream()), "r4_adam_step")
            geff, c, on = O.global_clip(g, grad_scale, clip)
            assert on == (clip_kind == "on")
            rel_g = 2 * O.U + (O.sumsq_rel(n, 1024) if on else 0.0)
            st = O.adam(p0, geff, m0, v0, step, 1e-3, rel_g=rel_g)
            _check_step("adam_step n%d s%d %s gs%g" % (n, step, clip_kind, grad_scale), st, P, M, V)
            assert all(b.sentinel_ok() for b in (P, G, M, V, N))
            assert np.array_equal(G.host(), g.astype(np.float64))


# ---- r4_ddpg_apply ------------------------------------------------------------------------------------------------------
DDPG_CASES = ((1, 0, 0.005), (2, 1, 1.0), (10, 0, 1.0), (10000, 4999, 0.005))     # (critic_step, actor_step, tau)


@pytest.mark.parametrize("twin", [0, 1])
@pytest.mark.parametrize("D", [2, 32])
def test_ddpg_apply(D, twin):
    """Both ends of action_dim, with and without the twin critic: l2 = 1e-2 on kernels of |p| ~ 0.1 (a term far above the
    bound, so l2 on a bias would show), actor_lr 1e-3 and critic_lr 3e-4, actor_step 0 (the actor's params, m and v
    bit-identical, its target still moving) and > 0, tau 0.005 and 1, grad_scale 0.5."""
    lib = _lib()
    n, na, kern = O.ddpg_layout(D, twin)
    assert lib.r4_ddpg_num_params(D, twin) == n
    for critic_step, actor_step, tau in DDPG_CASES:
        p0, g, m0, v0 = _state(n, 7 * D + twin + critic_step)
        t0 = (p0 + 0.01 * np.random.RandomState(critic_step).randn(n)).astype(np.float32)
        P, T, G, M, V = Padded(p0), Padded(t0), Padded(g), Padded(m0), Padded(v0)
        _ok(lib.r4_ddpg_apply(P.ptr, T.ptr, G.ptr, M.ptr, V.ptr, D, twin, actor_step, critic_step, 1e-3, 3e-4, 1e-2, tau,
                              0.5, _stream()), "r4_ddpg_apply")
        st, _ = O.ddpg_apply(p0, t0, g, m0, v0, D, twin, actor_step, critic_step, 1e-3, 3e-4, 1e-2, tau, 0.5)
        what = "ddpg_apply D%d twin%d s%d a%d tau%g" % (D, twin, critic_step, actor_step, tau)
        if actor_step == 0:
            assert np.array_equal(P.host()[:na], p0[:na]) and np.array_equal(M.host()[:na], m0[:na])
            assert np.array_equal(V.host()[:na], v0[:na])
        else:
            _check_step(what + " actor", _sub(st, 0, na), P, M, V, 0, na)
        _check_step(what + " critic", _sub(st, na, n), P, M, V, na, n)
        tgt, bt = O.soft_target(P.host(), t0, tau)
        if tau == 1.0:
            assert np.array_equal(T.host(), P.host())
        else:
            _cmp(what + " target", T.host(), tgt, bt)
        assert all(b.sentinel_ok() for b in (P, T, G, M, V))


def _sub(st, lo, hi):
    return O.Step(*(getattr(st, k)[lo:hi] for k in ("p", "m", "v", "bp", "bm", "bv")))


# ---- r4_rainbow_apply ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("A,Z", [(2, 2), (284, 8), (512, 8), (128, 32)])
def test_rainbow_apply(A, Z):
    """From (2, 2) to A Z = MAXAZ (aw2 of 128 x 4096 over 32 CTAs that each sum its norm): a clip between two tensor norms,
    so it engages on some tensors only; copy_target 0 (target bit-identical) and 1 (target = params bit for bit)."""
    import torch
    from rl4rs_b200.policy import DistributionalQNetwork
    lib = _lib()
    slices = DistributionalQNetwork(A, torch.device("cpu"), seed=0, num_atoms=Z).slices
    n = slices[-1][1]
    assert lib.r4_rainbow_num_params(A, Z) == n
    for step in STEPS:
        p0, g, m0, v0 = _state(n, A * Z + step)
        norms = sorted(math.sqrt(float((g[lo:hi].astype(np.float64) ** 2).sum())) for lo, hi in slices)
        gaps = [(norms[k + 1] / norms[k], k) for k in range(len(norms) - 1) if norms[k] > 0]
        r, k = max(gaps)
        assert r > 1.01
        clip = math.sqrt(norms[k] * norms[k + 1])
        copy = int(step in (2, 10000))
        t0 = (p0 + 0.01).astype(np.float32)
        P, T, G, M, V = Padded(p0), Padded(t0), Padded(g), Padded(m0), Padded(v0)
        _ok(lib.r4_rainbow_apply(P.ptr, T.ptr, G.ptr, M.ptr, V.ptr, A, Z, step, 5e-4, 1e-8, clip, copy, _stream()),
            "r4_rainbow_apply")
        geff, which = O.clip_per_tensor(g, slices, clip)
        assert 0 < sum(on for _, _, on in which) < len(which)
        for (lo, hi, on), name in zip(which, ("w1", "b1", "w2", "b2", "aw1", "ab1", "aw2", "ab2", "sw1", "sb1", "sw2", "sb2")):
            rel_g = 2 * O.U + (O.sumsq_rel(hi - lo, 256) if on else 0.0)
            st = O.adam(p0[lo:hi], geff[lo:hi], m0[lo:hi], v0[lo:hi], step, 5e-4, rel_g=rel_g)
            _check_step("rainbow_apply A%d Z%d s%d %s" % (A, Z, step, name), st, P, M, V, lo, hi)
        assert np.array_equal(T.host(), P.host() if copy else t0.astype(np.float64))
        assert all(b.sentinel_ok() for b in (P, T, G, M, V))


# ---- r4_batchrl_apply ---------------------------------------------------------------------------------------------------
def _max_k(A):
    """The largest obs_dim the batch-RL kernels take at action_size A."""
    lib = _lib()
    lo, hi = 11, 4096
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if lib.r4_batchrl_num_params(0, mid, A) > 0 else (lo, mid - 1)
    return lo


def _bq_shapes():
    out = []
    for A in (2, 284, 512):
        for K in sorted({11, 266, 3082, _max_k(A)}):
            if K <= _max_k(A):
                out.append((K, A))
    return out


@pytest.mark.parametrize("algo", ["BC", "BCQ", "CQL"])
def test_batchrl_apply(algo):
    """BC / BCQ / CQL at obs_dim 11, 266, 3082 and the largest the shared planes take, action_size 2, 284 and 512.  With
    copy_target, target[:ntgt] equals params bit for bit, target_size is ntgt, and nothing past ntgt is written."""
    from rl4rs_b200.batchrl import ALGOS
    lib = _lib()
    k = ALGOS[algo]
    for K, A in _bq_shapes():
        n, ntgt = O.bq_layout(algo, K, A)
        assert lib.r4_batchrl_num_params(k, K, A) == n and lib.r4_batchrl_target_size(k, K, A) == ntgt
        for step in STEPS:
            p0, g, m0, v0 = _state(n, K + A + step)
            copy = int(step in (2, 10000))
            t0 = (p0[:ntgt] + 0.01).astype(np.float32)
            P, T, G, M, V = Padded(p0), Padded(t0), Padded(g), Padded(m0), Padded(v0)
            _ok(lib.r4_batchrl_apply(k, K, A, P.ptr, T.ptr, G.ptr, M.ptr, V.ptr, step, 1e-3, 1e-8, copy, _stream()),
                "r4_batchrl_apply")
            st, _ = O.bq_apply(p0, t0, g, m0, v0, ntgt, step, 1e-3, 1e-8, copy)
            _check_step("batchrl_apply %s K%d A%d s%d" % (algo, K, A, step), st, P, M, V)
            assert np.array_equal(T.host(), P.host()[:ntgt] if copy else t0.astype(np.float64))
            assert all(b.sentinel_ok() for b in (P, T, G, M, V))


# ---- r4_batchrl_epoch: the copy schedule and the split into single steps --------------------------------------------------
@pytest.mark.parametrize("algo", ["BC", "BCQ", "CQL"])
def test_batchrl_epoch_copies_on_schedule_and_splits_bitwise(algo):
    """step0 = 13 and a target interval of 3 over 7 minibatches (plus a partial one, dropped): the epoch equals, bit for
    bit, seven single-minibatch epochs with step0 advanced, and seven r4_batchrl_grad + r4_batchrl_apply pairs that copy
    the target exactly after the steps with (step - 1) % 3 == 0."""
    import torch
    from rl4rs_b200 import _capi
    from rl4rs_b200.batchrl import ALGOS, BatchRLDataPtrs
    lib = _lib()
    k = ALGOS[algo]
    K, A, mb, steps, step0, interval = 266, 284, 32, 7, 13, 3
    dev = torch.device("cuda")
    net = R.bq_net(algo, K, A, dev)
    data = R.bq_data(K, A, steps * mb + 5, dev, seed=5)
    hp = R.bq_hyper(algo)
    hc = _capi.BatchRLHyper(*(hp[f] for f in ("gamma", "beta", "alpha", "log_flex", "reward_mean", "reward_den")))
    tables = BatchRLDataPtrs(net)
    d = tables.data(data)
    perm = torch.randperm(data.n, generator=torch.Generator(device="cuda").manual_seed(3), device=dev)[:steps * mb + 5]
    perm = perm.contiguous()
    n = net.n_params
    _, _, m0, v0 = _state(n, 17)
    scratch_n = lib.r4_batchrl_scratch_size(k, K, A, mb)

    def fresh():
        tgt = net.target.clone() if net.n_target else torch.zeros(1, device=dev)
        return (net.flat.detach().clone(), tgt, torch.from_numpy(m0).to(dev), torch.from_numpy(v0).to(dev),
                torch.zeros(scratch_n, device=dev))

    def epoch(s, p, pm, st0, stats):
        prm, tgt, m, v, scr = s
        return lib.r4_batchrl_epoch(k, K, A, _ptr(prm), _ptr(tgt), _ptr(m), _ptr(v), C.byref(d), C.byref(hc), _ptr(pm),
                                    pm.numel(), mb, st0, 1e-3, 1e-8, interval, _ptr(scr), _ptr(stats), _stream())

    a = fresh()
    sa = torch.zeros(steps * 3, device=dev)
    assert epoch(a, None, perm, step0, sa) == steps
    b = fresh()
    sb = torch.zeros(steps * 3, device=dev)
    for j in range(steps):
        assert epoch(b, None, perm[j * mb:(j + 1) * mb].contiguous(), step0 + j, sb[3 * j:3 * j + 3]) == 1
    c = fresh()
    prm, tgt, m, v, scr = c
    grad = torch.zeros(n, device=dev)
    copies = []
    for j in range(steps):
        step = step0 + j + 1
        copy = int(net.n_target > 0 and (step - 1) % interval == 0)
        copies.append(copy)
        _ok(lib.r4_batchrl_grad(k, K, A, _ptr(prm), _ptr(tgt), C.byref(d), C.byref(hc), _ptr(perm[j * mb:(j + 1) * mb].contiguous()),
                                mb, _ptr(scr), _ptr(grad), None, _stream()), "r4_batchrl_grad")
        _ok(lib.r4_batchrl_apply(k, K, A, _ptr(prm), _ptr(tgt), _ptr(grad), _ptr(m), _ptr(v), step, 1e-3, 1e-8, copy,
                                 _stream()), "r4_batchrl_apply")
    assert sum(copies) == (2 if net.n_target else 0)        # steps 16 and 19
    for x in (b, c):
        for u, w in zip(a[:4], x[:4]):
            assert torch.equal(u, w), algo
    assert torch.equal(sa, sb)
    assert float((a[0] - net.flat.detach()).abs().max()) > 1e-4
    if net.n_target:
        assert not torch.equal(a[1], net.target)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


# ---- r4_cqlc_epoch / r4_bcqc_epoch: one Adam group at a time -------------------------------------------------------------
def _conti_groups(algo, K, D, Lat):
    return O.cqlc_groups(K, D) if algo == "CQL-conti" else O.bcqc_groups(K, D, Lat)


@pytest.mark.parametrize("algo,active", [("CQL-conti", g) for g in ("temp", "alpha", "critic", "actor")] +
                         [("BCQ-conti", g) for g in ("imitator", "critic", "actor")])
def test_conti_epoch_one_group_at_a_time(algo, active):
    """One minibatch with every learning rate 0 but the active group's: that group's update is float64 Adam of the gradient
    r4_cqlc_grad / r4_bcqc_grad reports at the same step, from carried moments; every other group's parameters are
    bit-identical; m and v of the active group and of the groups updated before it are Adam's of that gradient; the
    target moves by tau towards the new parameters on exactly its documented range."""
    import torch
    from test_gpu_batchrl_conti import _dataset, _model
    K, D, mb, step0 = 266, 32, 64, 4
    ds = _dataset(K, D, E=40)
    m = _model(K, D, ds, algo=algo, batch_size=mb)
    lat = int(m.hp.get("latent_size", 0))
    groups = _conti_groups(algo, K, D, lat)
    n = m.net.n_params
    lr_key = dict((name, key) for name, key, _ in m.PHASES)
    for name, _, _ in m.PHASES:
        m.hp[lr_key[name]] = 1e-3 if name == active else 0.0
    tau, eps = float(m.hp["tau"]), float(m.hp["eps"])
    data = m._device_data(ds)
    perm = torch.randperm(data.n, generator=torch.Generator(device="cuda").manual_seed(1), device="cuda")[:mb].contiguous()
    _, _, mc, vc = _state(n, 23)
    with torch.no_grad():
        m.m.copy_(torch.from_numpy(mc)); m.v.copy_(torch.from_numpy(vc))
        m.net.target.add_(0.01 * torch.randn(m.net.n_target, generator=torch.Generator().manual_seed(2)).cuda())
    m.step = step0
    p0, t0 = m.net.flat.detach().double().cpu().numpy(), m.net.target.double().cpu().numpy()
    m.grad_kernels(data, perm, step=step0 + 1)
    g = m.grad.float().cpu().numpy()
    stats = torch.zeros(5, device="cuda")
    assert m._epoch_call(data, perm, stats) == 1
    torch.cuda.synchronize()
    p, t = m.net.flat.detach().double().cpu().numpy(), m.net.target.double().cpu().numpy()
    mm, vv = m.m.double().cpu().numpy(), m.v.double().cpu().numpy()
    what = "%s %s" % (algo, active)
    before = True
    for name, (lo, hi), _, _ in groups:
        st = O.adam(p0[lo:hi].astype(np.float32), g[lo:hi], mc[lo:hi], vc[lo:hi], step0 + 1, 1e-3 if name == active else 0.0,
                    eps=eps)
        if name == active:
            _cmp(what + " p", p[lo:hi], st.p, st.bp)
        else:
            assert np.array_equal(p[lo:hi], p0[lo:hi]), (what, name)
        if before:
            _cmp("%s %s m" % (what, name), mm[lo:hi], st.m, st.bm)
            _cmp("%s %s v" % (what, name), vv[lo:hi], st.v, st.bv)
        if name == active:
            before = False
    off = O.cqlc_sizes(K, D)[2] if algo == "CQL-conti" else 0
    ntgt = m.net.n_target
    tgt, bt = O.soft_target(p[off:off + ntgt], t0, tau)
    _cmp(what + " target", t, tgt, bt)
    assert float(np.abs(t - t0).max()) > 0


# ---- the clipped PPO / A2C steps are bit-reproducible ---------------------------------------------------------------------
def test_clipped_ppo_epochs_are_bit_identical_between_runs():
    """r4_ppo_epoch and r4_gauss_ppo_epoch with the global-norm clip engaged, run twice from the same state: params, m, v
    and the statistics bit for bit (the clip's norm is summed in one CTA in a fixed order)."""
    import torch
    from rl4rs_b200.policy import GaussianPolicy, MaskedPolicy
    from rl4rs_b200.trainer import GaussKernelOps, KernelOps
    dev = torch.device("cuda")
    n, mb = 2048, 256
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(4)).to(dev)
    hp = R.PG_HP[0]
    for kind in ("mask", "gauss"):
        if kind == "mask":
            pol = MaskedPolicy(284, dev, seed=3)
            data = R.mask_batch(pol, n, 284, dev, seed=5)
            mk = lambda: KernelOps(284, dev, pol.n_params)
        else:
            pol = GaussianPolicy(32, dev, seed=3)
            data = R.gauss_batch(pol, n, 32, dev, seed=5)
            mk = lambda: GaussKernelOps(32, dev, pol.n_params)
        runs = []
        for _ in range(2):
            ops = mk()
            flat = pol.flat.detach().clone()
            assert ops.ppo_epoch(flat, data, perm, n, mb, hp, 1e-3, 1e-3) == n // mb
            torch.cuda.synchronize()
            runs.append((flat, ops.m.clone(), ops.v.clone(), ops.stats.clone(), float(ops.norm)))
        (a, ma, va, sa, na), (b, mb_, vb, sb, nb) = runs
        assert math.sqrt(na) > 2e-3, kind           # the clip (1e-3) engaged on the last minibatch at least
        assert torch.equal(a, b) and torch.equal(ma, mb_) and torch.equal(va, vb) and torch.equal(sa, sb), kind
        assert float((a - pol.flat).abs().max()) > 1e-5
