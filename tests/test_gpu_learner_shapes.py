"""GPU: every learner kernel against the float64 reference of tests/learner_ref64.py, tensor by tensor, at the shapes the
C-ABI accepts and at batch sizes that cut the kernels' tiles and chunks (TS = 8 rows per CTA, WK = 32, SNT = 1024,
Gauss CH = 2048, BatchRL EGCH = 2048 ids = 205 samples), plus the replay kernels against a NumPy float64 oracle and the
rejection of the first shape outside each range.

Rows: a candidate pool is drawn, the reference runs over it, and only rows whose every discrete decision is clear of its
switch point (learner_ref64.TIE, RELU_TIE) go to the kernel; fewer than MAX_DROP of the pool may be dropped.
Bound: max |g - ref| <= tol * max |ref| for every tensor of the flat layout; per-sample rows within tol of max(1, |ref|);
statistics within 1e-4 of max(1, |ref|); act outputs within tol of the largest |ref| and the actions equal where the
reference's margin is clear.  Every comparison is recorded as a `learner ...` row of the session's margin table.

Measured on an H100 80GB HBM3 (SM clock up to 1980 MHz), worst err/bound over the whole grid at the bounds below:
gradients of tensors with more than SMALL elements (GRAD_TOL) policy PPO 0.09 / A2C 0.08, gauss PPO 0.25 / A2C 0.11,
DDPG 0.10, TD3 0.12, rainbow 0.26, BC 0.03, BCQ 0.11, CQL 0.01; tensors of at most SMALL elements (SMALL_TOL) 0.19
(rainbow sb2), 0.02 elsewhere; per-sample rows (1e-4) DDPG / TD3 0.01, rainbow 0.08; statistics (1e-4) at most 0.02;
act outputs (1e-4) at most 0.04.  A 1 % error on the largest element of any tensor, a bias included, is 0.01 / tol times
its bound: 10x for the small tensors, 100x (batch RL) to 1000x (policy, DDPG / TD3) for the others.
"""
import ctypes as C
import math

import numpy as np
import pytest

import golden_util
import learner_ref64 as R

pytestmark = pytest.mark.gpu

NS = (1, 7, 9, 33, 1025)
TOL = 1e-4
# the per-tensor gradient bound of each family: 1e-4 where the first H100 run left less than ten-fold headroom, tighter
# where it left more (worst err/bound at 1e-4 over the grid: policy 0.031, gauss 0.048, ddpg 0.013, rainbow 0.052,
# batchrl 0.137)
GRAD_TOL = {"policy": 1e-5, "gauss": 2e-5, "ddpg": 1e-5, "rainbow": 2e-5, "batchrl": 1e-4}
# Tensors of at most SMALL elements (value and output biases, RAINBOW's score bias) are each a sum over the batch of
# per-row terms that largely cancel, so their fp32 rounding is set by the terms, not by the sum: RAINBOW's sb2 at
# (A, Z) = (2, 2), n = 9 sums terms of ~1e-1 to 3.4e-4 and carries 6.6e-8 of rounding, 1.9e-4 of its max |ref|.  They are
# held to SMALL_TOL, which still puts a 1 % error at 10x the bound; every larger tensor has stayed within 0.26 of GRAD_TOL.
SMALL, SMALL_TOL = 32, 1e-3
# the tie filter may drop at most this share of a pool.  Measured over 1143-row pools on the CPU: at most 2.4 % for DDPG /
# TD3 and 1.3 % for BC / CQL; BCQ at K = 4096 drops 4.1 % (2.5 % at its argmax, imitator-threshold and huber decisions,
# 1.6 % at relu kinks), the largest of the grid, so the cap leaves room for a pool's sampling spread above that
MAX_DROP = 0.08
ACT_CLEAR = 0.9       # the act checks run over the whole pool; at least this share of it must have a clear argmax


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _lib():
    from rl4rs_b200 import _capi
    return _capi.load_library()


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ok(rc, what):
    if rc != 0:
        raise AssertionError("%s failed (%d): %s" % (what, rc, (_lib().r4_last_error(None) or b"?").decode()))


def _grid(shapes, default, extra=()):
    """The full shape grid at n = 9 and 1025, every n (and `extra`) at the default shape."""
    out = [(s, n) for s in shapes for n in (9, 1025)]
    return out + [(default, n) for n in NS + tuple(extra) if (default, n) not in out]


def _pool(n):
    """Candidate rows for n clear ones: at least 256, so the dropped share is a measured rate and not a handful of rows."""
    return max(256, n + n // 10 + 16)


def _select(ref, n, what):
    """The first n clear rows of a reference over the pool; asserts the filter dropped fewer than MAX_DROP."""
    import torch
    clear = ref.clear()
    drop = 1.0 - float(clear.double().mean())
    assert drop < MAX_DROP, "%s: the tie filter dropped %.1f %% of the pool" % (what, 100 * drop)
    sel = torch.nonzero(clear).reshape(-1)[:n]
    assert sel.numel() == n, (what, sel.numel(), n)
    return sel


def _cmp(what, got, ref, bound):
    import torch
    if torch.is_tensor(bound):
        bound = bound.detach().double().cpu().numpy().reshape(-1)
    got = got.detach().double().cpu().numpy().reshape(-1)
    ref = ref.detach().double().cpu().numpy().reshape(-1)
    err = np.abs(got - ref)
    bound = np.broadcast_to(np.asarray(bound, dtype=np.float64), err.shape)
    golden_util.record_margin("learner " + what, err, bound, ref)
    return float((err / bound).max()) if err.size else 0.0


def _check_grad(what, grad, ref, twin):
    worst = []
    for name, sl in R.tensors(twin):
        r = ref[sl]
        tol = GRAD_TOL[what.split()[0]] if r.numel() > SMALL else SMALL_TOL
        scale = max(float(r.abs().max()), 1e-30)
        q = _cmp("%s %s" % (what, name), grad[sl], r, tol * scale)
        if q > 1:
            worst.append((name, tol, q))
    assert not worst, "%s: tensors outside tol * their max |ref| (name, tol, err/bound): %s" % (what, worst)


def _check_rows(what, got, ref, tol=TOL):
    q = _cmp(what + " rows", got, ref, tol * ref.detach().abs().clamp_min(1.0))
    assert q <= 1, (what, q)


def _check_actions(what, got, ref_pick, margin, allowed=None):
    """The kernel's actions equal the reference's argmax on every row whose margin is clear, and those rows are at least
    ACT_CLEAR of the batch (so the comparison cannot go empty); with `allowed`, every action is an allowed one."""
    import torch
    clear = margin > R.TIE
    assert float(clear.double().mean()) >= ACT_CLEAR, "%s: only %d of %d rows have a clear argmax" % (
        what, int(clear.sum()), clear.numel())
    assert torch.equal(got.long()[clear], ref_pick.argmax(1)[clear]), what
    if allowed is not None:
        rows = allowed.any(1)
        assert bool(allowed[torch.arange(len(got), device=got.device), got.long()][rows].all()), what


def _check_stats(what, got, ref, keep=None):
    import torch
    keep = list(range(len(ref))) if keep is None else keep
    g, r = got[keep], ref[keep]
    q = _cmp(what + " stats", g, r, 1e-4 * r.detach().abs().clamp_min(1.0))
    assert q <= 1, (what, g.tolist(), r.tolist())


# ---- mask policy (PPO / A2C) --------------------------------------------------------------------------------------------
def _pg_check(what, ops, flat, mode, data, n, ref, twin):
    inv_n = 1.0 / n if mode == 0 else 1.0
    ops.stats.zero_()
    ops.policy_grad(mode, flat, data, None, 0, n, R.PG_HP[mode], inv_n, inv_n)
    _check_grad(what, ops.grad, ref.grad, twin)
    _check_stats(what, ops.stats.double(), ref.stats * inv_n, keep=[0, 1, 2, 3, 4] if mode == 0 else [0, 1, 3, 4])


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("A,n", _grid((2, 31, 284, 512), 284))
def test_policy_grad_and_act(A, n, mode):
    import torch
    from rl4rs_b200.policy import MaskedPolicy
    from rl4rs_b200.trainer import KernelOps
    dev = torch.device("cuda")
    pol = MaskedPolicy(A, dev, seed=3)
    with torch.no_grad():
        pol.flat.add_(0.05 * torch.randn(pol.n_params, generator=torch.Generator().manual_seed(4)).to(dev))
    what = "policy %s A%d n%d" % ("PPO" if mode == 0 else "A2C", A, n)
    pool = R.mask_batch(pol, _pool(n), A, dev, seed=A + n)
    inv = 1.0 / n if mode == 0 else 1.0
    sel = _select(R.policy_grad(pol, pol.flat, mode, *pool, R.PG_HP[mode], inv), n, what)
    data = tuple(x[sel].contiguous() for x in pool)
    ref = R.policy_grad(pol, pol.flat, mode, *data, R.PG_HP[mode], inv)
    ops = KernelOps(A, dev, pol.n_params)
    _pg_check(what, ops, pol.flat, mode, data, n, ref, pol)
    if mode == 1:
        return
    obs, mask = pool[0], pool[1]                   # act over the whole pool
    P = obs.shape[0]
    a = torch.empty(P, dtype=torch.int32, device=dev)
    lp, v, lg = torch.empty(P, device=dev), torch.empty(P, device=dev), torch.empty(P, A, device=dev)
    ops.act(pol.flat, obs, mask, False, 1, a, lp, v, lg)
    rl, rv, rlp, ra, margin = R.policy_act(pol, pol.flat, obs, mask)
    ok = mask.bool()
    scale = float(rl[ok].abs().max())
    assert _cmp(what + " act logits", lg[ok], rl[ok], TOL * scale) <= 1 and bool((lg[~ok] < -1e30).all())
    assert _cmp(what + " act value", v, rv, TOL * max(1.0, float(rv.abs().max()))) <= 1
    clear = margin > R.TIE                          # logp is of the chosen action: compare it where the choice is clear
    assert _cmp(what + " act logp", lp[clear], rlp[clear], TOL * rlp[clear].abs().clamp_min(1.0)) <= 1
    _check_actions(what + " act", a, rl, margin, ok)


# ---- Gaussian policy (PPO_conti / A2C_conti) ------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("D,n", _grid((2, 32, 64), 32, extra=(2048, 2049)))
def test_gauss_grad_and_act(D, n, mode):
    import torch
    from rl4rs_b200.policy import GaussianPolicy
    from rl4rs_b200.trainer import GaussKernelOps
    dev = torch.device("cuda")
    pol = GaussianPolicy(D, dev, seed=3)
    with torch.no_grad():
        pol.flat.add_(0.02 * torch.randn(pol.n_params, generator=torch.Generator().manual_seed(3)).to(dev))
    what = "gauss %s D%d n%d" % ("PPO" if mode == 0 else "A2C", D, n)
    pool = R.gauss_batch(pol, _pool(n), D, dev, seed=D + n)
    inv = 1.0 / n if mode == 0 else 1.0
    sel = _select(R.gauss_grad(pol, pol.flat, mode, *pool, R.PG_HP[mode], inv), n, what)
    data = tuple(x[sel].contiguous() for x in pool)
    ref = R.gauss_grad(pol, pol.flat, mode, *data, R.PG_HP[mode], inv)
    ops = GaussKernelOps(D, dev, pol.n_params)
    kdata = data if mode == 0 else (data[0], data[1], None, None, None, data[5], data[6])
    _pg_check(what, ops, pol.flat, mode, kdata, n, ref, pol)
    if mode == 1:
        return
    e = lambda *s: torch.empty(*s, device=dev)
    a, ea, lp, v, d = e(n, D), e(n, D), e(n), e(n), e(n, 2 * D)
    ops.act(pol.flat, data[0], False, 1, a, ea, lp, v, d)
    rd, rv = R.gauss_act(pol, pol.flat, data[0])
    assert _cmp(what + " act dist", d, rd, TOL * float(rd.abs().max())) <= 1
    assert _cmp(what + " act value", v, rv, TOL * max(1.0, float(rv.abs().max()))) <= 1
    assert torch.equal(a, d[:, :D]) and torch.equal(ea, a.clamp(-1.0, 1.0))


# ---- DDPG / TD3 ---------------------------------------------------------------------------------------------------
# (algo, importance weights, target smoothing): the whole grid with DDPG's and TD3's defaults (prioritized replay for DDPG,
# smoothing for TD3), and every other combination at the default shape
DDPG_CASES = [(s, n, c) for s, n in _grid((2, 7, 32), 32) for c in (("DDPG", True, False), ("TD3", False, True))] + \
    [(32, n, c) for n in (9, 1025) for c in (("DDPG", False, False), ("DDPG", True, True), ("TD3", False, False),
                                           ("TD3", True, False), ("TD3", True, True))]


@pytest.mark.parametrize("D,n,case", DDPG_CASES)
def test_ddpg_grad_and_act(D, n, case):
    import torch
    algo, with_w, with_noise = case
    from rl4rs_b200.policy import DeterministicActorCritic
    dev = torch.device("cuda")
    twin = algo == "TD3"
    pol = DeterministicActorCritic(D, dev, seed=5, twin=twin)
    g = torch.Generator().manual_seed(D + n)
    with torch.no_grad():
        pol.flat.add_(0.01 * torch.randn(pol.n_params, generator=g).to(dev))
        pol.target.copy_(pol.flat.detach() + 0.01 * torch.randn(pol.n_params, generator=g).to(dev))
    P = _pool(n)
    obs, nobs = torch.randn(P, 256, generator=g).to(dev), torch.randn(P, 256, generator=g).to(dev)
    act = (torch.rand(P, D, generator=g) * 2 - 1).to(dev)
    rew = torch.randn(P, generator=g).to(dev)
    done = (torch.rand(P, generator=g) < 0.3).to(torch.uint8).to(dev)
    w = (torch.rand(P, generator=g) + 0.5).to(dev) if with_w else None
    noise = torch.randn(P, D, generator=g).to(dev).contiguous() if with_noise else None
    gamma, tn, nc = 0.99, 0.2, 0.5
    what = "ddpg %s%s%s D%d n%d" % (algo, " weights" if with_w else "", " smooth" if with_noise else "", D, n)
    pool_ref = R.ddpg_grad(pol, pol.flat, pol.target, obs, act, rew, nobs, done, w, noise, gamma, tn, nc, 1.0)
    sel = _select(pool_ref, n, what)
    pick = lambda x: None if x is None else x[sel].contiguous()
    ref = R.ddpg_grad(pol, pol.flat, pol.target, *map(pick, (obs, act, rew, nobs, done, w, noise)), gamma, tn, nc, 1.0 / n)
    lib = _lib()
    grad = torch.zeros(pol.n_params, device=dev)
    td, stats = torch.zeros(n, device=dev), torch.zeros(3, device=dev)
    scratch = torch.zeros(lib.r4_ddpg_scratch_size(D, int(twin), n), device=dev)
    w_n, noise_n = pick(w), pick(noise)          # held here: the kernel reads them after this line
    _ok(lib.r4_ddpg_grad(_p(pol.flat), _p(pol.target), D, int(twin), _p(obs), _p(act), _p(rew), _p(nobs), _p(done),
                         _p(sel), _p(w_n), _p(noise_n), n, gamma, tn, nc, 1.0 / n,
                         _p(scratch), _p(grad), _p(td), _p(stats), _stream()), "r4_ddpg_grad")
    _check_grad(what, grad, ref.grad, pol)
    _check_rows(what, td, ref.rows)
    _check_stats(what, stats.double(), ref.stats)
    a = torch.empty(n, D, device=dev)
    x = obs[sel].contiguous()
    _ok(lib.r4_ddpg_act(_p(pol.flat), _p(x), n, D, 0, 0, 0, None, None, 0.0, 0.0, 0.0, _p(a), _stream()), "r4_ddpg_act")
    ra = R.ddpg_act(pol, pol.flat, obs[sel])
    assert _cmp(what + " act", a, ra, TOL) <= 1


# ---- RAINBOW ------------------------------------------------------------------------------------------------------
RB_SHAPES = ((2, 2), (284, 8), (512, 8), (128, 32), (2, 32))


@pytest.mark.parametrize("vrange", [(0.0, 1000.0), (-10.0, 10.0)])
@pytest.mark.parametrize("AZ,n", _grid(RB_SHAPES, (284, 8)))
def test_rainbow_grad_and_act(AZ, n, vrange):
    import torch
    from rl4rs_b200.policy import DistributionalQNetwork
    dev = torch.device("cuda")
    A, Z = AZ
    v_min, v_max = vrange
    pol = DistributionalQNetwork(A, dev, seed=2, num_atoms=Z, v_min=v_min, v_max=v_max)
    g = torch.Generator().manual_seed(A * Z + n)
    with torch.no_grad():
        pol.target.add_(0.3 * torch.randn(pol.n_params, generator=g).to(dev))
    P = _pool(n)
    obs, nobs = torch.randn(P, 256, generator=g).to(dev), torch.randn(P, 256, generator=g).to(dev)
    act = torch.randint(0, A, (P,), generator=g, dtype=torch.int32).to(dev)
    rew = R.rb_rewards(P, Z, v_min, v_max, g).to(dev)
    done = (torch.arange(P) % 3 == 0).to(torch.uint8).to(dev)
    w = (torch.rand(P, generator=g) + 0.5).to(dev)
    gamma_n = 1.0 if v_min == 0.0 else 0.729
    what = "rainbow A%d Z%d v%g..%g n%d" % (A, Z, v_min, v_max, n)
    sel = _select(R.rainbow_grad(pol, pol.flat, pol.target, obs, act, rew, nobs, done, w, gamma_n, 1.0), n, what)
    pick = lambda x: x[sel].contiguous()
    ref = R.rainbow_grad(pol, pol.flat, pol.target, *map(pick, (obs, act, rew, nobs, done, w)), gamma_n, 1.0 / n)
    lib = _lib()
    grad = torch.zeros(pol.n_params, device=dev)
    td, stats = torch.zeros(n, device=dev), torch.zeros(3, device=dev)
    scratch = torch.zeros(lib.r4_rainbow_scratch_size(A, Z, n), device=dev)
    w_n = pick(w)                                # held here: the kernel reads it after this line
    _ok(lib.r4_rainbow_grad(_p(pol.flat), _p(pol.target), A, Z, v_min, v_max, _p(obs), _p(act), _p(rew), _p(nobs), _p(done),
                            _p(sel), _p(w_n), n, gamma_n, 1.0 / n, _p(scratch), _p(grad), _p(td), _p(stats), _stream()),
        "r4_rainbow_grad")
    _check_grad(what, grad, ref.grad, pol)
    _check_rows(what, td, ref.rows)
    _check_stats(what, stats.double(), ref.stats)
    a = torch.empty(P, dtype=torch.int32, device=dev)   # act over the whole pool
    q = torch.empty(P, A, device=dev)
    _ok(lib.r4_rainbow_act(_p(pol.flat), _p(obs), P, A, Z, v_min, v_max, 0, 5, 0, _p(a), _p(q), _stream()), "r4_rainbow_act")
    rq = R.rainbow_act(pol, pol.flat, obs)
    assert _cmp(what + " act q", q, rq, TOL * max(1.0, float(rq.abs().max()))) <= 1
    _check_actions(what + " act", a, rq, R.argmax_margin(rq))


# ---- BC / BCQ / CQL -----------------------------------------------------------------------------------------------
BQ_SHAPES = ((11, 2), (266, 284), (3082, 284), (4096, 284), (2998, 512), (266, 512))


@pytest.mark.parametrize("algo", ["BC", "BCQ", "CQL"])
@pytest.mark.parametrize("KA,n", _grid(BQ_SHAPES, (266, 284), extra=(205,)))
def test_batchrl_grad_and_act(KA, n, algo):
    import torch
    from rl4rs_b200 import _capi
    from rl4rs_b200.batchrl import ALGOS, BatchRLDataPtrs
    dev = torch.device("cuda")
    K, A = KA
    net = R.bq_net(algo, K, A, dev)
    data = R.bq_data(K, A, _pool(n), dev, seed=K + A + n)
    hp = R.bq_hyper(algo)
    what = "batchrl %s K%d A%d n%d" % (algo, K, A, n)
    pool = torch.randperm(data.n, generator=torch.Generator(device="cuda").manual_seed(n), device=dev)[:_pool(n)]
    sel = pool[_select(R.batchrl_grad(net, net.flat, net.target, *data.batch(pool), hp), n, what)].contiguous()
    ref = R.batchrl_grad(net, net.flat, net.target, *data.batch(sel), hp)
    lib = _lib()
    k = ALGOS[algo]
    grad = torch.zeros(net.n_params, device=dev)
    stats = torch.zeros(3, device=dev)
    scratch = torch.zeros(lib.r4_batchrl_scratch_size(k, K, A, n), device=dev)
    tables = BatchRLDataPtrs(net)
    hc = _capi.BatchRLHyper(*(hp[f] for f in ("gamma", "beta", "alpha", "log_flex", "reward_mean", "reward_den")))
    _ok(lib.r4_batchrl_grad(k, K, A, _p(net.flat), _p(net.target), C.byref(tables.data(data)), C.byref(hc), _p(sel), n,
                            _p(scratch), _p(grad), _p(stats), _stream()), "r4_batchrl_grad")
    _check_grad(what, grad, ref.grad, net)
    _check_stats(what, stats.double(), ref.stats)
    x = data.batch(pool)[0].contiguous()           # act over the whole pool
    P = x.shape[0]
    a = torch.empty(P, dtype=torch.int32, device=dev)
    probs, vals = torch.empty(P, A, device=dev), torch.empty(P, A, device=dev)
    raw, rp, keep, picks = R.batchrl_act(net, net.flat, x, hp["log_flex"])
    assert bool(keep.any(1).all()) and not bool(keep.all())       # the mask rules items out, and leaves some on every row
    assert bool((~keep.gather(1, rp.argmax(1, keepdim=True))).any())    # and it changes mode 0's pick on some rows
    for mode, (pick, margin) in enumerate(picks):
        _ok(lib.r4_batchrl_act(k, K, A, _p(net.flat), _p(x), 0, P, C.byref(tables.tables()), mode, hp["log_flex"], _p(a),
                               _p(probs), _p(vals), _stream()), "r4_batchrl_act")
        assert _cmp(what + " act values", vals, raw, TOL * float(raw.abs().max())) <= 1
        assert _cmp(what + " act probs", probs, rp, TOL * max(1.0, float(rp.abs().max()))) <= 1
        # mode 0 (predict_with_mask): the argmax over the items keep allows, and never an excluded item
        _check_actions("%s act mode %d" % (what, mode), a, pick, margin, keep if mode == 0 else None)


# ---- replay -------------------------------------------------------------------------------------------------------
def _np_store(ring, pos, obs, fin, act, rew, done, max_prio, alpha):
    """The NumPy oracle of r4_replay_store / r4_replay_store_nstep's slot rule: only the last C rows are written."""
    C_ = ring["reward"].shape[0]
    T, B = rew.shape
    n = T * B
    nxt = np.concatenate([obs[1:].reshape(-1, 256), fin.reshape(B, 256)])
    for r in range(max(0, n - C_), n):
        s = (pos + r) % C_
        ring["obs"][s], ring["new_obs"][s] = obs.reshape(n, 256)[r], nxt[r]
        ring["action"][s] = act.reshape(n, *ring["action"].shape[1:])[r]
        ring["reward"][s], ring["done"][s] = rew.reshape(n)[r], done.reshape(n)[r]
        ring["prio"][s] = np.float32(max_prio) ** np.float32(alpha)


def _nstep_np(obs, fin, rew, done, n_step, gamma):
    T, B = rew.shape
    nxt = np.concatenate([obs[1:], fin.reshape(1, B, 256)])
    src = np.minimum(np.arange(T) + n_step - 1, T - 1)
    R_, gj = rew.copy(), np.float32(1.0)
    for j in range(1, min(n_step, T)):
        gj = np.float32(gj * np.float32(gamma))
        R_[:T - j] = R_[:T - j] + gj * rew[j:]
    return nxt[src], R_, done[src]


@pytest.mark.parametrize("nstep", [False, True])
def test_replay_store_more_rows_than_the_ring(nstep):
    """9 x 64 rows into 500 slots in one call (only the last 500 are written), then a second call that wraps around."""
    import torch
    lib = _lib()
    dev = torch.device("cuda")
    Cap, T, B, D, alpha = 500, 9, 64, 7, 0.6
    ring_t = {"obs": torch.zeros(Cap, 256, device=dev), "new_obs": torch.zeros(Cap, 256, device=dev),
              "action": torch.zeros(Cap, dtype=torch.int32, device=dev) if nstep else torch.zeros(Cap, D, device=dev),
              "reward": torch.zeros(Cap, device=dev), "done": torch.zeros(Cap, dtype=torch.uint8, device=dev),
              "prio": torch.zeros(Cap, device=dev)}
    ring = {k: v.cpu().numpy().copy() for k, v in ring_t.items()}
    max_prio = torch.tensor([2.5], device=dev)
    rs = np.random.RandomState(0)
    pos = 0
    for call in range(2):
        obs = rs.randn(T, B, 256).astype(np.float32)
        fin = rs.randn(B, 256).astype(np.float32)
        act = rs.randint(0, 284, (T, B)).astype(np.int32) if nstep else rs.uniform(-1, 1, (T, B, D)).astype(np.float32)
        rew = rs.randn(T, B).astype(np.float32)
        done = (rs.rand(T, B) < 0.2).astype(np.uint8)
        done[-1] = 1
        tt = {k: torch.as_tensor(v).to(dev).contiguous() for k, v in (("obs", obs), ("fin", fin), ("act", act), ("rew", rew),
                                                                     ("done", done))}
        rp = [_p(ring_t[k]) for k in ("obs", "action", "reward", "new_obs", "done", "prio")]
        if nstep:
            _ok(lib.r4_replay_store_nstep(*rp, _p(max_prio), Cap, pos, alpha, 3, 0.9, _p(tt["obs"]), _p(tt["fin"]),
                                          _p(tt["act"]), _p(tt["rew"]), _p(tt["done"]), T, B, _stream()), "r4_replay_store_nstep")
            nxt, R_, dn = _nstep_np(obs, fin, rew, done, 3, 0.9)
            # the fold gives new_obs / done directly: store with those and the folded rewards
            n = T * B
            for r in range(max(0, n - Cap), n):
                s = (pos + r) % Cap
                ring["obs"][s], ring["new_obs"][s] = obs.reshape(n, 256)[r], nxt.reshape(n, 256)[r]
                ring["action"][s], ring["reward"][s], ring["done"][s] = act.reshape(n)[r], R_.reshape(n)[r], dn.reshape(n)[r]
                ring["prio"][s] = np.float32(2.5) ** np.float32(alpha)
        else:
            _ok(lib.r4_replay_store(*rp, _p(max_prio), Cap, D, pos, alpha, _p(tt["obs"]), _p(tt["fin"]), _p(tt["act"]),
                                    _p(tt["rew"]), _p(tt["done"]), T, B, _stream()), "r4_replay_store")
            _np_store(ring, pos, obs, fin, act, rew, done, 2.5, alpha)
        pos += T * B
        for k in ("obs", "new_obs", "action", "reward", "done"):
            assert np.array_equal(ring_t[k].cpu().numpy(), ring[k]), (k, call)
        np.testing.assert_allclose(ring_t["prio"].cpu().numpy(), ring["prio"], rtol=1e-6)


@pytest.mark.parametrize("size", [1, 7, 1000, 1024, 1025, 5000])
def test_replay_sample_against_exact_prefix_sums(size):
    """Priorities that are small integers or powers of two: the float64 prefix sums are exact, so the indices must match
    the oracle's exactly; the weights within 1e-6."""
    import torch
    lib = _lib()
    dev = torch.device("cuda")
    rs = np.random.RandomState(size)
    prio = rs.choice(np.array([0.25, 0.5, 1, 2, 3, 4, 7], dtype=np.float32), size)
    prio_t = torch.as_tensor(prio).to(dev)
    cum = np.cumsum(prio.astype(np.float64))
    total = cum[-1]
    beta = 0.4
    for n in (1, 1024, 1025, 3000):
        u = rs.rand(n).astype(np.float32)
        u[:min(n, 3)] = np.float32([0.0, 0.5, np.nextafter(np.float32(1), np.float32(0))])[:min(n, 3)]
        u_t = torch.as_tensor(u).to(dev)
        idx, w = torch.empty(n, dtype=torch.int64, device=dev), torch.empty(n, device=dev)
        _ok(lib.r4_replay_sample(_p(prio_t), size, n, beta, _p(u_t), _p(idx), _p(w), _stream()), "r4_replay_sample")
        ref = np.minimum(np.searchsorted(cum, u.astype(np.float64) * total, side="right"), size - 1)
        assert np.array_equal(idx.cpu().numpy(), ref), (size, n)
        p = prio.astype(np.float64) / total
        rw = (p[ref] * size) ** -beta / (p.min() * size) ** -beta
        np.testing.assert_allclose(w.cpu().numpy(), rw, rtol=1e-6)
        _ok(lib.r4_replay_sample(None, size, n, beta, _p(u_t), _p(idx), _p(w), _stream()), "r4_replay_sample")
        assert np.array_equal(idx.cpu().numpy(), np.minimum(np.floor(u.astype(np.float64) * size), size - 1).astype(np.int64))
        assert bool((w == 1).all())


def test_replay_update_priorities_later_position_wins():
    """Indices repeated more than 1024 positions apart (past one CTA's first sweep): the later position's td wins."""
    import torch
    lib = _lib()
    dev = torch.device("cuda")
    Cap, n, alpha, eps = 5000, 3000, 0.6, 1e-6
    rs = np.random.RandomState(1)
    idx = rs.randint(0, Cap, n).astype(np.int64)
    idx[2500] = idx[10]
    idx[1100] = idx[20]
    idx[2999] = idx[1100]
    td = (rs.randn(n) * 3).astype(np.float32)
    prio = torch.ones(Cap, device=dev)
    mp = torch.ones(1, device=dev)
    idx_t, td_t = torch.as_tensor(idx).to(dev), torch.as_tensor(td).to(dev)      # held: the kernel reads them later
    _ok(lib.r4_replay_update_priorities(_p(prio), _p(mp), _p(idx_t), _p(td_t), n, alpha, eps, _stream()),
        "r4_replay_update_priorities")
    ref = np.ones(Cap, np.float32)
    for i in range(n):                          # RLlib's sequential loop
        ref[idx[i]] = (np.abs(np.float64(td[i])) + np.float64(np.float32(eps))) ** alpha
    np.testing.assert_allclose(prio.cpu().numpy(), ref, rtol=1e-6)
    assert float(mp) == pytest.approx(max(1.0, float(np.abs(td).max()) + eps), rel=1e-6)


# ---- rejection on the device path -----------------------------------------------------------------------------------
def test_first_rejected_shape_launches_nothing():
    """At the first shape outside each range the *_grad and *_act entry points return R4_ERR_ARG with their message and
    leave every output as it was."""
    import torch
    from rl4rs_b200 import _capi
    lib = _lib()
    dev = torch.device("cuda")
    from rl4rs_b200.policy import BatchRLNet, DeterministicActorCritic, DistributionalQNetwork, GaussianPolicy
    # Every buffer is as large as a launch at the rejected shape would touch, so that if a range check were ever dropped
    # the test fails on its assertions instead of writing out of bounds: `out` (gradients, statistics, Q, probs) holds
    # the largest parameter vector of the rejected shapes, `big` (parameters, observations, scratch) twice that or twice
    # the largest scratch of the nearest accepted shapes, whichever is more.
    bq = lambda K, A: BatchRLNet("BCQ", K, np.ones((4, A)), [0], A, "cpu").n_params
    n_out = max(GaussianPolicy(66, "cpu").n_params, DeterministicActorCritic(33, "cpu", twin=True).n_params,
                DistributionalQNetwork(241, "cpu", num_atoms=17).n_params,
                DistributionalQNetwork(513, "cpu", num_atoms=2).n_params, bq(4097, 284), bq(2999, 512), bq(266, 513))
    n_in = 2 * max(n_out, lib.r4_gauss_scratch_size(64), lib.r4_ddpg_scratch_size(32, 1, 8),
                   lib.r4_rainbow_scratch_size(256, 16, 8), lib.r4_batchrl_scratch_size(1, 4096, 284, 8),
                   lib.r4_batchrl_scratch_size(1, 2998, 512, 8))
    big = torch.zeros(n_in, device=dev)
    out = torch.full((n_out,), 7.0, device=dev)
    i32 = torch.full((1024,), -5, dtype=torch.int32, device=dev)
    idx = torch.zeros(64, dtype=torch.int64, device=dev)
    u8 = torch.ones(1 << 20, dtype=torch.uint8, device=dev)
    s = _stream()

    def rejected(rc, name):
        torch.cuda.synchronize()
        assert rc == -1, (name, rc)
        assert (lib.r4_last_error(None) or b"").decode().startswith(name), (name, lib.r4_last_error(None))
        assert bool((out == 7.0).all()) and bool((i32 == -5).all()), name

    hp = (0.3, 1.0, 0.5, 0.2, 0.01)
    for A in (1, 513):
        rejected(lib.r4_policy_grad(0, _p(big), _p(big), _p(u8), _p(idx), _p(big), _p(big), _p(big), _p(big), _p(big), None, 8,
                                    A, *hp, 1.0, _p(big), 1, _p(out), _p(out), 1.0, s), "r4_policy_grad")
        rejected(lib.r4_policy_act(_p(big), _p(big), _p(u8), 8, A, 0, 0, 0, _p(i32), _p(out), _p(out), _p(out), s),
                 "r4_policy_act")
    for D in (3, 66, 0):
        rejected(lib.r4_gauss_grad(0, _p(big), _p(big), _p(big), _p(big), _p(big), _p(big), _p(big), _p(big), None, 8, D,
                                   *hp, 1.0, _p(big), _p(out), _p(out), 1.0, s), "r4_gauss_grad")
        rejected(lib.r4_gauss_act(_p(big), _p(big), 8, D, 0, 0, 0, _p(out), _p(out), _p(out), _p(out), None, s),
                 "r4_gauss_act")
    for D in (33, 1):
        rejected(lib.r4_ddpg_grad(_p(big), _p(big), D, 1, _p(big), _p(big), _p(big), _p(big), _p(u8), _p(idx), None, None, 8,
                                  0.99, 0.2, 0.5, 0.125, _p(big), _p(out), _p(out), _p(out), s), "r4_ddpg_grad")
        rejected(lib.r4_ddpg_act(_p(big), _p(big), 8, D, 0, 0, 0, None, None, 0.0, 0.0, 0.0, _p(out), s), "r4_ddpg_act")
    for A, Z in ((513, 2), (2, 33), (128, 33), (241, 17), (1, 8)):
        rejected(lib.r4_rainbow_grad(_p(big), _p(big), A, Z, 0.0, 10.0, _p(big), _p(i32), _p(big), _p(big), _p(u8), _p(idx),
                                     None, 8, 1.0, 0.125, _p(big), _p(out), _p(out), _p(out), s), "r4_rainbow_grad")
        rejected(lib.r4_rainbow_act(_p(big), _p(big), 8, A, Z, 0.0, 10.0, 0, 0, 0, _p(i32), _p(out), s), "r4_rainbow_act")
    d = _capi.BatchRLData(*[big.data_ptr()] * 4 + [idx.data_ptr(), u8.data_ptr(), u8.data_ptr()])
    h = _capi.BatchRLHyper(*R.BQ_HP.values())
    for K, A in ((2999, 512), (10, 284), (4097, 284), (266, 513), (266, 1)):
        for algo in (0, 1, 2):
            before = lib.r4_batchrl_launch_count()
            rejected(lib.r4_batchrl_grad(algo, K, A, _p(big), _p(big), C.byref(d), C.byref(h), _p(idx), 8, _p(big), _p(out),
                                         _p(out), s), "r4_batchrl_grad")
            rejected(lib.r4_batchrl_act(algo, K, A, _p(big), _p(big), 0, 8, C.byref(d), 0, -1.2, _p(i32), _p(out), _p(out), s),
                     "r4_batchrl_act")
            assert lib.r4_batchrl_launch_count() == before, (K, A, algo)
