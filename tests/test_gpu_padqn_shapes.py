"""GPU: the PA-DQN kernels (csrc/r4_padqn.cuh) against the float64 reference of tests/padqn_ref64.py at the shapes the
C-ABI accepts -- num_actions A in 2..512, emb_dim D in 1..512, n rows in 1..4194240 -- and the rejection of the first
shape outside each edge.

  pair scorer + act   A from 2 to 512 (both sides of the act warp's 32 lanes and of 128), D from 1 to 512 and one-hot
                      items, n from 1 to 8192 (the 8-row act CTAs,
                      the 64-row S tiles, and the 128-pair tiles just below and above one per SM), three mask regimes,
                      and A = 512 at n = 65536 on sampled rows.  Qm within 1e-4 of max |Qm| of the live entries, masked
                      entries exactly float32.min, argmax exact where the float64 top-two gap clears twice the bar and on
                      every planted tie (items with identical vectors: the kernel must take the first), SoftQ equal to
                      the float64 rule on the kernel's own uniforms away from a CDF step
  r4_padqn_grad       a subset of that grid at n from 1 to 2049 (TS = 8 rows per CTA, WK = 32; k_padqn_rows' shared
                      memory passes 48 KB above D = 256), weights given and NULL,
                      gamma 0, 0.9 and 1, terminal and all-masked next states, inv_n != 1 / n once, rewards placing td on
                      both Huber branches (padqn_ref64.grad_case); every tensor within GRAD_TOL of its max |ref| (SMALL_TOL
                      for tensors of at most 32 elements), td within 1e-4 of max(1, |ref|), the statistics within 1e-4 of
                      max(1, |ref|)
  r4_padqn_apply      steps 1, 2 and 10 carrying m and v, a clip that engages on some tensors only, copy_target on and off;
                      the caches equal a fresh r4_padqn_refresh byte for byte
  r4_padqn_train_step (A, D) = (2, 1), (284, 32), (512, 512), prioritised replay on and off: 11 / 10 launches, equal bit for
                      bit to its parts called one by one, and to a rerun
  r4_padqn_store      bit-exact against a NumPy ring at T = 1 and across the wrap
  rejections          R4_ERR_ARG with no launch one step past each edge

Every comparison is recorded as a `padqn ...` row of the session's margin table.  Measured on an H100 80GB HBM3 at a 700 W
power limit (SM clock up to 1980 MHz), worst err/bound over the grid with every bound at 1e-4 (b3 at SMALL_TOL): act Qm
0.063 (A 284 one-hot, n 1); gradient w1 0.025, w2 0.026, w3 0.017, b1 0.039, b2 0.053, b3 0.157 at 1e-3 (1.57 at
1e-4: A 129, D 1, n 2049); td 0.050; statistics 0.013; apply: the step 0.21, m 0.004, v 0.13.  The gradient tensors of
more than SMALL elements left 19x headroom at 1e-4 and are held to GRAD_TOL = 2e-5 (worst 0.26 there, b2).  The module
takes about 25 s and peaks at 1.4 GB of device memory (torch.cuda.max_memory_allocated).
"""
import ctypes as C

import numpy as np
import pytest

import golden_util
import padqn_ref64 as ref

pytestmark = pytest.mark.gpu

TOL = 1e-4
GRAD_TOL = 2e-5                    # gradient tensors of more than SMALL elements: worst 0.053 of 1e-4 on the first run
SMALL, SMALL_TOL = 32, 1e-3        # b3 (1 element) is a sum over the rows whose terms cancel: test_gpu_learner_shapes' rule
MAXN = 65535 * 64
NS = (1, 7, 8, 9, 63, 64, 65, 1000, 8192)
GRAD_NS = (1, 7, 8, 9, 31, 32, 33, 257, 2049)
# (A, D, onehot): every A of {2, 31, 32, 33, 127, 128, 129, 284, 511, 512} and every D of {1, 7, 32, 33, 256, 257, 512}
PAIR_GRID = [(2, 1, False), (2, 512, False), (31, 7, False), (32, 32, False), (33, 33, False), (127, 256, False),
             (128, 257, False), (129, 512, False), (284, 32, False), (284, 1, False), (511, 7, False), (512, 512, False),
             (512, 33, False), (284, 284, True), (512, 512, True)]
# (A, D, onehot, gamma, weighted, inv_n scale)
GRAD_GRID = [(2, 1, False, 0.9, True, 1.0), (31, 7, False, 1.0, False, 1.0), (33, 33, False, 0.0, True, 1.0),
             (128, 257, False, 0.9, False, 1.0), (284, 32, False, 0.9, True, 0.37), (284, 284, True, 1.0, False, 1.0),
             (512, 512, False, 1.0, True, 1.0), (129, 1, False, 0.9, True, 1.0)]


def _p(t, off=0):
    return C.c_void_p(t.data_ptr() + off) if t is not None else C.c_void_p(0)


def _lib():
    from rl4rs_b200 import _capi
    return _capi.load_library()


def _st():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ok(rc, what):
    assert rc == 0, "%s failed (%d): %s" % (what, rc, (_lib().r4_last_error(None) or b"?").decode())


def _cmp(what, got, want, bound):
    import torch
    if torch.is_tensor(bound):
        bound = bound.detach().double().cpu().numpy().reshape(-1)
    got = got.detach().double().cpu().numpy().reshape(-1)
    want = want.detach().double().cpu().numpy().reshape(-1)
    err = np.abs(got - want)
    bound = np.broadcast_to(np.asarray(bound, dtype=np.float64), err.shape)
    golden_util.record_margin("padqn " + what, err, bound, want)
    return float((err / bound).max()) if err.size else 0.0


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def tile_edge_ns(A=284):
    """The n at A whose 128-pair tile count is the largest below the SM count, and the next n (a tile count above it)."""
    lo = (sm_count() - 1) * 128 // A
    return lo, lo + 1


def _net(A, D, onehot, seed=0):
    """A ParametricQNetwork over item_vectors(A, D, dup=True) moved off its init (Q of order 1), its target perturbed,
    and PADQNKernelOps with both caches refreshed."""
    import torch
    from rl4rs_b200.policy import ParametricQNetwork
    from rl4rs_b200.trainer import PADQNKernelOps
    emb = ref.item_vectors(A, D, seed=seed, onehot=onehot, dup=not onehot)
    pol = ParametricQNetwork(emb, "cuda", seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        pol.flat.add_(0.05 * torch.randn(pol.n_params, generator=g).cuda())
        pol.flat[pol.slices[4][0]:pol.slices[4][1]] *= 2.0
        pol.target.copy_(pol.flat.detach() + 0.05 * torch.randn(pol.n_params, generator=g).cuda())
    ops = PADQNKernelOps(pol.emb, "cuda", pol.n_params, 64)
    ops.refresh(pol)
    return pol, ops


def _masks(regime, n, A, seed):
    import torch
    m = {"ones": lambda: np.ones((n, A), np.uint8), "env": lambda: ref.env_like_masks(n, A, seed),
         "planted": lambda: ref.planted_masks(n, A, seed)}[regime]()
    return torch.as_tensor(ref.plant_ties(m, A)).cuda()


def _check_act(tag, pol, ops, obs, mask, rows=None, ties=True):
    """Qm, argmax and SoftQ of ops.act over obs against qm_t (over `rows` only when given) -> worst err/bar.  ties: the
    plant_ties rows are ties (item_vectors with dup) and must take the first item of their pair."""
    import torch
    n, A = mask.shape
    q = torch.empty(n, A, device="cuda")
    a = torch.empty(n, dtype=torch.int32, device="cuda")
    ops.act(pol, obs, mask, False, 3, 0, a, q)
    s1 = torch.empty(n, dtype=torch.int32, device="cuda")
    ops.act(pol, obs, mask, True, 5, 1000, s1)
    u = ref.uniforms(5, 1000, n)
    if rows is not None:
        obs, mask, q, a, s1, u = obs[rows], mask[rows], q[rows], a[rows], s1[rows], u[rows.cpu().numpy()]
    q64 = ref.qm_t(ref.params_t(pol.flat, pol.D, "cuda"), obs, mask, pol.emb)
    live = mask.bool()
    assert torch.equal(q == ref.FLOAT_MIN, ~live), tag
    scale = float(q64[live].abs().max()) if bool(live.any()) else 1.0
    bar = TOL * scale
    worst = _cmp("act %s qm" % tag, q[live], q64[live], bar) if bool(live.any()) else 0.0
    assert worst <= 1, (tag, worst)
    clear = ref.top_gap(q64) > 2 * bar
    assert int((~clear).sum()) <= max(2, len(q64) // 10), tag
    assert torch.equal(a.long()[clear], q64.argmax(1)[clear]), tag
    tie = torch.arange(3, max(3, len(q64)), 11, device="cuda")
    if ties and rows is None and tie.numel():
        first = torch.tensor([min(pr) for pr in ref.tie_pairs(A)], device="cuda")[torch.arange(tie.numel(), device="cuda") %
                                                                                   len(ref.tie_pairs(A))]
        assert bool(clear[tie].all()) and torch.equal(a.long()[tie], first), tag
        assert torch.equal(q64.argmax(1)[tie], first), tag
    dead = ~live.any(1)
    assert bool((a[dead] == 0).all()), tag
    qh = q64.cpu().numpy()
    e = np.exp(qh - qh.max(1, keepdims=True))
    cdf = np.cumsum(e, 1) / e.sum(1, keepdims=True)
    margin = np.abs(cdf - u[:, None]).min(1) > 1e-3
    assert np.array_equal(s1.cpu().numpy()[margin], ref.act(qh, u)[margin]), tag
    assert bool(live[torch.arange(len(s1), device="cuda")[~dead], s1.long()[~dead]].all()), tag
    return worst


@pytest.mark.parametrize("A,D,onehot", PAIR_GRID)
@pytest.mark.parametrize("regime", ["ones", "env", "planted"])
def test_pair_scorer_and_act(A, D, onehot, regime, record_property):
    import torch
    pol, ops = _net(A, D, onehot, seed=A + D)
    ns = NS + (tile_edge_ns() if A == 284 else ())
    worst = 0.0
    for n in ns:
        g = torch.Generator().manual_seed(n)
        obs = torch.randn(n, 256, generator=g).cuda()
        worst = max(worst, _check_act("A%d D%d%s %s n%d" % (A, D, " onehot" if onehot else "", regime, n), pol, ops, obs,
                                      _masks(regime, n, A, n), ties=not onehot))
    record_property("worst_err_over_bar", worst)


def test_pair_scorer_at_65536_rows_on_sampled_rows():
    """A = 512, n = 65536: 262144 tiles over the persistent CTAs; the first and last rows, the rows of the tiles that
    start each pass of the persistent loop, and a random sample, each against float64."""
    import torch
    A, n = 512, 65536
    pol, ops = _net(A, 32, False, seed=9)
    g = torch.Generator().manual_seed(9)
    obs = torch.randn(n, 256, generator=g).cuda()
    mask = _masks("env", n, A, 9)
    sms = sm_count()
    passes = [k * sms * 128 // A for k in range(1, n * A // (128 * sms) + 1, 97)]
    rows = sorted(set(range(64)) | set(range(n - 64, n)) | {r + d for r in passes for d in (-1, 0, 1) if 0 <= r + d < n} |
                  set(torch.randint(0, n, (256,), generator=g).tolist()))
    _check_act("A512 D32 n65536 sampled", pol, ops, obs, mask, torch.tensor(rows, device="cuda"))


def _caches(A):
    import torch
    cb = _lib().r4_padqn_cache_size(A)
    return torch.zeros(cb, dtype=torch.uint8, device="cuda"), torch.zeros(cb, dtype=torch.uint8, device="cuda")


def _refresh(params, emb, A, D):
    c, _ = _caches(A)
    _ok(_lib().r4_padqn_refresh(_p(params), _p(emb), A, D, _p(c), None, _st()), "r4_padqn_refresh")
    return c


def _grad(pol, case, gamma, scratch=None):
    """r4_padqn_grad over the case's pool -> (grad, td, stats, launches)."""
    import torch
    lib = _lib()
    A, D = pol.A, pol.D
    n = case["idx"].numel()
    scratch = torch.zeros(lib.r4_padqn_scratch_size(A, D, n), device="cuda") if scratch is None else scratch
    grad, td, stats = torch.zeros(pol.n_params, device="cuda"), torch.zeros(n, device="cuda"), torch.zeros(3, device="cuda")
    c_on, c_tg = _refresh(pol.flat, pol.emb, A, D), _refresh(pol.target, pol.emb, A, D)
    l0 = lib.r4_learner_launch_count()
    rc = lib.r4_padqn_grad(_p(pol.flat), _p(pol.target), _p(c_on), _p(c_tg), _p(pol.emb), A, D, _p(case["obs"]),
                           _p(case["action"]), _p(case["reward"]), _p(case["new_obs"]), _p(case["done"]),
                           _p(case["next_mask"]), _p(case["idx"]), _p(case["weights"]), n, gamma, case["inv_n"],
                           _p(scratch), _p(grad), _p(td), _p(stats), _st())
    torch.cuda.synchronize()
    _ok(rc, "r4_padqn_grad")
    return grad, td, stats, lib.r4_learner_launch_count() - l0


def _check_grad(tag, pol, grad, r):
    worst = 0.0
    for (lo, hi), name in zip(pol.slices, ref.NAMES):
        want = r["grads"][name].reshape(-1)
        tol = GRAD_TOL if hi - lo > SMALL else SMALL_TOL
        q = _cmp("grad %s %s" % (tag, name), grad[lo:hi], want, tol * max(float(want.abs().max()), 1e-30))
        assert q <= 1, (tag, name, q)
        worst = max(worst, q)
    return worst


@pytest.mark.parametrize("A,D,onehot,gamma,weighted,inv_scale", GRAD_GRID)
def test_grad_matches_float64(A, D, onehot, gamma, weighted, inv_scale, record_property):
    pol, _ = _net(A, D, onehot, seed=2 * A + D)
    worst = 0.0
    for n in GRAD_NS:
        tag = "A%d D%d%s g%g%s n%d" % (A, D, " onehot" if onehot else "", gamma, " w" if weighted else "", n)
        case = ref.grad_case(pol.flat.detach(), pol.target, pol.emb, n, gamma, weighted, seed=n,
                             inv_n=inv_scale / n)
        grad, td, stats, launches = _grad(pol, case, gamma)
        assert launches == 7
        r = case["ref"]
        worst = max(worst, _check_grad(tag, pol, grad, r))
        assert _cmp("grad %s td" % tag, td, r["td"], TOL * r["td"].abs().clamp_min(1.0)) <= 1, tag
        assert _cmp("grad %s stats" % tag, stats, r["stats"], TOL * r["stats"].abs().clamp_min(1.0)) <= 1, tag
    record_property("worst_err_over_bar", worst)


def test_grad_with_non_terminal_all_masked_next_states():
    """Rows 5 mod 13 of the pool have every next action masked and are not terminal: a* = 0 and y = r + gamma float32.min,
    so td is about 3e38 there.  td, Q and the gradient (those rows sit on the linear Huber branch, dQ = w inv_n) are held to
    float64.  The loss and mean-td statistics are not: each is a float32 sum of several terms near 3e38, which overflows
    to inf, as the reference's float32 reduce_mean would; the mean Q statistic is still held to float64."""
    import torch
    pol, _ = _net(284, 32, False, seed=5)
    case = ref.grad_case(pol.flat.detach(), pol.target, pol.emb, 64, 0.9, True, seed=5, dead_next=True)
    r = case["ref"]
    dead = ~case["next_mask"][case["idx"]].bool().any(1) & (case["done"][case["idx"]] == 0)
    assert int(dead.sum()) >= 3 and bool((r["td"][dead] > 1e38).all())
    grad, td, stats, _ = _grad(pol, case, 0.9)
    _check_grad("dead-next A284 D32 n64", pol, grad, r)
    assert _cmp("grad dead-next td", td, r["td"], TOL * r["td"].abs().clamp_min(1.0)) <= 1
    assert _cmp("grad dead-next mean q", stats[2:], r["stats"][2:], TOL * r["stats"][2:].abs().clamp_min(1.0)) <= 1
    assert bool(torch.isinf(stats[:2]).all())


def _apply(pol, grad, m, v, cache, tcache, step, clip, copy):
    lib = _lib()
    l0 = lib.r4_learner_launch_count()
    _ok(lib.r4_padqn_apply(_p(pol.flat), _p(pol.target), _p(grad), _p(m), _p(v), _p(pol.emb), pol.A, pol.D, _p(cache),
                           _p(tcache), step, 5e-4, 1e-8, clip, int(copy), _st()), "r4_padqn_apply")
    return lib.r4_learner_launch_count() - l0


@pytest.mark.parametrize("A,D", [(2, 1), (284, 32), (512, 512)])
def test_apply_steps_clip_and_caches(A, D):
    """Steps 1, 2 and 10 with m and v carried over; the gradient's per-tensor norms are 5, 0.3, 2, 0.1, 0.5 and 3 against a
    clip of 1, so the clip engages on w1, w2 and b3 only.  Each step against padqn_ref64.apply from the kernel's state
    before it.  After each step both caches equal a fresh r4_padqn_refresh byte for byte."""
    import torch
    pol, _ = _net(A, D, False, seed=A)
    pol.flat.requires_grad_(False)
    m, v = torch.zeros(pol.n_params, device="cuda"), torch.zeros(pol.n_params, device="cuda")
    cache, tcache = _refresh(pol.flat, pol.emb, A, D), _refresh(pol.target, pol.emb, A, D)
    g = torch.Generator().manual_seed(A)
    norms = (5.0, 0.3, 2.0, 0.1, 0.5, 3.0)
    for step, copy in ((1, False), (2, True), (10, False)):
        grad = torch.empty(pol.n_params)
        for (lo, hi), nrm in zip(pol.slices, norms):
            x = torch.randn(hi - lo, generator=g, dtype=torch.float64)
            grad[lo:hi] = (x * nrm / x.norm()).float()
        grad = grad.cuda()
        f0, t0, m0, v0 = (x.double().cpu().numpy() for x in (pol.flat, pol.target, m, v))
        tc0 = tcache.clone()
        assert _apply(pol, grad, m, v, cache, tcache, step, 1.0, copy) == 2
        torch.cuda.synchronize()
        f1, t1, m1, v1 = ref.apply(f0, t0, grad.double().cpu().numpy(), m0, v0, step, D, clip=1.0, copy_target=copy)
        tag = "apply A%d D%d step%d" % (A, D, step)
        for (lo, hi), name in zip(pol.slices, ref.NAMES):
            dk = torch.as_tensor(pol.flat[lo:hi].double().cpu().numpy() - f0[lo:hi])
            dr = torch.as_tensor(f1[lo:hi] - f0[lo:hi])
            ulp = float(np.abs(f0[lo:hi]).max()) * 2.0 ** -23
            assert _cmp("%s %s step" % (tag, name), dk, dr, TOL * float(dr.abs().max()) + ulp) <= 1, (tag, name)
            for what, got, want in (("m", m, m1), ("v", v, v1)):
                want = torch.as_tensor(want[lo:hi])
                assert _cmp("%s %s %s" % (tag, name, what), got[lo:hi], want, TOL * float(want.abs().max())) <= 1
        if copy:
            assert torch.equal(pol.target, pol.flat)
            assert torch.equal(tcache, cache)
        else:
            assert np.array_equal(pol.target.double().cpu().numpy(), t1)
            assert torch.equal(tcache, tc0)
        assert torch.equal(cache, _refresh(pol.flat, pol.emb, A, D))
        assert torch.equal(tcache, _refresh(pol.target, pol.emb, A, D))


def _trainer(A, D, prio, seed=0):
    import torch
    from test_trainer_padqn_cpu import FakeEnv
    from rl4rs_b200.trainer import get_rl_model
    tr = get_rl_model("PADQN", {"buffer_size": 300, "train_batch_size": 64, "prioritized_replay": prio},
                      env=FakeEnv(8, A=A, D=D), device="cuda", seed=seed)
    assert tr.use_kernels
    g = torch.Generator().manual_seed(1)
    T, B = 9, 40
    obs, fin = torch.randn(T, B, 256, generator=g).cuda(), torch.randn(B, 256, generator=g).cuda()
    mask = torch.as_tensor(ref.env_like_masks(T * B, A, 1)).view(T, B, A).cuda()
    fmask = torch.as_tensor(ref.env_like_masks(B, A, 2)).cuda()
    act = torch.randint(0, A, (T, B), generator=g, dtype=torch.int32).cuda()
    rew = torch.randn(T, B, generator=g).cuda()
    done = torch.zeros(T, B, dtype=torch.uint8).cuda()
    done[-1] = 1
    tr.replay.store(obs, fin, act, rew, done, mask, fmask)
    return tr


def _state(tr):
    out = {"flat": tr.policy.flat.detach().clone(), "target": tr.policy.target.clone(), "m": tr.ops.m.clone(),
           "v": tr.ops.v.clone(), "cache": tr.ops.cache.clone(), "target_cache": tr.ops.target_cache.clone()}
    if tr.replay.prio is not None:
        out["prio"] = tr.replay.prio.clone()
        out["max_prio"] = tr.replay.max_prio.clone()
    return out


@pytest.mark.parametrize("A,D", [(2, 1), (284, 32), (512, 512)])
@pytest.mark.parametrize("prio", [True, False])
def test_train_step_is_its_parts_and_reruns_bit_identically(A, D, prio):
    import torch
    runs = []
    for composed in (False, False, True):
        tr = _trainer(A, D, prio)
        hp = tr._hp()
        u = torch.rand(64, generator=torch.Generator().manual_seed(4)).cuda()
        for step, copy in ((1, True), (2, False)):
            if composed:
                ops, pol, rb = tr.ops, tr.policy, tr.replay
                idx, w = ops.replay_sample(rb, u, hp["beta"])
                ops.grad_(pol, rb, idx, w if prio else None, hp["gamma"], 1.0 / 64)
                ops.apply(pol, step, hp, copy)
                if prio:
                    ops.replay_priorities(rb, idx, ops.td, hp["eps"])
            else:
                l0 = tr.ops.launches
                tr.ops.train_step(tr.policy, tr.replay, u, step, copy, hp)
                torch.cuda.synchronize()
                assert tr.ops.launches - l0 == (11 if prio else 10)
        torch.cuda.synchronize()
        runs.append(_state(tr))
    assert not torch.equal(runs[0]["flat"], _trainer(A, D, prio).policy.flat.detach())
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), ("rerun", k)
        assert torch.equal(runs[0][k], runs[2][k]), ("parts", k)


def _ring(C, A):
    import torch
    z = lambda *s, dt=torch.float32: torch.full(s, 7, dtype=dt, device="cuda")
    return [z(C, 256), z(C, dt=torch.int32), z(C), z(C, 256), z(C, dt=torch.uint8), z(C, A, dt=torch.uint8), z(C)]


@pytest.mark.parametrize("A", [2, 512])
@pytest.mark.parametrize("T,B,C,pos", [(1, 13, 50, 45), (9, 8, 50, 47), (5, 40, 64, 1000003)])
def test_store_matches_a_numpy_ring(A, T, B, C, pos):
    """T = 1: every row takes the final observation and mask.  T B > C: only the last C rows are written, from pos near
    (or far past) a wrap.  Every ring tensor bit for bit; the priorities max_prio^alpha within 2 ulp."""
    import torch
    g = torch.Generator().manual_seed(A + T)
    obs, fin = torch.randn(T, B, 256, generator=g), torch.randn(B, 256, generator=g)
    mask = torch.randint(0, 2, (T, B, A), generator=g, dtype=torch.uint8)
    fmask = torch.randint(0, 2, (B, A), generator=g, dtype=torch.uint8)
    act = torch.randint(0, A, (T, B), generator=g, dtype=torch.int32)
    rew, done = torch.randn(T, B, generator=g), torch.randint(0, 2, (T, B), generator=g, dtype=torch.uint8)
    ring = _ring(C, A)
    want = [x.cpu().numpy().copy() for x in ring]
    max_prio, alpha = torch.tensor([2.25], device="cuda"), 0.6
    lib = _lib()
    l0 = lib.r4_learner_launch_count()
    inputs = [x.cuda() for x in (obs, fin, mask, fmask, act, rew, done)]
    _ok(lib.r4_padqn_store(*[_p(x) for x in ring[:6]], _p(ring[6]), _p(max_prio), C, A, pos, alpha,
                           *[_p(x) for x in inputs], T, B, _st()), "r4_padqn_store")
    torch.cuda.synchronize()
    assert lib.r4_learner_launch_count() - l0 == 1
    n = T * B
    o, m = obs.reshape(n, 256).numpy(), mask.reshape(n, A).numpy()
    nxt = np.concatenate([o[B:], fin.numpy()])
    nmask = np.concatenate([m[B:], fmask.numpy()])
    for r in range(max(0, n - C), n):
        s = (pos + r) % C
        want[0][s], want[1][s], want[2][s] = o[r], act.reshape(-1)[r], rew.reshape(-1)[r]
        want[3][s], want[4][s], want[5][s] = nxt[r], done.reshape(-1)[r], nmask[r]
        want[6][s] = np.float32(2.25 ** 0.6)
    for k in range(6):
        assert np.array_equal(ring[k].cpu().numpy(), want[k]), k
    p = ring[6].cpu().numpy()
    assert np.all(np.abs(p.view(np.int32).astype(np.int64) - want[6].view(np.int32).astype(np.int64)) <= 2)


def test_rejections_one_step_past_each_edge():
    """R4_ERR_ARG and no launch at A = 1 and 513, D = 0 and 513, n = 0 and n = 4194241 (at A = 2, 284, 512), a cache or
    scratch 8 bytes off 16, cache == cache2 and step 0.  The scratch size is asserted -1 at a refused n before r4_padqn_grad
    or r4_padqn_train_step is called there, since both read idx[0..n)."""
    import torch
    lib = _lib()
    A, D, n = 284, 32, 16
    buf = torch.zeros(1 << 20, device="cuda")                     # 4 MB: every pointer below is inside it
    p, off = _p(buf), _p(buf, 8)
    st = _st()
    l0 = lib.r4_learner_launch_count()

    def act(A_, D_, n_, cache=p, scratch=p):
        return lib.r4_padqn_act(p, cache, p, p, n_, A_, D_, 0, 0, 0, p, None, scratch, st)

    def grad(A_, D_, n_, cache=p, scratch=p):
        return lib.r4_padqn_grad(p, p, cache, p, p, A_, D_, p, p, p, p, p, p, p, None, n_, 0.9, 0.1, scratch, p, None, None,
                                 st)

    def apply(A_, D_, step=1, cache=p, tcache=_p(buf, 1 << 10)):
        return lib.r4_padqn_apply(p, p, p, p, p, p, A_, D_, cache, tcache, step, 5e-4, 1e-8, 40.0, 0, st)

    def train(A_, D_, n_, step=1, cache=p, tcache=_p(buf, 1 << 10), scratch=p):
        return lib.r4_padqn_train_step(p, p, p, p, p, cache, tcache, A_, D_, p, p, p, p, p, p, p, p, 100, n_, p, 0.4, 0.6,
                                       1e-6, 1.0, step, 5e-4, 1e-8, 40.0, 0, scratch, None, st)

    got = []
    for A_, D_ in ((1, D), (513, D), (A, 0), (A, 513)):
        assert lib.r4_padqn_scratch_size(A_, D_, n) == -1 and lib.r4_padqn_num_params(A_, D_) == -1
        got += [act(A_, D_, n), grad(A_, D_, n), apply(A_, D_), train(A_, D_, n),
                lib.r4_padqn_refresh(p, p, A_, D_, p, None, st)]
    assert lib.r4_padqn_cache_size(1) == -1 and lib.r4_padqn_cache_size(513) == -1
    assert lib.r4_padqn_scratch_size(A, D, 0) == -1
    got += [act(A, D, 0), grad(A, D, 0), train(A, D, 0)]
    for A_ in (2, 284, 512):
        assert lib.r4_padqn_scratch_size(A_, D, MAXN) > 0
        assert lib.r4_padqn_scratch_size(A_, D, MAXN + 1) == -1, A_    # before any call at that n
    for A_ in (2, 284, 512):
        got += [act(A_, D, MAXN + 1), grad(A_, D, MAXN + 1), train(A_, D, MAXN + 1)]
    got += [act(A, D, n, cache=off), act(A, D, n, scratch=off), grad(A, D, n, cache=off), grad(A, D, n, scratch=off),
            apply(A, D, cache=off, tcache=p), train(A, D, n, scratch=off), train(A, D, n, cache=off),
            lib.r4_padqn_refresh(p, p, A, D, off, None, st), lib.r4_padqn_refresh(p, p, A, D, p, off, st)]
    got += [lib.r4_padqn_refresh(p, p, A, D, p, p, st), apply(A, D, tcache=p), train(A, D, n, tcache=p)]
    got += [apply(A, D, step=0), train(A, D, n, step=0)]
    torch.cuda.synchronize()
    assert lib.r4_learner_launch_count() == l0
    assert got == [-1] * len(got), got
