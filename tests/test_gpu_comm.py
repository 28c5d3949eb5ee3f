"""GPU: the data-parallel learner -- every entry point that takes an r4_comm -- against its single-GPU form, and the
refusal of a communicator that is not ready or was made for another parameter count.

One GPU (a world-1 communicator).  A world-1 communicator is ready when r4_comm_create returns; its exchange publishes its
own flag and waits on that same flag, so k_exchange_adam cannot wait on anything outside the kernel.  The single-GPU
paths are held to float64 by test_gpu_learner_shapes.py and test_gpu_optim_shapes.py, so the bar here is bit identity
with them, which a dropped partial, a wrong scale, a missing flat store or a statistic summed twice all break:
- r4_grad_exchange_n at n_params around one 256-thread block and at every learner's size, G from 1 to the SM count,
  forty calls on one communicator (its step count runs through both inbox parities): flat_grad is the float32 sum of
  the G partials in c order from +0.0, stats_accum += (the same sum of the statistics) * stat_scale as ONE fma (the
  SASS of the parent build already contracted the product into FFMA here, in k_reduce_adam and in k_grad_reduce; the
  kernel now says fmaf, as k_dense_wgrad's Stats do), the partials untouched and NaN sentinels around every written
  buffer intact;
- r4_ppo_epoch_dist / r4_gauss_ppo_epoch_dist against r4_ppo_epoch / r4_gauss_ppo_epoch (grad_clip 0), the A2C pairs
  (r4_policy_grad_partial + r4_grad_exchange against r4_policy_grad; the Gaussian r4_gauss_grad + r4_grad_exchange_n
  against r4_gauss_grad), r4_impala_step / r4_gauss_impala_step and r4_ddpg_train_step / r4_rainbow_train_step with
  the communicator against NULL: every output bit for bit, and the launch count pinned per path (the exchange replaces
  k_reduce_adam / k_grad_reduce / k_adam where the single-GPU form has one, and adds one launch where it has none);
- refusals: r4_comm_create / r4_comm_open argument edges, and each of the eight entry points given a world-2
  communicator that was never opened (R4_ERR_STATE) or a world-1 one made for another parameter count (R4_ERR_ARG)
  returns that code with no launch and every output and scratch buffer unchanged.  At the parent commit the two PPO
  epochs and the DDPG / RAINBOW steps launched their gradient kernels (and the replay sample) before refusing, and
  r4_impala_step / r4_gauss_impala_step answered an unopened communicator with R4_ERR_ARG: those ten cases failed.

Several ranks (test_multi_rank_*): one process per visible GPU, needing at least two GPUs that can map each other, else
skipped with the count found; world 2, 3 (order bugs show from three ranks on: float addition is commutative) and every
visible GPU up to 8, each rank set up through trainer.PeerComm.  C1 / C6: the raw exchange on four live communicators
against the rank-order sum of the all-gathered partials, and a refusal made alike on every rank leaving the protocol
intact.  C2 / C3: the two PPO epochs, per step the summed gradient against float64 over the union of the ranks' rows at
1/(mb W), params / m / v within optim_ref64's Adam bounds from the kernel's own gradient, this rank's statistics at 1/mb
(not rescaled by W), replicas bit-identical, and one two-step call equal to the loop.  C4: the A2C pairs and IMPALA steps
of both policies against float64 over the union at inv_n = 1 (V-trace rank-local), the clip on the global norm.  C5: the
DDPG / TD3 / RAINBOW steps equal to r4_*_apply of the rank-order sum of r4_*_grad at 1/(n W).  C7: PPO, A2C, PPO_conti
and A2C_conti on the CUDA env, the peer path against the NCCL fallback (the bound is derived above _phase_trainers).
test_rank_checks_in_one_process runs C1 - C5 through the same harness with one rank, so their references and bounds are
exercised on any single GPU; the sums across ranks, and so the world-size scale mutants (the epoch's loss at 1/mb, its
statistics at 1/(mb W), DDPG's inv_n without W), are only seen from two GPUs on.  The multi-rank tests have not yet run
where two GPUs were visible: on a single H100 they skip.

Each mutant below failed these tests on one H100 run: k_exchange_adam's partial loop starting at c = 1 (every
test_raw_exchange case and the stats-less one), the `if (flat)` store dropped (all 42 cases of the two epoch tests), the
up-front communicator check of the two PPO epochs and the DDPG / RAINBOW steps removed, with the launcher's own check
left as the backstop (their 8 refusal cases: the kernels launched before the refusal).
"""
import contextlib
import math
import ctypes as C
import os

import numpy as np
import pytest

import golden_util
import learner_ref64 as R

pytestmark = pytest.mark.gpu

R4_ERR_ARG, R4_ERR_STATE = -1, -2            # include/rl4rs_b200.h
PAD = 64
CALLS = 40


def _lib():
    from rl4rs_b200 import _capi
    return _capi.load_library()


def _err():
    return (_lib().r4_last_error(None) or b"?").decode()


def _ok(rc, what):
    if rc != 0:
        raise AssertionError("%s failed (%d): %s" % (what, rc, _err()))


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _bits(t):
    import torch
    t = t.detach().contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _same(a, b):
    import torch
    return torch.equal(_bits(a), _bits(b))


def _launched(fn):
    """-> (fn's result, the learner kernels it launched as the library counts them)."""
    import torch
    lib = _lib()
    torch.cuda.synchronize()
    n0 = lib.r4_learner_launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, lib.r4_learner_launch_count() - n0


class Comm(object):
    """An r4_comm of this process on the current device: ready at once for world 1; for world > 1 never opened here."""
    ok = True                                        # as trainer.PeerComm's flag: a world-1 communicator is ready

    def __init__(self, n_params, world=1, rank=0):
        self.h = C.c_void_p()
        _ok(_lib().r4_comm_create(rank, world, n_params, C.byref(self.h)), "r4_comm_create")
        assert self.h.value

    def close(self):
        if self.h is not None and self.h.value:
            _lib().r4_comm_destroy(self.h)
        self.h = None


@contextlib.contextmanager
def _comm(n_params, world=1, rank=0):
    c = Comm(n_params, world, rank)
    try:
        yield c
    finally:
        c.close()


def _record(what, got, want):
    """A bit-exact comparison as a `comm ...` row of the margin table (bound: one ulp of the larger magnitude)."""
    g, w = got.detach().double().cpu().numpy().reshape(-1), want.detach().double().cpu().numpy().reshape(-1)
    err = np.abs(g - w)
    ulp = np.spacing(np.maximum(np.abs(w), np.abs(g)).astype(np.float32)).astype(np.float64)
    golden_util.record_margin("comm " + what, err, np.maximum(ulp, 1e-45), w)


def _check_same(what, got, want, where=""):
    _record(what, got, want)
    assert _same(got, want), "%s%s: max |diff| %.3g" % (what, where, float((got.double() - want.double()).abs().max()))


# ---- A1: the raw exchange ---------------------------------------------------------------------------------------------
RAW_SIZES = (("n", 1), ("n", 255), ("n", 256), ("n", 257), ("policy", 2), ("policy", 284), ("gauss", 64),
             ("ddpg", (32, 1)), ("rainbow", (284, 8)))


def _n_params(kind, arg):
    lib = _lib()
    return {"n": lambda: arg, "policy": lambda: lib.r4_policy_num_params(arg), "gauss": lambda: lib.r4_gauss_num_params(arg),
            "ddpg": lambda: lib.r4_ddpg_num_params(*arg), "rainbow": lambda: lib.r4_rainbow_num_params(*arg)}[kind]()


class Padded(object):
    """A float32 device buffer between two PAD-element NaN sentinels."""

    def __init__(self, x):
        import torch
        self.n = x.numel()
        self.full = torch.full((self.n + 2 * PAD,), float("nan"), dtype=torch.float32, device="cuda")
        self.full[PAD:PAD + self.n] = x.reshape(-1)
        self.t = self.full[PAD:PAD + self.n]

    @property
    def ptr(self):
        return C.c_void_p(self.full.data_ptr() + 4 * PAD)

    def sentinel_ok(self):
        import torch
        return bool(torch.isnan(self.full[:PAD]).all()) and bool(torch.isnan(self.full[PAD + self.n:]).all())


def _partials(G, n, gen):
    """G partial gradients [G, n] then their statistics [G, 5]: magnitudes over six decades, both signs, exact zeros and
    values that cancel between partials."""
    import torch
    x = torch.randn(G * (n + 5), generator=gen, device="cuda")
    x = x * torch.pow(10.0, torch.randint(-3, 3, (x.numel(),), generator=gen, device="cuda").float())
    x[3::7] = 0.0                                   # not element 0: at n = 1 it is the whole of partial 0
    if G > 1:
        x[n:2 * n:3] = -x[0:n:3]                     # partial 1 cancels partial 0 on every third element
    return x


def _csum(rows):
    """The float32 sum of rows [G, k] in row order from +0.0, one IEEE rounding per addition."""
    import torch
    s = torch.zeros(rows.shape[1], dtype=torch.float32, device=rows.device)
    for c in range(rows.shape[0]):
        s = s + rows[c]
    return s


SCALES = (1.0, 0.5, float(np.float32(1.0 / 3.0)))


def _fma32(a, b, c):
    """float32 fmaf(a, b, c) element by element: the exact a b + c (as a fraction) rounded once, to nearest even."""
    from fractions import Fraction
    out = []
    for x, y, z in zip(np.asarray(a, np.float32), np.asarray(b, np.float32), np.asarray(c, np.float32)):
        e = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        f = np.float32(float(e))
        cands = (f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf)))
        out.append(min(cands, key=lambda q: (abs(Fraction(float(q)) - e), int(np.float32(q).view(np.int32)) & 1)))
    return np.array(out, dtype=np.float32)


@pytest.mark.parametrize("kind,arg", RAW_SIZES)
def test_raw_exchange(kind, arg):
    """r4_grad_exchange_n, forty calls on one world-1 communicator, G in {1, 15, 16, 17, 64, SM count}, stat_scale 1, 0.5
    and float32(1/3): the statistics restated as one correctly rounded fma, which at 1/3 differs from a rounded product
    added after it (two roundings)."""
    import torch
    lib = _lib()
    n = _n_params(kind, arg)
    assert n > 0
    Gs = (1, 15, 16, 17, 64, _sms())
    gen = torch.Generator(device="cuda").manual_seed(n)
    with _comm(n) as comm:
        flat = Padded(torch.zeros(n, device="cuda"))
        stats = Padded(torch.randn(5, generator=gen, device="cuda"))
        want_stats = stats.t.clone()
        for k in range(CALLS):
            G, scale = Gs[k % len(Gs)], SCALES[(k // len(Gs)) % len(SCALES)]
            part = _partials(G, n, gen)
            keep = part.clone()
            flat.t.fill_(-3.5)
            _, launches = _launched(lambda: _ok(lib.r4_grad_exchange_n(comm.h, _p(part), G, n, flat.ptr, stats.ptr, scale,
                                                                       _stream()), "r4_grad_exchange_n"))
            assert launches == 1
            what, where = "exchange %s n%d" % (kind, n), " call %d G %d scale %g" % (k, G, scale)
            _check_same(what + " flat", flat.t, _csum(part[:G * n].view(G, n)), where)
            a = _csum(part[G * n:].view(G, 5)).cpu().numpy()
            want_stats = torch.from_numpy(_fma32(a, np.full(5, scale, np.float32), want_stats.cpu().numpy())).cuda()
            _check_same(what + " stats", stats.t, want_stats, where)
            assert _same(part, keep), what + where + ": the partials changed"
            assert flat.sentinel_ok() and stats.sentinel_ok(), what + where


def test_raw_exchange_without_stats_writes_only_flat():
    """stats_accum NULL: flat_grad alone is written (the replay learners' form)."""
    import torch
    lib = _lib()
    n, G = 257, 3
    gen = torch.Generator(device="cuda").manual_seed(1)
    with _comm(n) as comm:
        part = _partials(G, n, gen)
        flat = Padded(torch.zeros(n, device="cuda"))
        _ok(lib.r4_grad_exchange_n(comm.h, _p(part), G, n, flat.ptr, None, 1.0, _stream()), "r4_grad_exchange_n")
        torch.cuda.synchronize()
        _check_same("exchange nostats flat", flat.t, _csum(part[:G * n].view(G, n)))
        assert flat.sentinel_ok()


# ---- A2: the PPO epoch ------------------------------------------------------------------------------------------------
def _carried(n, seed):
    import torch
    import optim_ref64 as O
    _, m, v = O.carried(n, seed)
    return torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda()


def _mask_setup(A, n, seed):
    import torch
    from rl4rs_b200.policy import MaskedPolicy
    dev = torch.device("cuda")
    pol = MaskedPolicy(A, dev, seed=3)
    with torch.no_grad():
        pol.flat.add_(0.05 * torch.randn(pol.n_params, generator=torch.Generator().manual_seed(seed)).to(dev))
    return pol, R.mask_batch(pol, n, A, dev, seed=seed)


def _gauss_setup(D, n, seed):
    import torch
    from rl4rs_b200.policy import GaussianPolicy
    dev = torch.device("cuda")
    pol = GaussianPolicy(D, dev, seed=3)
    with torch.no_grad():
        pol.flat.add_(0.02 * torch.randn(pol.n_params, generator=torch.Generator().manual_seed(seed)).to(dev))
    return pol, R.gauss_batch(pol, n, D, dev, seed=seed)


def _epoch_pair(make_ops, pol, data, n, mb, step0, seed):
    """-> the single-GPU and the world-1 data-parallel epoch from the same state: (steps, launches, flat, ops) each."""
    import torch
    m0, v0 = _carried(pol.n_params, seed)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(seed)).cuda()
    hp = R.PG_HP[0]
    out = []
    for dist in (False, True):
        ops = make_ops()
        ops.m.copy_(m0)
        ops.v.copy_(v0)
        ops.step = step0
        flat = pol.flat.detach().clone()
        if dist:
            with _comm(pol.n_params) as comm:
                steps, launches = _launched(lambda: ops.ppo_epoch_dist(comm, flat, data, perm, n, mb, hp, 1e-3))
        else:
            steps, launches = _launched(lambda: ops.ppo_epoch(flat, data, perm, n, mb, hp, 1e-3, None))
        out.append((steps, launches, flat, ops))
    return out


def _check_epoch(what, single, dist, steps):
    (s0, l0, f0, o0), (s1, l1, f1, o1) = single, dist
    assert s0 == s1 == steps, (what, s0, s1, steps)
    assert l0 == l1, (what, l0, l1)
    for name, a, b in (("params", f1, f0), ("m", o1.m, o0.m), ("v", o1.v, o0.v), ("flat_grad", o1.grad, o0.grad),
                       ("stats", o1.stats, o0.stats)):
        _check_same("%s %s" % (what, name), a, b)
    assert o1.step == o0.step


@pytest.mark.parametrize("step0", [0, 10000])
@pytest.mark.parametrize("n,mb", [(1, 1), (7, 4), (2048, 256), (1000, 257), (4096, 4096)])
@pytest.mark.parametrize("A", [2, 284, 512])
def test_ppo_epoch_dist_is_the_single_gpu_epoch(A, n, mb, step0):
    """r4_ppo_epoch_dist on a world-1 communicator against r4_ppo_epoch with grad_clip 0 (the fused k_reduce_adam
    path): (7, 4) leaves rows unused, (4096, 4096) caps G at the SM count."""
    from rl4rs_b200.trainer import KernelOps
    pol, data = _mask_setup(A, n, seed=A + n + mb)
    single, dist = _epoch_pair(lambda: KernelOps(A, pol.flat.device, pol.n_params), pol, data, n, mb, step0, seed=A + mb)
    _check_epoch("ppo_epoch A%d n%d mb%d s%d" % (A, n, mb, step0), single, dist, n // mb)
    assert single[1] == 2 * (n // mb)                # k_policy_grad + k_reduce_adam, or + k_exchange_adam


# ---- A3: the Gaussian PPO epoch ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("mb", [1, 256, 2048, 2049])
@pytest.mark.parametrize("D", [2, 32, 64])
def test_gauss_ppo_epoch_dist_is_the_single_gpu_epoch(D, mb):
    """r4_gauss_ppo_epoch_dist against r4_gauss_ppo_epoch (grad_clip 0) over two minibatches and a leftover row; at
    mb = 2049 each step takes two k_gauss_rows chunks.  The exchange replaces k_adam: the same launch count."""
    from rl4rs_b200.trainer import GaussKernelOps
    n = 2 * mb + 1
    pol, data = _gauss_setup(D, n, seed=D + mb)
    single, dist = _epoch_pair(lambda: GaussKernelOps(D, pol.flat.device, pol.n_params), pol, data, n, mb, 0, seed=D + mb)
    _check_epoch("gauss_epoch D%d mb%d" % (D, mb), single, dist, n // mb)
    assert single[1] == n // mb * (2 * -(-mb // 2048) + 1)


# ---- A4: the A2C pairs ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 5, 284, 4096])
@pytest.mark.parametrize("A", [2, 284, 512])
@pytest.mark.parametrize("mode", [0, 1])
def test_policy_grad_partial_and_exchange_is_policy_grad(mode, A, n):
    """r4_policy_grad_partial + r4_grad_exchange against r4_policy_grad, at the trainer's G and at G = 1: flat_grad and
    the statistics bit for bit, and two launches either way (k_policy_grad, then k_grad_reduce or the exchange)."""
    import torch
    from rl4rs_b200.trainer import KernelOps, _hp
    lib = _lib()
    pol, data = _mask_setup(A, n, seed=A + n + mode)
    hp = R.PG_HP[mode]
    inv_n, stat_scale = (1.0 / n if mode == 0 else 1.0), 1.0 / n
    for G in sorted({max(1, min((n + 3) // 4, _sms())), 1}):
        what = "a2c mask mode%d A%d n%d G%d" % (mode, A, n, G)
        a = KernelOps(A, pol.flat.device, pol.n_params)
        b = KernelOps(A, pol.flat.device, pol.n_params)
        for ops in (a, b):
            ops.stats.copy_(torch.tensor([0.5, -1.0, 0.25, 2.0, 3.0]))
        _, la = _launched(lambda: a.policy_grad(mode, pol.flat, data, None, 0, n, hp, inv_n, stat_scale, G=G))
        with _comm(pol.n_params) as comm:
            def pair():
                _ok(lib.r4_policy_grad_partial(mode, _p(pol.flat), *map(_p, data), None, n, A, *_hp(hp), inv_n,
                                               _p(b.scratch), G, _stream()), "r4_policy_grad_partial")
                _ok(lib.r4_grad_exchange(comm.h, _p(b.scratch), G, A, _p(b.grad), _p(b.stats), stat_scale, _stream()),
                    "r4_grad_exchange")
            _, lb = _launched(pair)
        assert la == lb == 2, (what, la, lb)
        _check_same(what + " flat_grad", b.grad, a.grad)
        _check_same(what + " stats", b.stats, a.stats)


@pytest.mark.parametrize("n", [1, 300, 2049])
@pytest.mark.parametrize("D", [2, 32, 64])
@pytest.mark.parametrize("mode", [0, 1])
def test_gauss_grad_exchange_is_gauss_grad(mode, D, n):
    """GaussKernelOps.policy_grad_exchange (r4_gauss_grad into [np + 5], then r4_grad_exchange_n with G = 1) against
    r4_gauss_grad: bit for bit, one launch more (the exchange)."""
    import torch
    from rl4rs_b200.trainer import GaussKernelOps
    pol, data = _gauss_setup(D, n, seed=D + n + mode)
    if mode == 1:
        data = (data[0], data[1], None, None, None, data[5], data[6])
    hp = R.PG_HP[mode]
    inv_n, stat_scale = (1.0 / n if mode == 0 else 1.0), 1.0 / n
    a = GaussKernelOps(D, pol.flat.device, pol.n_params)
    b = GaussKernelOps(D, pol.flat.device, pol.n_params)
    for ops in (a, b):
        ops.stats.copy_(torch.tensor([0.5, -1.0, 0.25, 2.0, 3.0]))
    _, la = _launched(lambda: a.policy_grad(mode, pol.flat, data, None, 0, n, hp, inv_n, stat_scale))
    with _comm(pol.n_params) as comm:
        _, lb = _launched(lambda: b.policy_grad_exchange(comm, mode, pol.flat, data, n, hp, inv_n, stat_scale))
    what = "a2c gauss mode%d D%d n%d" % (mode, D, n)
    assert lb == la + 1 == 2 * -(-n // 2048) + 1, (what, la, lb)
    _check_same(what + " flat_grad", b.grad, a.grad)
    _check_same(what + " stats", b.stats, a.stats)


# ---- A5: IMPALA -------------------------------------------------------------------------------------------------------
IMPALA_CASES = [(False, 284, 9, 7), (False, 512, 2, 1), (False, 149, 36, 7), (True, 32, 2, 7), (True, 32, 9, 4096)]


@pytest.mark.parametrize("clip", [0.0, 10.0])
@pytest.mark.parametrize("conti,size,T,B", IMPALA_CASES)
def test_impala_step_with_comm_is_the_single_gpu_step(conti, size, T, B, clip):
    """r4_impala_step / r4_gauss_impala_step with the world-1 communicator against NULL, from the same warm moments:
    params, m, v, flat_grad, stats, logp, value, vs and pg_adv bit for bit.  The mask policy's exchange replaces
    k_grad_reduce (the same count); the Gaussian step adds it (one more)."""
    import torch
    from test_gpu_trainer_impala import HP, _hp_tuple, _setup, _warm, _work
    pol, ops, buf, _, _ = _setup(conti, size, T, B, seed=size + T + B)
    _warm(ops, pol)
    hp = _hp_tuple(HP, not (conti and T == 2))
    flat0, m0, v0, step0 = pol.flat.detach().clone(), ops.m.clone(), ops.v.clone(), ops.step
    runs = []
    for comm_on in (False, True):
        with torch.no_grad():
            pol.flat.copy_(flat0)
        ops.m.copy_(m0); ops.v.copy_(v0); ops.step = step0
        ops.stats.fill_(0.75); ops.grad.fill_(-2.0)
        work = _work(T, B)
        with _comm(pol.n_params) as comm:
            _, launches = _launched(lambda: ops.impala_step(comm if comm_on else None, pol.flat, buf, hp, 1e-3, clip, work))
        runs.append((launches, (pol.flat.detach().clone(), ops.m.clone(), ops.v.clone(), ops.grad.clone(), ops.stats.clone())
                     + work))
    (l0, r0), (l1, r1) = runs
    what = "impala %s %d T%d B%d clip%g" % ("gauss" if conti else "mask", size, T, B, clip)
    assert l1 == l0 + (1 if conti else 0), (what, l0, l1)
    for name, a, b in zip(("params", "m", "v", "flat_grad", "stats", "logp", "value", "vs", "pg_adv"), r1, r0):
        _check_same("%s %s" % (what, name), a, b)
    assert not _same(r0[0], flat0)


# ---- A6: the replay learners ------------------------------------------------------------------------------------------
def _replay_state(tk):
    rb = tk.replay
    return [tk.policy.flat, tk.policy.target, tk.ops.m, tk.ops.v, tk.ops.stats] + \
        ([rb.prio, rb.max_prio] if rb.prio is not None else [])


def _replay_pair(tk, step):
    """Runs step(comm) from the same state with comm None and with a world-1 communicator -> (launches, state) each."""
    import torch
    state0 = [t.detach().clone() for t in _replay_state(tk)]
    out = []
    for comm_on in (False, True):
        with torch.no_grad():
            for t, t0 in zip(_replay_state(tk), state0):
                t.copy_(t0)
        with _comm(tk.policy.n_params) as comm:
            _, launches = _launched(lambda: step(comm if comm_on else None))
        out.append((launches, [t.detach().clone() for t in _replay_state(tk)]))
    return out


DDPG_STEP_CASES = [("DDPG", True, 1), ("DDPG", False, 3), ("TD3", False, 0), ("TD3", True, 2)]


@pytest.mark.parametrize("algo,prio,actor_step", DDPG_STEP_CASES)
def test_ddpg_train_step_with_comm_is_the_single_gpu_step(algo, prio, actor_step):
    """r4_ddpg_train_step with the world-1 communicator against NULL (DDPG and TD3, actor_step 0 and > 0, prioritized
    replay on and off): params, target, m, v, stats, priorities and max_prio bit for bit; one launch more (the exchange
    into the scratch's second gradient)."""
    from test_gpu_trainer_ddpg import _fill, _pair
    tk, _ = _pair(algo, prioritized_replay=prio, train_batch_size=64)
    _fill((tk,))
    assert (tk.replay.prio is not None) == prio
    u, noise = tk.draws()
    hp = tk._hp()
    (l0, s0), (l1, s1) = _replay_pair(tk, lambda comm: tk.ops.train_step(comm, tk.policy, tk.replay, u, noise, actor_step, 4,
                                                                         hp))
    what = "ddpg_step %s prio%d a%d" % (algo, prio, actor_step)
    assert l0 == (5 if prio else 4) and l1 == l0 + 1, (what, l0, l1)
    for name, a, b in zip(("params", "target", "m", "v", "stats", "prio", "max_prio"), s1, s0):
        _check_same("%s %s" % (what, name), a, b)


@pytest.mark.parametrize("copy", [0, 1])
@pytest.mark.parametrize("prio", [True, False])
def test_rainbow_train_step_with_comm_is_the_single_gpu_step(prio, copy):
    """r4_rainbow_train_step with the world-1 communicator against NULL (prioritized replay on and off, copy_target on
    and off): params, target, m, v, stats, priorities and max_prio bit for bit; one launch more."""
    from test_gpu_trainer_rainbow import _fill, _pair
    tk, _ = _pair(prioritized_replay=prio, train_batch_size=64)
    _fill((tk,))
    assert (tk.replay.prio is not None) == prio
    (u,) = tk.draws()
    hp = tk._hp()
    (l0, s0), (l1, s1) = _replay_pair(tk, lambda comm: tk.ops.train_step(comm, tk.policy, tk.replay, u, 3, bool(copy), hp))
    what = "rainbow_step prio%d copy%d" % (prio, copy)
    assert l0 == (5 if prio else 4) and l1 == l0 + 1, (what, l0, l1)
    for name, a, b in zip(("params", "target", "m", "v", "stats", "prio", "max_prio"), s1, s0):
        _check_same("%s %s" % (what, name), a, b)


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_comm_create_and_open_refuse_bad_arguments():
    """r4_comm_create: world 0 and 17, rank -1 and rank = world, n_params 0, out NULL -> R4_ERR_ARG with *out untouched;
    r4_comm_open with a handle count other than world or no handles -> R4_ERR_ARG; r4_comm_destroy(NULL) is a no-op.
    None of them launches a learner kernel."""
    import torch
    lib = _lib()

    def edges():
        for rank, world, n in ((0, 0, 10), (0, 17, 10), (-1, 2, 10), (2, 2, 10), (0, 1, 0)):
            h = C.c_void_p(0x5eed)
            assert lib.r4_comm_create(rank, world, n, C.byref(h)) == R4_ERR_ARG, (rank, world, n)
            assert h.value == 0x5eed, (rank, world, n)
        assert lib.r4_comm_create(0, 1, 10, None) == R4_ERR_ARG
        with _comm(10, world=2) as comm:
            blob = (C.c_uint8 * 64)()
            assert lib.r4_comm_open(comm.h, blob, 1) == R4_ERR_ARG
            assert lib.r4_comm_open(comm.h, blob, 3) == R4_ERR_ARG
            assert lib.r4_comm_open(comm.h, None, 2) == R4_ERR_ARG
        lib.r4_comm_destroy(None)
    _, launches = _launched(edges)
    assert launches == 0
    torch.cuda.synchronize()


class _Refusal(object):
    """One entry point called with a given communicator through the product's own ctypes front (rl4rs_b200.trainer),
    its return code captured instead of raised, and the buffers it may write."""

    def __init__(self, ops, n_params, call, written, canaried):
        self.ops, self.n_params, self.call, self.written = ops, n_params, call, written
        import torch
        g = torch.Generator(device="cuda").manual_seed(11)
        for t in canaried:                           # a value no kernel would leave there
            t.copy_(torch.randn(t.shape, generator=g, device="cuda") * 1e3 + 7.25)

    def run(self, comm):
        codes = []
        step = getattr(self.ops, "step", None)       # the epoch front adds the return code to its step count
        self.ops._check = lambda rc, what: codes.append(rc)
        rc = self.call(comm)
        if step is not None and codes:
            self.ops.step = step
        return codes[0] if codes else rc


def _refusal(entry):
    import torch
    from rl4rs_b200.trainer import GaussKernelOps, KernelOps
    lib = _lib()
    dev = torch.device("cuda")
    if entry in ("ppo_epoch_dist", "grad_exchange", "grad_exchange_n"):
        A, n = 284, 64
        pol, data = _mask_setup(A, n, seed=1)
        ops = KernelOps(A, dev, pol.n_params)
        flat = pol.flat.detach().clone()
        perm = torch.arange(n, device=dev)
        bufs = [flat, ops.m, ops.v, ops.grad, ops.stats, ops.scratch]
        call = {
            "ppo_epoch_dist": lambda comm: ops.ppo_epoch_dist(comm, flat, data, perm, n, 16, R.PG_HP[0], 1e-3),
            "grad_exchange": lambda comm: lib.r4_grad_exchange(comm.h, _p(ops.scratch), 3, A, _p(ops.grad), _p(ops.stats), 1.0,
                                                               _stream()),
            "grad_exchange_n": lambda comm: ops._exchange(comm, ops.scratch, 3, 1.0)}[entry]
        return _Refusal(ops, pol.n_params, call, bufs, bufs[1:])
    if entry == "gauss_ppo_epoch_dist":
        D, n = 32, 64
        pol, data = _gauss_setup(D, n, seed=1)
        ops = GaussKernelOps(D, dev, pol.n_params)
        flat = pol.flat.detach().clone()
        perm = torch.arange(n, device=dev)
        bufs = [flat, ops.m, ops.v, ops.grad, ops.stats, ops.scratch]
        return _Refusal(ops, pol.n_params, lambda comm: ops.ppo_epoch_dist(comm, flat, data, perm, n, 16, R.PG_HP[0], 1e-3),
                        bufs, bufs[1:])
    if entry in ("impala_step", "gauss_impala_step"):
        from test_gpu_trainer_impala import HP, _hp_tuple, _setup, _work
        conti = entry == "gauss_impala_step"
        T, B = 9, 7
        pol, ops, buf, _, _ = _setup(conti, 32 if conti else 284, T, B, seed=2)
        work = _work(T, B)
        bufs = [pol.flat, ops.m, ops.v, ops.grad, ops.stats, ops.scratch, ops.norm] + list(work)
        return _Refusal(ops, pol.n_params,
                        lambda comm: ops.impala_step(comm, pol.flat, buf, _hp_tuple(HP, True), 1e-3, 10.0, work),
                        bufs, bufs[1:])
    if entry == "ddpg_train_step":
        from test_gpu_trainer_ddpg import _fill, _pair
        tk, _ = _pair("DDPG", prioritized_replay=True, train_batch_size=64)
        _fill((tk,))
        u, noise = tk.draws()
        hp = tk._hp()
        bufs = [tk.policy.flat, tk.policy.target, tk.ops.m, tk.ops.v, tk.ops.stats, tk.ops.scratch, tk.replay.prio,
                tk.replay.max_prio]
        return _Refusal(tk.ops, tk.policy.n_params,
                        lambda comm: tk.ops.train_step(comm, tk.policy, tk.replay, u, noise, 1, 1, hp), bufs,
                        [tk.ops.m, tk.ops.v, tk.ops.stats, tk.ops.scratch])
    assert entry == "rainbow_train_step"
    from test_gpu_trainer_rainbow import _fill, _pair
    tk, _ = _pair(prioritized_replay=True, train_batch_size=64)
    _fill((tk,))
    (u,) = tk.draws()
    hp = tk._hp()
    bufs = [tk.policy.flat, tk.policy.target, tk.ops.m, tk.ops.v, tk.ops.stats, tk.ops.scratch, tk.replay.prio,
            tk.replay.max_prio]
    return _Refusal(tk.ops, tk.policy.n_params, lambda comm: tk.ops.train_step(comm, tk.policy, tk.replay, u, 1, True, hp),
                    bufs, [tk.ops.m, tk.ops.v, tk.ops.stats, tk.ops.scratch])


ENTRIES = ("ppo_epoch_dist", "gauss_ppo_epoch_dist", "grad_exchange", "grad_exchange_n", "impala_step", "gauss_impala_step",
           "ddpg_train_step", "rainbow_train_step")


@pytest.mark.parametrize("why", ["unopened", "other_n_params"])
@pytest.mark.parametrize("entry", ENTRIES)
def test_refusal_launches_and_writes_nothing(entry, why):
    """Each entry point given a world-2 communicator that was created and never opened (rank 0 here; no peer is mapped,
    so nothing could wait) returns R4_ERR_STATE, and given a world-1 communicator made for one parameter more returns
    R4_ERR_ARG: no learner launch, every output and scratch buffer (canary-filled where the call may write) unchanged.
    A correct communicator then runs the same call (the refusal is the communicator's, not the arguments')."""
    import torch
    r = _refusal(entry)
    torch.cuda.synchronize()
    before = [t.detach().clone() for t in r.written]
    if why == "unopened":
        cm, want = _comm(r.n_params, world=2, rank=0), R4_ERR_STATE
    else:
        cm, want = _comm(r.n_params + 1), R4_ERR_ARG
    with cm as comm:
        rc, launches = _launched(lambda: r.run(comm))
    assert rc == want, (entry, why, rc, _err())
    assert launches == 0, (entry, why, launches)
    for k, (a, b) in enumerate(zip(r.written, before)):
        assert _same(a, b), (entry, why, "buffer %d written" % k)
    with _comm(r.n_params) as comm:
        rc, launches = _launched(lambda: r.run(comm))
    assert rc >= 0 and launches > 0, (entry, rc, _err())


# ---- several ranks ----------------------------------------------------------------------------------------------------
# One process per GPU (torch.multiprocessing spawn, a file:// process group under tmp_path), each rank set up through
# trainer.PeerComm.  Hang safety: every rank makes the same exchanges in the same order (shapes, step counts and G
# schedules are functions of the case alone); no check raises between two exchanges (a failed comparison is recorded
# and the rank carries on); each phase starts with a timed host barrier that every rank reaches only after its data and
# setup return codes are in hand; refusals are made only where the host decides them, and alike on every rank; the
# parent kills and reaps every rank past DEADLINE, and each rank logs the last call it entered.
MAX_WORLD = 8
DEADLINE = 900.0
LR = 1e-3


class _Rank(object):
    """One rank's view: its device, the host (gloo) group for timed barriers, its failures and comparison maxima."""

    def __init__(self, rank, world, out_dir):
        import torch
        import torch.distributed as dist
        self.rank, self.world, self.dist = rank, world, dist
        self.dev = torch.device("cuda", rank)
        self.log = open(os.path.join(out_dir, "%d.log" % rank), "w", buffering=1)
        self.host = dist.new_group(backend="gloo")
        self.failures, self.cmp = [], {}

    def note(self, msg):
        self.log.write(msg + "\n")

    def check(self, what, fn):
        """fn() with any exception recorded as a failure of `what` (never raised: the peers keep to the schedule)."""
        try:
            fn()
        except Exception as exc:
            self.failures.append("%s: %s: %s" % (what, type(exc).__name__, str(exc)[:400]))

    def barrier(self, ok=True):
        """All ranks agree that every rank got here with ok; a timed host barrier follows.  -> the agreement."""
        import datetime
        import torch
        flag = torch.tensor([1 if ok else 0])
        self.dist.all_reduce(flag, op=self.dist.ReduceOp.MIN, group=self.host)
        self.dist.monitored_barrier(group=self.host, timeout=datetime.timedelta(seconds=300))
        return bool(flag.item())

    def gather(self, t):
        if self.world == 1:
            return [t]
        every = [torch_empty_like(t) for _ in range(self.world)]
        self.dist.all_gather(every, t.contiguous())
        return every

    def comm(self, n):
        """A ready communicator for n parameters: trainer.PeerComm from two ranks on, a world-1 one alone."""
        if self.world == 1:
            return Comm(n)
        from rl4rs_b200.trainer import PeerComm
        return PeerComm(n, self.dev)

    def same(self, key, got, want):
        """Bit identity of got and want, recorded under key (max |diff|, max |want|, count)."""
        d = float((got.double() - want.double()).abs().max()) if got.numel() else 0.0
        r = float(want.double().abs().max()) if want.numel() else 0.0
        c = self.cmp.setdefault(key, [0.0, 0.0, 0])
        c[0], c[1], c[2] = max(c[0], d), max(c[1], r), c[2] + got.numel()
        if not _same(got, want):
            self.failures.append("%s: max |diff| %.3g" % (key, d))

    def replicas(self, key, tensors):
        """Every tensor bit-identical to rank 0's."""
        for name, t in tensors:
            every = self.gather(t.detach())
            self.same("%s replicas %s" % (key, name), t, every[0])


def torch_empty_like(t):
    import torch
    return torch.empty_like(t)


def _union(ctx, data, lo, hi):
    """Rows [lo, hi) of every rank's columns, concatenated in rank order (None columns stay None)."""
    import torch
    return tuple(None if x is None else torch.cat(ctx.gather(x[lo:hi].contiguous())) for x in data)


def _screened(ref_fn, pool, n, ctx, what):
    """The first n rows of the pool whose decisions are clear under ref_fn's reference (all n, recorded, if too few)."""
    import torch
    clear = ref_fn(pool).clear()
    sel = torch.nonzero(clear).reshape(-1)[:n]
    if sel.numel() < n:
        ctx.failures.append("%s: only %d clear rows of %d" % (what, sel.numel(), clear.numel()))
        sel = torch.arange(n, device=clear.device)
    return tuple(None if x is None else x[sel].contiguous() for x in pool)


def _adam_check(ctx, what, p0, g, m0, v0, step, flat, m, v, clip=0.0, rel_g=0.0):
    """params, m and v within optim_ref64.adam's bounds from the kernel's own gradient g and the previous state; with
    clip, the global-norm clip of g (the summed gradient's norm) first."""
    import optim_ref64 as O
    from test_gpu_optim_shapes import _cmp
    c = lambda t: t.detach().float().cpu().numpy()
    g64, _, on = O.global_clip(c(g), 1.0, clip)
    st = O.adam(c(p0), g64, c(m0), c(v0), step, LR, rel_g=2 * O.U + (O.sumsq_rel(g.numel(), 1024) if on else 0.0) + rel_g)
    ctx.check(what + " adam p", lambda: _cmp("%s p" % what, c(flat), st.p, st.bp))
    ctx.check(what + " adam m", lambda: _cmp("%s m" % what, c(m), st.m, st.bm))
    ctx.check(what + " adam v", lambda: _cmp("%s v" % what, c(v), st.v, st.bv))
    return on


# C1 / C6 ---------------------------------------------------------------------------------------------------------------
def _mr_sizes():
    lib = _lib()
    return (1, 257, lib.r4_policy_num_params(284), lib.r4_rainbow_num_params(284, 8))


def _mr_G(rank, k, sms):
    return 1 + (7 * k + 5 * rank) % min(sms, 64)


def _phase_raw(ctx):
    """Four live communicators, forty interleaved calls with G varying between calls and ranks: flat_grad = the
    rank-order float32 sum of the all-gathered per-rank partial sums on every rank, stats_accum this rank's statistics
    only (one fma at scale 1/3); then a parameter-count mismatch refused alike on every rank, and the exchanges after it
    still exact (the refusal did not advance the step count)."""
    import torch
    from rl4rs_b200 import _capi
    lib = _lib()
    sms = torch.cuda.get_device_properties(ctx.dev).multi_processor_count
    sizes = _mr_sizes()
    comms = [ctx.comm(n) for n in sizes]
    flats = [torch.zeros(n, device=ctx.dev) for n in sizes]
    stats = [torch.zeros(5, device=ctx.dev) for _ in sizes]
    want_stats = [np.zeros(5, np.float32) for _ in sizes]
    scale = SCALES[2]
    if not ctx.barrier(all(c.ok for c in comms)):
        ctx.failures.append("raw: a communicator is not ready")
        return
    st = C.c_void_p(torch.cuda.current_stream(ctx.dev).cuda_stream)

    def exchange(k, s):
        n, G = sizes[s], _mr_G(ctx.rank, k, sms)
        gen = torch.Generator(device=ctx.dev).manual_seed(1000003 * ctx.rank + 1009 * s + k)
        part = _partials(G, n, gen)
        ctx.note("raw call %d size %d G %d" % (k, s, G))
        rc = lib.r4_grad_exchange_n(comms[s].h, _capi.ptr(part), G, n, _capi.ptr(flats[s]), _capi.ptr(stats[s]), scale, st)
        if rc != 0:
            ctx.failures.append("raw call %d: rc %d" % (k, rc))
        torch.cuda.synchronize(ctx.dev)
        every = ctx.gather(_csum(part[:G * n].view(G, n)))
        want = torch.zeros(n, device=ctx.dev)
        for r in range(ctx.world):
            want = want + every[r]
        want_stats[s] = _fma32(_csum(part[G * n:].view(G, 5)).cpu().numpy(), np.full(5, scale, np.float32), want_stats[s])
        ctx.same("raw flat", flats[s], want)
        ctx.same("raw stats", stats[s], torch.from_numpy(want_stats[s]).to(ctx.dev))

    for k in range(CALLS):
        for s in ((k + j) % len(sizes) for j in range(len(sizes))):
            exchange(k, s)
    ctx.note("raw refusal")
    rc = lib.r4_grad_exchange_n(comms[1].h, _capi.ptr(flats[0]), 1, sizes[0], _capi.ptr(flats[0]), None, 1.0, st)
    if rc != R4_ERR_ARG:
        ctx.failures.append("raw: the mismatch refusal returned %d" % rc)
    ctx.barrier()
    for k in range(CALLS, CALLS + 4):
        for s in range(len(sizes)):
            exchange(k, s)
    for c in comms:
        c.close()


# C2 / C3 ---------------------------------------------------------------------------------------------------------------
def _policy_case(ctx, kind, size, mode, n, seed):
    """-> (policy, ops, hyper-parameters, float64 reference function, a pool of candidate rows for this rank): the
    policy is the same on every rank, the rows are the rank's own."""
    import torch
    from rl4rs_b200.policy import GaussianPolicy, MaskedPolicy
    from rl4rs_b200.trainer import GaussKernelOps, KernelOps
    dev = ctx.dev
    mask = kind == "mask"
    pol = (MaskedPolicy if mask else GaussianPolicy)(size, dev, seed=3)
    with torch.no_grad():
        pol.flat.add_((0.05 if mask else 0.02) * torch.randn(pol.n_params, generator=torch.Generator().manual_seed(4)).to(dev))
    ops = (KernelOps if mask else GaussKernelOps)(size, dev, pol.n_params)
    pool = (R.mask_batch if mask else R.gauss_batch)(pol, max(256, n + n // 10 + 16), size, dev, seed=seed + 7919 * ctx.rank)
    return pol, ops, R.PG_HP[mode], (R.policy_grad if mask else R.gauss_grad), pool


def _kernel_cols(kind, mode, rows):
    if kind == "gauss" and mode == 1:
        return (rows[0], rows[1], None, None, None, rows[5], rows[6])
    return rows


def _epoch_case(ctx, kind, size, mb):
    """C2 / C3: two single-step calls of the data-parallel epoch, then one two-step call from the same state."""
    import torch
    import optim_ref64 as O
    from test_gpu_learner_shapes import _check_grad, _check_stats
    W, steps = ctx.world, 2
    n = steps * mb
    what = "%s epoch-dist %d mb%d" % ("policy" if kind == "mask" else "gauss", size, mb)
    pol, ops, hp, grad_fn, pool = _policy_case(ctx, kind, size, 0, n, seed=size + mb)
    inv_union = 1.0 / (mb * W)
    data = _screened(lambda rows: grad_fn(pol, pol.flat, 0, *rows, hp, inv_union), pool, n, ctx, what)
    m0, v0 = (torch.from_numpy(x).to(ctx.dev) for x in O.carried(pol.n_params, 5)[1:])
    flat0 = pol.flat.detach().clone()
    perm = torch.arange(n, device=ctx.dev)
    comm = ctx.comm(pol.n_params)
    if not ctx.barrier(comm.ok):
        ctx.failures.append(what + ": communicator not ready")
        return
    flat = flat0.clone()
    ops.m.copy_(m0); ops.v.copy_(v0); ops.step = 0
    for s in range(steps):
        p0, pm, pv = flat.clone(), ops.m.clone(), ops.v.clone()
        ops.stats.zero_()
        ctx.note("%s step %d" % (what, s))
        rc = ops.ppo_epoch_dist(comm, flat, data, perm[s * mb:(s + 1) * mb].contiguous(), mb, mb, hp, LR)
        torch.cuda.synchronize(ctx.dev)
        if rc != 1:
            ctx.failures.append("%s step %d: rc %d" % (what, s, rc))
        union = _union(ctx, data, s * mb, (s + 1) * mb)
        own = tuple(x[s * mb:(s + 1) * mb] for x in data)

        def grad_check():        # (a) the summed gradient over the union at 1 / (mb W)
            r = grad_fn(pol, p0, 0, *union, hp, inv_union)
            if not bool(r.clear().all()):
                ctx.note("%s step %d: a union row is no longer clear; gradient check skipped" % (what, s))
                return
            _check_grad(what, ops.grad, r.grad, pol)

        def stats_check():       # (c) this rank's own statistics at 1 / mb, not rescaled by the world size
            r = grad_fn(pol, p0, 0, *own, hp, 1.0 / mb)
            _check_stats(what, ops.stats.double(), r.stats * (1.0 / mb))
        ctx.check(what + " grad", grad_check)
        _adam_check(ctx, what, p0, ops.grad, pm, pv, s + 1, flat, ops.m, ops.v)          # (b)
        ctx.check(what + " stats", stats_check)
        ctx.replicas(what, (("params", flat), ("m", ops.m), ("v", ops.v), ("flat_grad", ops.grad)))   # (d)
    loop = (flat, ops.m.clone(), ops.v.clone(), ops.grad.clone())
    flat2 = flat0.clone()
    ops.m.copy_(m0); ops.v.copy_(v0); ops.step = 0
    ctx.note("%s one call" % what)
    rc = ops.ppo_epoch_dist(comm, flat2, data, perm, n, mb, hp, LR)
    torch.cuda.synchronize(ctx.dev)
    if rc != steps:
        ctx.failures.append("%s one call: rc %d" % (what, rc))
    for name, a, b in zip(("params", "m", "v", "flat_grad"), (flat2, ops.m, ops.v, ops.grad), loop):
        ctx.same("%s one call = loop %s" % (what.split()[0], name), a, b)
    comm.close()


def _phase_ppo(ctx):
    for A in (2, 284, 512):
        for mb in (1, 256, 257):
            _epoch_case(ctx, "mask", A, mb)


def _phase_gauss(ctx):
    for D in (2, 32, 64):
        for mb in (256, 2049):
            _epoch_case(ctx, "gauss", D, mb)


# C4 --------------------------------------------------------------------------------------------------------------------
def _phase_a2c(ctx):
    """The A2C pairs of both policies: the exchanged gradient against float64 over the union at inv_n = 1, then Adam with
    the clip at half the union gradient's norm (engaged: the global norm clips), replicas bit-identical."""
    import torch
    from test_gpu_learner_shapes import _check_grad
    for kind, size in (("mask", 284), ("mask", 2), ("gauss", 32)):
        n = 300
        what = "%s a2c-dist %d" % ("policy" if kind == "mask" else "gauss", size)
        pol, ops, hp, grad_fn, pool = _policy_case(ctx, kind, size, 1, n, seed=size + 11)
        data = _screened(lambda rows: grad_fn(pol, pol.flat, 1, *rows, hp, 1.0), pool, n, ctx, what)
        union = _union(ctx, data, 0, n)
        r = grad_fn(pol, pol.flat, 1, *union, hp, 1.0)
        clip = torch.tensor([0.5 * float(r.grad.norm())])
        if ctx.world > 1:
            ctx.dist.all_reduce(clip, op=ctx.dist.ReduceOp.MIN, group=ctx.host)
        clip = float(clip)
        comm = ctx.comm(pol.n_params)
        if not ctx.barrier(comm.ok):
            ctx.failures.append(what + ": communicator not ready")
            return
        p0, m0, v0 = pol.flat.detach().clone(), ops.m.clone(), ops.v.clone()
        ctx.note(what)
        ctx.check(what + " call", lambda: ops.policy_grad_exchange(comm, 1, pol.flat, _kernel_cols(kind, 1, data), n, hp, 1.0,
                                                                   1.0 / n))
        torch.cuda.synchronize(ctx.dev)
        ctx.check(what + " grad", lambda: _check_grad(what, ops.grad, r.grad, pol))
        ops.adam(pol.flat, LR, 1.0, clip)
        torch.cuda.synchronize(ctx.dev)
        if not _adam_check(ctx, what, p0, ops.grad, m0, v0, ops.step, pol.flat, ops.m, ops.v, clip=clip):
            ctx.failures.append(what + ": the clip did not engage")
        ctx.replicas(what, (("params", pol.flat), ("m", ops.m), ("v", ops.v), ("flat_grad", ops.grad)))
        comm.close()


def _phase_impala(ctx):
    """r4_impala_step / r4_gauss_impala_step: V-trace rank-local against vtrace64 on this rank's episodes, the exchanged
    gradient against the rank-order sum of the per-rank float64 references, the clip on the global norm, replicas equal."""
    import torch
    from test_gpu_learner_shapes import TOL, _check_grad, _cmp
    from test_gpu_trainer_impala import HP, _hp_tuple, _setup, _warm, _work, impala_ref
    for conti, size, T, B in ((False, 284, 9, 64), (True, 32, 9, 64)):
        what = "%s impala-dist %d" % ("gauss" if conti else "policy", size)
        pol, ops, buf, inputs, action = _setup(conti, size, T, B, seed=101 + ctx.rank)
        if ctx.world > 1:
            ctx.dist.broadcast(pol.flat.data, 0)             # one learner; each rank's behaviour policy is its own
        _warm(ops, pol)
        flat0, m0, v0 = pol.flat.detach().clone(), ops.m.clone(), ops.v.clone()
        ref = impala_ref(pol, flat0, inputs, action, buf.logp, buf.reward, T, B, HP, True)
        refs = ctx.gather(ref["grad"].double().contiguous())
        g64 = refs[0].clone()
        for x in refs[1:]:
            g64 = g64 + x
        clip = 0.5 * float(g64.norm())
        comm = ctx.comm(pol.n_params)
        if not ctx.barrier(comm.ok):
            ctx.failures.append(what + ": communicator not ready")
            return
        work = _work(T, B)
        ops.stats.zero_()
        ctx.note(what)
        ctx.check(what + " call", lambda: ops.impala_step(comm, pol.flat, buf, _hp_tuple(HP, True), LR, clip, work))
        torch.cuda.synchronize(ctx.dev)
        k = (T - 1) * B
        vs, pg = work[2].reshape(-1), work[3].reshape(-1)
        vscale = max(1.0, float(ref["vs"].abs().max()))
        ctx.check(what + " vs", lambda: _assert_le1(_cmp(what + " vs", vs[:k], ref["vs"], TOL * vscale)))
        ctx.check(what + " pg_adv", lambda: _assert_le1(_cmp(what + " pg_adv", pg[:k], ref["pg"], TOL * vscale)))
        ctx.check(what + " grad", lambda: _check_grad(what, ops.grad, g64, pol))
        if not _adam_check(ctx, what, flat0, ops.grad, m0, v0, ops.step, pol.flat, ops.m, ops.v, clip=clip):
            ctx.failures.append(what + ": the clip did not engage")
        ctx.replicas(what, (("params", pol.flat), ("m", ops.m), ("v", ops.v), ("flat_grad", ops.grad)))
        comm.close()


def _assert_le1(q):
    assert q <= 1, q


# C5 --------------------------------------------------------------------------------------------------------------------
def _phase_replay(ctx):
    """r4_ddpg_train_step (DDPG, TD3) and r4_rainbow_train_step, each rank with its own replay and draws: params, target, m,
    v (and the priorities) equal, bit for bit, r4_ddpg_apply / r4_rainbow_apply (grad_scale 1) applied to the rank-order
    float32 sum of the ranks' r4_ddpg_grad / r4_rainbow_grad at inv_n = 1 / (n W) over the same indices; replicas equal."""
    import torch
    W = ctx.world
    for algo in ("DDPG", "TD3", "RAINBOW"):
        if algo == "RAINBOW":
            from test_gpu_trainer_rainbow import _fill, _pair
            tk, _ = _pair(train_batch_size=64 * W)
        else:
            from test_gpu_trainer_ddpg import _fill, _pair
            tk, _ = _pair(algo, prioritized_replay=algo == "DDPG", train_batch_size=64 * W)
        pol, ops, rb = tk.policy, tk.ops, tk.replay
        if W > 1:
            ctx.dist.broadcast(pol.flat.data, 0)
            ctx.dist.broadcast(pol.target, 0)
        _fill((tk,), seed=31 + ctx.rank)
        draws = tk.draws()
        hp = tk._hp()
        n = draws[0].numel()
        inv = float(np.float32(1.0) / np.float32(n * W))
        state = lambda: [pol.flat, pol.target, ops.m, ops.v, ops.stats] + ([rb.prio, rb.max_prio] if rb.prio is not None else [])
        names = ("params", "target", "m", "v", "stats", "prio", "max_prio")
        s0 = [t.detach().clone() for t in state()]
        comm = ctx.comm(pol.n_params) if W == 1 else tk.comm
        if not ctx.barrier(comm is not None and comm.ok):
            ctx.failures.append(algo + ": communicator not ready")
            return
        ctx.note(algo + " train step")
        if algo == "RAINBOW":
            ctx.check(algo + " step", lambda: ops.train_step(comm, pol, rb, draws[0], 3, True, hp))
        else:
            ctx.check(algo + " step", lambda: ops.train_step(comm, pol, rb, draws[0], draws[1], 1, 2, hp))
        torch.cuda.synchronize(ctx.dev)
        got = [t.detach().clone() for t in state()]
        ctx.replicas(algo, (("params", pol.flat), ("target", pol.target), ("m", ops.m), ("v", ops.v)))
        with torch.no_grad():
            for t, t0 in zip(state(), s0):
                t.copy_(t0)
        idx, w = ops.replay_sample(rb, draws[0], hp["beta"])
        weights = w if rb.prio is not None else None
        if algo == "RAINBOW":
            ops.grad_(pol, rb, idx, weights, hp["gamma_n"], inv)
        else:
            ops.grad_(pol, rb, idx, weights, draws[1], hp, inv)
        total = torch.zeros_like(ops.grad)
        for g in ctx.gather(ops.grad.clone()):
            total = total + g
        ops.grad.copy_(total)
        if algo == "RAINBOW":
            ops.apply(pol, 3, hp, True)
        else:
            ops.apply(pol, 1, 2, hp, 1.0)
        if rb.prio is not None:
            ops.replay_priorities(rb, idx, ops.td, hp["eps"])
        torch.cuda.synchronize(ctx.dev)
        for name, a, b in zip(names, got, state()):
            ctx.same("%s step = apply(sum of grads) %s" % (algo, name), a, b)
        if W == 1:
            comm.close()


# C7 --------------------------------------------------------------------------------------------------------------------
# The peer path and the NCCL path differ only in the order of the ranks' float32 gradient sums, so the two runs' Adam
# updates differ at most where a gradient element's rounding moves m_hat / sqrt(v_hat).  No order-free bound of that
# exists for Adam near g = 0 (the update is lr sign(g) at step 1), so the bound stated is the whole reach of both runs:
# each Adam step moves an element by at most lr (1 - b1) / sqrt(1 - b2) (Kingma & Ba 2015, section 2.1, the case
# 1 - b1 > sqrt(1 - b2) of torch's defaults: 3.17 lr), so after S steps from equal parameters |p_peer - p_nccl| <=
# 2 * 3.17 * lr * S per element.  The losses must agree within 1e-3 relative.
ADAM_REACH = (1 - 0.9) / math.sqrt(1 - 0.999)


def _phase_trainers(ctx):
    import torch
    from rl4rs_b200.trainer import get_rl_model
    from test_gpu_parity import _synthetic, make_env
    W, B = ctx.world, 64
    for algo in ("PPO", "A2C", "PPO_conti", "A2C_conti"):
        conti = algo.endswith("_conti")
        runs = {}
        for path in ("peer", "nccl"):
            if path == "nccl":
                os.environ["R4_NO_PEER_COMM"] = "1"
            else:
                os.environ.pop("R4_NO_PEER_COMM", None)
            flags = {"support_conti_env": True} if conti else {"support_rllib_mask": True}
            cfg, cat, log, w = _synthetic(B, False, is_eval=False, cache_size=4 * B, **flags)
            env = make_env(cfg, False, cat, log, w, output_format="torch", device=ctx.rank)
            env.seed(ctx.rank)
            np.random.seed(ctx.rank)
            tr = get_rl_model(algo, {"sgd_minibatch_size": 64 * W} if algo.startswith("PPO") else {}, env=env)
            flat0 = tr.policy.flat.detach().clone()
            ctx.barrier()
            ctx.note("%s %s" % (algo, path))
            st = [tr.train() for _ in range(2)]
            torch.cuda.synchronize(ctx.dev)
            uses = bool(tr.comm is not None and tr.comm.ok)
            if uses != (path == "peer"):
                ctx.failures.append("%s %s: peer path taken %s" % (algo, path, uses))
            ctx.replicas("%s %s" % (algo, path), (("params", tr.policy.flat),))
            steps = sum(int(s.get("sgd_steps", 1)) for s in st)
            runs[path] = (tr.policy.flat.detach().clone(), st[-1]["total_loss"], steps, flat0)
            if tr.comm is not None:
                tr.comm.close()
        os.environ.pop("R4_NO_PEER_COMM", None)
        (fp, lp, sp, f0), (fn, ln, _, _) = runs["peer"], runs["nccl"]
        lr = float(tr.config["lr"])
        bound = 2 * ADAM_REACH * lr * sp
        diff = float((fp - fn).abs().max())
        c = ctx.cmp.setdefault("%s peer vs nccl params (bound %.3g)" % (algo, bound), [0.0, 0.0, 0])
        c[0], c[1], c[2] = max(c[0], diff), bound, c[2] + fp.numel()
        if not diff <= bound:
            ctx.failures.append("%s: peer vs nccl params differ by %.3g > %.3g" % (algo, diff, bound))
        if not abs(lp - ln) <= 1e-3 * abs(ln):
            ctx.failures.append("%s: losses %.6g (peer) vs %.6g (nccl)" % (algo, lp, ln))
        if not float((fp - f0).abs().max()) > 0:
            ctx.failures.append("%s: the parameters did not move" % algo)


PHASES = {"raw": _phase_raw, "ppo": _phase_ppo, "gauss": _phase_gauss, "a2c": _phase_a2c, "impala": _phase_impala,
          "replay": _phase_replay, "trainers": _phase_trainers}


def _mr_worker(rank, world, init_file, out_dir, phases):
    """One rank: the phases in order; writes <rank>.json (failures, comparison maxima, margin rows) and <rank>.log."""
    import json
    import sys
    import torch
    import torch.distributed as dist
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for d in (root, os.path.join(root, "tests")):
        if d not in sys.path:
            sys.path.insert(0, d)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method="file://" + init_file, rank=rank, world_size=world,
                            device_id=torch.device("cuda", rank))
    ctx = _Rank(rank, world, out_dir)
    try:
        for ph in phases:
            ctx.note("phase " + ph)
            PHASES[ph](ctx)
        ctx.note("done")
    except Exception as exc:
        ctx.failures.append("%s: %s" % (type(exc).__name__, exc))
    finally:
        with open(os.path.join(out_dir, "%d.json" % rank), "w") as f:
            json.dump({"rank": rank, "failures": ctx.failures, "cmp": ctx.cmp, "margins": golden_util.MARGINS}, f)
        ctx.log.close()
        dist.destroy_process_group()


def _visible_peers():
    """-> (GPU count, None) when every pair of visible GPUs can map each other, else (count, why not)."""
    import torch
    k = torch.cuda.device_count()
    if k < 2:
        return k, "%d visible CUDA device%s; the data-parallel exchange needs two or more" % (k, "" if k == 1 else "s")
    for a in range(k):
        for b in range(k):
            if a != b and not torch.cuda.can_device_access_peer(a, b):
                return k, "%d visible CUDA devices, but device %d cannot map device %d" % (k, a, b)
    return k, None


def _worlds():
    import torch
    k = min(torch.cuda.device_count(), MAX_WORLD)
    return sorted({2, 3, k} & set(range(2, k + 1)))


def _run_ranks(world, phases, tmp_path):
    import json
    import time
    import torch.multiprocessing as mp
    ctx = mp.start_processes(_mr_worker, args=(world, str(tmp_path / "init"), str(tmp_path), phases), nprocs=world,
                             join=False, start_method="spawn")
    t0 = time.time()
    try:
        while not ctx.join(timeout=5):
            if time.time() - t0 > DEADLINE:
                last = {}
                for r in range(world):
                    p = tmp_path / ("%d.log" % r)
                    last[r] = p.read_text().splitlines()[-1:] if p.exists() else []
                pytest.fail("world %d did not finish within %d s; last call entered per rank: %s" % (world, DEADLINE, last))
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.terminate()
        for p in ctx.processes:
            p.join(10)
            if p.is_alive():
                p.kill()
                p.join()
    return [json.load(open(tmp_path / ("%d.json" % r))) for r in range(world)]


def _judge(world, res):
    """Margin rows (one per comparison key and world, the ranks merged) and every rank's failures."""
    for r in res:
        for key, (diff, ref, count) in r["cmp"].items():
            bound = ref if "bound" in key else max(float(np.spacing(np.float32(ref))), 1e-45)
            golden_util.record_margin("comm w%d %s" % (world, key), np.array([diff]), np.array([bound]), np.array([ref]))
        for key, m in r["margins"].items():
            k = "comm w%d %s" % (world, key)
            have = golden_util.MARGINS.setdefault(k, dict(m, n=0))
            have["n"] += m["n"]
            for f in ("floored_err_over_bound", "plain_rel_max"):
                have[f] = max(have[f], m[f])
    bad = [(world, r["rank"], r["failures"][:6]) for r in res if r["failures"]]
    assert not bad, bad


def _multi_rank(tmp_path, phases):
    k, why = _visible_peers()
    if why:
        pytest.skip(why)
    for world in _worlds():
        d = tmp_path / ("w%d" % world)
        d.mkdir()
        _judge(world, _run_ranks(world, phases, d))


def test_multi_rank_raw_exchange_and_refusal(tmp_path):
    """C1 and C6 at world 2, 3 and every visible GPU up to 8 (see _phase_raw)."""
    _multi_rank(tmp_path, ("raw",))


def test_multi_rank_learners(tmp_path):
    """C2 - C5: both PPO epochs, the A2C pairs and IMPALA steps of both policies, the DDPG / TD3 / RAINBOW steps."""
    _multi_rank(tmp_path, ("ppo", "gauss", "a2c", "impala", "replay"))


def test_multi_rank_trainers(tmp_path):
    """C7: PPO, A2C, PPO_conti and A2C_conti on the CUDA env, two iterations on the peer path and on the NCCL fallback."""
    _multi_rank(tmp_path, ("trainers",))


def test_rank_checks_in_one_process(tmp_path):
    """The multi-rank checks C1 - C5 run by the same harness with one rank (a world-1 communicator on GPU 0): their
    references, restatements and bounds are exercised wherever one GPU is, though the sums span one rank only."""
    _judge(1, _run_ranks(1, ("raw", "ppo", "gauss", "a2c", "impala", "replay"), tmp_path))
