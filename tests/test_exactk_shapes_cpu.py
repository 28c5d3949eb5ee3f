"""CPU companion of test_gpu_exactk_shapes.py: what its references, planted masks and planted rows must be for the GPU
checks to mean anything, shown without a device.

  rejections      every r4_exactk_* entry point refuses one step past each edge on the host (R4_ERR_ARG, no launch), and
                  r4_exactk_scratch_size returns -1 there, so the GPU module can repeat the calls without launching
  scratch cap     at every T in 9..500 the largest accepted n (n T^2 <= 4096 * 284^2) is accepted with a scratch of at most
                  the documented 47.4 GB, the next n is refused, and the Python front raises ValueError there
  twin            the torch twin equals the float64 reference across the T grid at n <= 7, in all three mask regimes,
                  all-masked steps included (their choice by rule, their CE log T, their zero gradient)
  planted masks   the sparse regime (and the env's own masks below T = 41) give every row an all-masked step
  planted rows    the reference over the reward-carrying rows with n_total = n equals the reference over all rows with zero
                  reward elsewhere to 1e-12, and leaving out one row's contribution misses it by more than 10 times the
                  GPU bar, so the sparse-row check at large n would see a kernel that drops a row
"""
import ctypes as C

import numpy as np
import pytest
import torch

from rl4rs_b200 import _capi
from rl4rs_b200 import exactk as ek

import exactk_ref64 as ref

BAR = 1e-4                               # the GPU module's bar: 1e-4 of each tensor's max |ref|
SCRATCH_CAP = 47.4e9                     # bytes, the documented largest generator scratch (at n = 4096, T = 284)
T_GRID = [9, 31, 32, 33, 64, 65, 255, 256, 257, 284, 500]


def test_rejections_on_the_host():
    lib = _capi.load_library()
    buf = (C.c_char * 64)()
    n0 = lib.r4_exactk_launch_count()
    got = ref.abi_rejections(lib, C.cast(buf, C.c_void_p))
    assert [x for x in got if x[1] != -1] == []
    assert lib.r4_exactk_launch_count() == n0
    assert len(got) == 57


def test_scratch_size_stays_under_the_cap():
    lib = _capi.load_library()
    worst = (0, None)
    for T in range(9, 501):
        n = min(ek.MAXN, ek.MAX_NTT // (T * T))
        size = lib.r4_exactk_scratch_size(ek.GENERATOR, n, T)
        assert 0 < size <= SCRATCH_CAP, (n, T, size)
        worst = max(worst, (size, (n, T)))
        if n < ek.MAXN:
            assert lib.r4_exactk_scratch_size(ek.GENERATOR, n + 1, T) == -1, (n + 1, T)
            with pytest.raises(ValueError, match="seq_length"):
                ek.check_shape(n + 1, T)
        ek.check_shape(n, T)
    assert worst[1] == (4096, 284) and worst[0] > 0.99 * SCRATCH_CAP, worst
    assert lib.r4_exactk_scratch_size(ek.GENERATOR, 1321, 500) > 0 and ek.MAX_NTT // 250000 == 1321
    for n in (1, 7, 4096):
        assert lib.r4_exactk_scratch_size(ek.CRITIC, n, 0) > 0
    with pytest.raises(ValueError, match="1322 rows at seq_length 500"):
        ek.build_nets({"batch_size": 1322, "action_size": 500, "catalog": _Cat()}, torch.device("cpu"))
    g = ek.Generator(*np.ones((4, 500)), seq_length=500, device="cpu")
    with pytest.raises(ValueError, match="seq_length 500"):
        g.draw(torch.zeros(1322, 256))
    with pytest.raises(ValueError, match="seq_length 500"):
        g.grad(torch.zeros(1322, 256), torch.zeros(1322, 9, dtype=torch.long), torch.zeros(1322))


class _Cat(object):
    special_items = [3]


def gen(T, regime, seed=3, rate=0.1, temperature=1.0, device="cpu"):
    """A generator over masks_for(T, regime) with LayerNorm moved off its init (where the second block's key / query
    masks are decided by roundoff)."""
    m = ref.masks_for(T, regime).numpy()
    g = ek.Generator(m[0], m[1], m[2], m[3], seq_length=T, device=device, seed=seed, dropout_rate=rate,
                     temperature=temperature)
    rng = torch.Generator(device=device).manual_seed(seed)
    with torch.no_grad():
        for k, v in g.params().items():
            if "ln" in k:
                v += 0.1 * torch.randn(v.shape, generator=rng, device=device)
    return g


CPU_POINTS = [(T, ("sparse", "ones", "slate")[i % 3], (0.1, 0.0, 0.5)[i % 3], (0.5, 1.0, 2.0)[i % 3])
              for i, T in enumerate(T_GRID)] + [(9, "slate", 0.1, 1.0), (32, "slate", 0.1, 1.0), (9, "ones", 0.1, 1.0)]


@pytest.mark.parametrize("T,regime,rate,temperature", CPU_POINTS)
def test_twin_matches_float64_across_T(T, regime, rate, temperature):
    n = 7 if T <= 284 else 3
    torch.manual_seed(T)
    g = gen(T, regime, rate=rate, temperature=temperature)
    user = torch.randn(n, 256)
    for mode, gap in ((ek.SAMPLE, 1e-5), (ek.GREEDY, 1e-4)):
        path, lg = g.draw(user, mode)
        want, margin, mm, dead = ref.ref_decode(g.flat, user, g.masks, mode, g.seed, g.call, g.rate, temperature)
        ok = (margin > gap) & (mm > 1e-4)
        assert int((~ok).sum()) <= max(2, n // 4)
        assert torch.equal(path[ok], want[ok])
        assert torch.equal(dead, ~(lg > ek.NEG / 2).any(2))         # the twin's all-masked steps are the reference's
    reward = torch.randn(n)
    flat = g.flat.double().clone().requires_grad_(True)
    lg, _ = ek.twin_forward(ek.unflatten(flat, ek.generator_shapes()), user.double(), g.masks, ek.TRAIN, g.seed, g.call,
                            g.rate, target=path)
    loss = ek.policy_loss(lg, path, reward.double())
    loss.backward()
    want_grad, want_loss, _ = ref.generator_grad(g.flat, user, g.masks, path, reward, g.seed, g.call, g.rate)
    assert abs(float(loss.detach()) - float(want_loss)) <= 1e-6 * max(1.0, abs(float(want_loss)))
    for name, (err, scale) in ref.tensor_errors(flat.grad, want_grad).items():
        assert err <= 1e-6 * max(scale, 1e-30), (name, err, scale)
    g.call -= 1                                                          # the same call: the same dropout draws
    _, tl = g.grad(user, path, reward)                                   # the float32 twin: CE log T on all-masked steps
    assert abs(float(tl) - float(want_loss)) <= 1e-4 * max(1.0, abs(float(want_loss)))


@pytest.mark.parametrize("T,regime", [(9, "sparse"), (32, "sparse"), (9, "slate"), (32, "slate"), (100, "sparse")])
def test_planted_masks_give_all_masked_steps(T, regime):
    n = 16
    torch.manual_seed(1)
    g = gen(T, regime)
    user = torch.randn(n, 256)
    for mode in (ek.SAMPLE, ek.GREEDY):
        path, lg = g.draw(user, mode)
        dead = ~(lg > ek.NEG / 2).any(2)
        assert bool(dead.any(1).all()), (mode, dead)
        if regime == "sparse":
            assert bool(dead[:, 8].all())
        # the rule: GREEDY takes 0, SAMPLE the uniform inverse CDF of the row's draw
        rows = torch.arange(n).unsqueeze(1).expand(n, 9)[dead]
        steps = torch.arange(9).unsqueeze(0).expand(n, 9)[dead]
        want = torch.stack([ref.dead_pick(mode, g.seed, g.call, r.view(1), int(t), T, 1.0)[0] for r, t in zip(rows, steps)])
        assert torch.equal(path[dead], want)
        if mode == ek.SAMPLE:
            assert len(set(want.tolist())) > 1


def _planted_case(n=20, T=32):
    torch.manual_seed(5)
    g = gen(T, "sparse")
    user = torch.randn(n, 256)
    path, _ = g.draw(user, ek.GREEDY)
    rows = torch.tensor([0, 9, 10, 19])
    reward = torch.zeros(n)
    reward[rows] = torch.randn(rows.numel())
    return g, user, path, reward, rows


def test_planted_rows_equal_the_full_reference():
    g, user, path, reward, rows = _planted_case()
    n = user.shape[0]
    full, fl, _ = ref.generator_grad(g.flat, user, g.masks, path, reward, g.seed, g.call, g.rate)
    part, pl, _ = ref.grad_rows(g.flat, user, g.masks, path, reward, g.seed, g.call, g.rate, rows, n)
    assert abs(pl - float(fl)) <= 1e-12 * abs(float(fl))
    for name, (err, scale) in ref.tensor_errors(part, full).items():
        assert err <= 1e-12 * max(scale, 1e-300), (name, err, scale)


def test_a_missing_row_misses_by_ten_bars():
    """Leave out one reward-carrying row -- the first, an interior one at a 64-row-tile-like boundary pair, or the last
    (the row a short last tile or split-K partial holds) -- and the worst tensor misses by more than 10 GPU bars."""
    g, user, path, reward, rows = _planted_case()
    n = user.shape[0]
    full, _, _ = ref.grad_rows(g.flat, user, g.masks, path, reward, g.seed, g.call, g.rate, rows, n)
    for drop in range(rows.numel()):
        keep = torch.cat([rows[:drop], rows[drop + 1:]])
        part, _, _ = ref.grad_rows(g.flat, user, g.masks, path, reward, g.seed, g.call, g.rate, keep, n)
        worst = max(err / max(scale, 1e-30) for err, scale in ref.tensor_errors(part, full).values())
        print("without row %d: worst tensor misses by %.0f bars" % (int(rows[drop]), worst / BAR))
        assert worst >= 10 * BAR, int(rows[drop])
    tail = rows[rows < n // 2]                                          # the last half of the batch dropped
    part, _, _ = ref.grad_rows(g.flat, user, g.masks, path, reward, g.seed, g.call, g.rate, tail, n)
    assert max(err / max(scale, 1e-30) for err, scale in ref.tensor_errors(part, full).values()) >= 10 * BAR


def test_adam64_matches_the_cpu_update():
    """The float64 restatement is the update exactk._Adam makes on the CPU (the twin of r4_exactk_adam)."""
    flat = ek.init_critic(1).double()
    opt = ek._Adam(ek.CRITIC, flat.clone(), 0.005)
    m = v = torch.zeros_like(flat)
    p = flat
    for step in range(1, 4):
        gr = torch.randn(flat.shape, dtype=torch.float64)
        opt.apply(gr)
        p, m, v = ref.adam64(p, gr, m, v, step, 0.005)
    assert torch.allclose(opt.flat, p, rtol=0, atol=1e-15) and torch.allclose(opt.m, m) and torch.allclose(opt.v, v)
