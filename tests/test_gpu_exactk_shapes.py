"""GPU: the Exact-K kernels (r4_exactk_*) against the float64 restatement tests/exactk_ref64.py at every seq_length and
batch their C-ABI accepts, tensor by tensor, at one bar: 1e-4 of each tensor's max |ref|.

  generator   T in {9, 31, 32, 33, 64, 65, 255, 256, 257, 284, 500} (the warp-per-row softmax at 32, the 64 x 64 GEMM
              tiles at 64, the 256-thread row loops at 256) at n in {1, 7, 114}; n in {1, 7, 113, 114, 512, 4096} at T = 284
              (the decoder's split-K gains a second partial at n = 114); (4096, 9) and (1321, 500), the largest n the
              n T^2 bound accepts at T = 500.  Dropout 0 / 0.1 / 0.5 and SAMPLE temperature 0.5 / 1 / 2 over the n = 7
              points; the three mask regimes of exactk_ref64.masks_for, with all-masked steps at T = 9, 32 and 33.  At each
              point: the SAMPLE and GREEDY slates, the TRAIN logits and loss, every gradient tensor, and the launch counts.
  large n     at n >= 512 only planted rows carry reward (a row with zero reward adds exactly zero to every gradient):
              the first and last rows, the rows either side of each 64-row tile and each split-K chunk boundary of the
              decoder (9n rows) and the encoder (nT rows), and 32 random rows; the reference runs over them with n_total = n
  critic      n in {1, 7, 1023, 1024, 1025, 2049, 4096}: pred, loss and every tensor's gradient, over rows whose relu
              pre-activations all lie clear of 0
  Adam        both nets at steps 1, 2 and 1000 and two (lr, eps) pairs against TF1's ResourceApplyAdam in float64
  also        two runs at (T 257, n 114, dropout 0.1) are bit-identical; every entry point refuses one step past each edge
              with R4_ERR_ARG, launches nothing and leaves its canary-filled outputs untouched

Worst err / bound per group (bound: BAR times the tensor's max |ref|), measured on an H100 80GB HBM3 at a 700 W power
limit: generator gradients 0.11 (g_w_q at (1321, 500)), TRAIN logits 0.020, loss 0.0009; critic pred 0.058, gradients
0.010, loss 0.010; Adam 0.010.  The module runs in about 25 s there and peaks at 50.6 GB of device memory.  Before the
all-masked CE fix every point with an all-masked step missed its loss bar (by 217 to 6939 times).
"""
import numpy as np
import pytest
import torch

import golden_util
from rl4rs_b200 import _capi
from rl4rs_b200 import exactk as ek

import exactk_ref64 as ref

pytestmark = pytest.mark.gpu

BAR = 1e-4
GREEDY_GAP, CDF_GAP, MASK_GAP = 1e-4, 1e-5, 1e-4
DECODE, GRAD, CRITIC_PRED, CRITIC_TRAIN = 122, 349, 5, 27
EK_KC, EK_SPLITS = 1024, 128                        # split-K: rows per partial at least, partials at most (r4_learn.cu)

REGIME = {9: "sparse", 32: "sparse", 31: "ones", 64: "ones", 256: "ones"}          # the rest: the env's own masks
T_GRID = [9, 31, 32, 33, 64, 65, 255, 256, 257, 284, 500]
POINTS = ([(n, T, REGIME.get(T, "slate"), 0.1, (1.0,)) for n in (1, 114) for T in T_GRID] +
          [(7, T, REGIME.get(T, "slate"), (0.1, 0.0, 0.5)[i % 3], (0.5, 1.0, 2.0)) for i, T in enumerate(T_GRID)] +
          [(7, 9, "ones", 0.1, (1.0,)), (7, 9, "slate", 0.1, (1.0,)), (7, 32, "slate", 0.1, (1.0,))] +
          [(113, 284, "slate", 0.1, (1.0,)), (512, 284, "slate", 0.1, (1.0,)), (4096, 284, "slate", 0.1, (1.0,)),
           (4096, 9, "sparse", 0.1, (1.0,)), (ek.MAX_NTT // 250000, 500, "slate", 0.1, (1.0,))])
PLANT_FROM = 512


@pytest.fixture(autouse=True)
def _release():
    yield
    torch.cuda.empty_cache()


def _gen(T, regime, rate, seed=3):
    m = ref.masks_for(T, regime).numpy()
    g = ek.Generator(m[0], m[1], m[2], m[3], seq_length=T, device="cuda", seed=seed, dropout_rate=rate)
    rng = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        for k, v in g.params().items():
            if "ln" in k:
                v += 0.1 * torch.randn(v.shape, device="cuda", generator=rng)
    return g


def _splits(R):
    S = min(EK_SPLITS, (R + EK_KC - 1) // EK_KC)
    return S, (R + S - 1) // S


def planted_rows(n, T, k=32, seed=0):
    """The first and last rows, both sides of each 64-row tile and of each split-K chunk boundary of the decoder (rows
    t n + b over the nine steps) and of the encoder (rows b T + t), and k random rows."""
    s = {0, n - 1}
    for b in range(64, n, 64):
        s |= {b - 1, b}
    S, kc = _splits(9 * n)
    for j in range(1, S):
        b = (j * kc) % n
        s |= {b - 1, b}
    S, kc = _splits(n * T)
    for j in range(1, S):
        b = (j * kc) // T
        s |= {b - 1, b, b + 1}
    s |= set(np.random.RandomState(seed).choice(n, k, replace=False).tolist())
    return torch.tensor(sorted(x for x in s if 0 <= x < n), dtype=torch.int64, device="cuda")


def _record(key, err, bound, want):
    golden_util.record_margin("exactk " + key, err, bound, want)
    return float(np.max(err / bound)) if np.size(err) else 0.0


def _cmp(key, got, want, scale=None):
    got, want = got.detach().double().reshape(-1), want.detach().double().to(got.device).reshape(-1)
    scale = max(float(want.abs().max()) if scale is None else scale, 1e-30)
    return _record(key, (got - want).abs().cpu().numpy(), BAR * scale, want.cpu().numpy())


def _launches(lib, fn):
    c0 = lib.r4_exactk_launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, lib.r4_exactk_launch_count() - c0


def _check_paths(tag, g, user, rows, mode, temperature):
    lib = _capi.load_library()
    g.temperature = temperature
    (path, _), k = _launches(lib, lambda: g.draw(user, mode))
    assert k == DECODE, (tag, k)
    want, margin, mm, dead = ref.ref_decode(g.flat, user, g.masks, mode, g.seed, g.call, g.rate, temperature, rows)
    ok = (margin > (CDF_GAP if mode == ek.SAMPLE else GREEDY_GAP)) & (mm > MASK_GAP)
    m = rows.numel()
    print("%s mode %d temp %g: %d of %d rows near a decision, %d all-masked steps" %
          (tag, mode, temperature, int((~ok).sum()), m, int(dead.sum())))
    assert int((~ok).sum()) <= max(2, m // 4), tag
    assert torch.equal(path[rows][ok], want[ok]), tag
    return path, dead[ok]


def _point(n, T, regime, rate, temps):
    tag = "n%d T%d %s r%g" % (n, T, regime, rate)
    torch.manual_seed(n * 1000 + T)
    lib = _capi.load_library()
    g = _gen(T, regime, rate)
    user = torch.randn(n, 256, device="cuda")
    rows = planted_rows(n, T) if n >= PLANT_FROM else torch.arange(n, device="cuda")
    dead_seen = 0
    for temp in temps:
        _, dead = _check_paths(tag, g, user, rows, ek.SAMPLE, temp)
        dead_seen += int(dead.sum())
    path, dead = _check_paths(tag, g, user, rows, ek.GREEDY, 1.0)
    dead_seen += int(dead.sum())
    if regime == "sparse" or (regime == "slate" and T < 149):
        assert dead_seen > 0, tag                          # all-masked steps are compared, not skipped
    # TRAIN: reward only on the compared rows clear of a key / query mask decision
    call = g.call + 1
    w64 = ref.unflat64(g.flat)
    mm = torch.cat([ref.mask_margin(w64, user[r].double(), g.seed, call, g.rate, T, r) for r in ref.chunks(rows, T)])
    reward = torch.zeros(n, device="cuda")
    reward[rows] = torch.randn(rows.numel(), device="cuda") * (mm > MASK_GAP)
    (grad, loss), k = _launches(lib, lambda: g.grad(user, path, reward))
    assert k == GRAD, (tag, k)
    keep = ref.device_relu_decisions(g, n)
    got_logits = torch.empty(n, 9, T, device="cuda")
    tgt = path.to(torch.int32).contiguous()
    _, k = _launches(lib, lambda: _capi.check(lib, None, lib.r4_exactk_decode(
        _capi.ptr(g.flat), _capi.ptr(user), n, T, _capi.ptr(g.masks), ek.TRAIN, 1.0, g.seed, call, g.rate, _capi.ptr(tgt),
        _capi.ptr(got_logits), _capi.ptr(g._scr(n)), _capi.stream(g.device)), "r4_exactk_decode"))
    assert k == DECODE, (tag, k)
    want_grad, want_loss, lgs = ref.grad_rows(g.flat, user, g.masks, path, reward, g.seed, call, g.rate, rows, n, keep)
    q = {}
    wl = torch.cat([lg for _, lg in lgs])
    gl = got_logits[rows].double()
    live = wl > ref.NEG / 2
    assert torch.equal(live, gl > ref.NEG / 2), tag
    assert bool((gl[~live] == np.float32(ref.NEG)).all()), tag
    q["logits"] = _cmp("logits " + tag, gl[live], wl[live])
    ce = -torch.log_softmax(wl, -1).gather(2, path[rows].unsqueeze(2)).squeeze(2).sum(1)
    loss_scale = float((reward[rows].double().abs() * ce).sum()) / n
    q["loss"] = _cmp("loss " + tag, loss, torch.tensor([want_loss]), loss_scale)
    for name, (err, scale) in ref.tensor_errors(grad, want_grad).items():
        q["grad " + name] = _record("grad %s %s" % (tag, name), np.array([err]), np.array([BAR * max(scale, 1e-30)]),
                                    np.array([scale]))
    worst = sorted(q.items(), key=lambda kv: -kv[1])[:4]
    print("%s: err / bound, worst: %s" % (tag, ", ".join("%s %.2g" % kv for kv in worst)))
    assert worst[0][1] <= 1, (tag, worst)


@pytest.mark.parametrize("n,T,regime,rate,temps", POINTS)
def test_generator_matches_float64(n, T, regime, rate, temps):
    _point(n, T, regime, rate, temps)


def test_two_runs_are_bit_identical():
    n, T = 114, 257
    out = []
    for _ in range(2):
        torch.manual_seed(0)
        g = _gen(T, "slate", 0.1)
        user = torch.randn(n, 256, device="cuda")
        path, lg = g.draw(user, ek.SAMPLE)
        grad, loss = g.grad(user, path, torch.randn(n, device="cuda"))
        out.append((path, lg, grad, loss))
    assert all(torch.equal(a, b) for a, b in zip(*out))


def _critic_pool(d, n):
    """n rows whose relu pre-activations (float64) all lie at least 1e-5 of their layer's rms from 0, from a pool of
    rows; fewer than 10 % of the pool are dropped."""
    w = ek.unflatten(d.flat.double(), ek.critic_shapes())
    pool = torch.randn(int(n * 1.25) + 8, 256, device="cuda", dtype=torch.float64)
    x, clear = pool, torch.ones(pool.shape[0], dtype=torch.bool, device="cuda")
    for i in (1, 2, 3):
        z = x @ w["w%d" % i] + w["b%d" % i]
        clear &= (z.abs() > 1e-5 * z.pow(2).mean().sqrt()).all(1)
        x = torch.relu(z)
    assert float(clear.double().mean()) > 0.9
    return pool[clear][:n].float().contiguous()


@pytest.mark.parametrize("n", [1, 7, 1023, 1024, 1025, 2049, 4096])
def test_critic_matches_float64(n):
    torch.manual_seed(n)
    lib = _capi.load_library()
    d = ek.Discriminator(device="cuda")
    user = _critic_pool(d, n)
    target = torch.randn(n, device="cuda")
    pred, k = _launches(lib, lambda: d.predict(user))
    assert k == CRITIC_PRED
    (p2, grad, loss), k = _launches(lib, lambda: d._run(user, target))
    assert k == CRITIC_TRAIN
    wp, wg, wl = ref.critic(d.flat, user, target)
    q = {"pred": _cmp("critic pred n%d" % n, pred, wp), "pred2": _cmp("critic pred n%d" % n, p2, wp),
         "loss": _cmp("critic loss n%d" % n, loss, wl.view(1))}
    for name, (err, scale) in ref.tensor_errors(grad, wg, ek.critic_shapes()).items():
        q[name] = _record("critic grad n%d %s" % (n, name), np.array([err]), np.array([BAR * max(scale, 1e-30)]),
                          np.array([scale]))
    print("critic n=%d err / bound: %s" % (n, ", ".join("%s %.2g" % kv for kv in sorted(q.items(), key=lambda kv: -kv[1]))))
    assert max(q.values()) <= 1, q


@pytest.mark.parametrize("net", [ek.GENERATOR, ek.CRITIC])
@pytest.mark.parametrize("lr,eps", [(1e-3, 1e-8), (5e-3, 1e-3)])
@pytest.mark.parametrize("step", [1, 2, 1000])
def test_adam_matches_float64(net, lr, eps, step):
    lib = _capi.load_library()
    gen = torch.Generator(device="cuda").manual_seed(step * 10 + net)
    num = lib.r4_exactk_num_params(net)
    p0 = torch.randn(num, device="cuda", generator=gen) * 0.1
    grad = torch.randn(num, device="cuda", generator=gen)
    m0 = torch.randn(num, device="cuda", generator=gen) * 0.1
    v0 = torch.rand(num, device="cuda", generator=gen) ** 4 * 1e-2        # some v far below eps^2, some above
    p, m, v = p0.clone(), m0.clone(), v0.clone()
    _, k = _launches(lib, lambda: _capi.check(lib, None, lib.r4_exactk_adam(
        net, _capi.ptr(p), _capi.ptr(grad), _capi.ptr(m), _capi.ptr(v), step, lr, 0.9, 0.98, eps, None), "r4_exactk_adam"))
    assert k == 1
    wp, wm, wv = ref.adam64(p0, grad, m0, v0, step, lr, 0.9, 0.98, eps)
    tag = "adam net%d step%d lr%g eps%g" % (net, step, lr, eps)
    q = [_cmp(tag + " update", p.double() - p0.double(), wp - p0.double()), _cmp(tag + " m", m, wm), _cmp(tag + " v", v, wv)]
    assert max(q) <= 1, (tag, q)


def test_rejections_launch_nothing_and_write_nothing():
    lib = _capi.load_library()
    canary = torch.full((1 << 16,), 1234.5, device="cuda")
    n0 = lib.r4_exactk_launch_count()
    got = ref.abi_rejections(lib, _capi.ptr(canary))
    torch.cuda.synchronize()
    assert [x for x in got if x[1] != -1] == []
    assert lib.r4_exactk_launch_count() == n0
    assert bool((canary == 1234.5).all())


def test_peak_device_memory():
    """Runs last in the module: the peak of the module's device memory (the (4096, 284) scratch of 47.4 GB dominates)."""
    peak = torch.cuda.max_memory_allocated()
    print("exactk shapes: peak device memory %.1f GB" % (peak / 1e9))
    assert peak < 70e9
