"""GPU: the simulator-training kernels (csrc/r4_simtrain.cuh) against the float64 reference of tests/simtrain_ref.py at the
shapes the C-ABI accepts, beyond the one hash size of test_gpu_simtrain.py.

  gradient grid   n = 1, 8, 9, 63, 64, 65 at H = 9 (every embedding run mixes the two sequences and the query slots;
                  the 8-sample recurrence CTAs and 64-row GEMM tiles cut at every edge), n = 256, 1024, 4096 at H = 100 000,
                  n = 65, 2049 at H = 4 000 000 (radix keys of 14 / 18 / 23 bits; the sequence and head weights near offset
                  1.03e9).  The reference runs on the GPU in torch float64 over the compacted tables of the ids a batch
                  touches; every other embedding row of the kernel's gradient must be exactly zero over the whole table.
  eval / metrics  r4_simtrain_eval's probabilities, and its f64 accumulator against simtrain.Metrics on the same
                  probabilities; r4_simtrain_grad's accumulator at drop rate 0 equal to eval's bit for bit
  chained steps   r4_simtrain_step equal to r4_simtrain_grad + r4_simtrain_apply bit for bit; after a step the next gradient
                  into the same buffer matches the reference and holds no row of the previous batch
  dropout draw    keep_out equal to the NumPy restatement of the counter-based draw; a supplied keep_in is used and returned
  rejections      every out-of-range argument returns R4_ERR_ARG and writes nothing

Bound, as in test_gpu_simtrain.py: max |g - ref| <= 1e-4 max |ref| per tensor, 1e-3 for the attention MLPs and emb_cat.
Every comparison is recorded as a `simtrain ... n... H...` row of the margin report.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import simtrain_ref as R  # noqa: E402
from golden_util import assert_close_rel, record_margin  # noqa: E402

from rl4rs_b200 import _capi, simtrain, synth  # noqa: E402

pytestmark = pytest.mark.gpu

TOL, TOL_CANCEL = 1e-4, 1e-3          # test_gpu_simtrain.py states why the attention MLPs and emb_cat get 1e-3
MAXH, MAXN = 4000000, 4096
ERR_ARG = -1
KINDS = ("default", "stress")
SEED, COUNTER = 5, 77
# (H, n, weights, drop rate)
GRID = ([(9, n, k, r) for n in (1, 8, 9, 63, 64, 65) for k in KINDS for r in (0.0, 0.2)]
        + [(100000, 256, "default", 0.2), (100000, 1024, "default", 0.2)]
        + [(100000, 4096, "default", 0.0), (100000, 4096, "default", 0.2), (100000, 4096, "stress", 0.0)]
        + [(MAXH, 65, k, r) for k in KINDS for r in (0.0, 0.2)]
        + [(MAXH, 2049, "default", 0.2), (MAXH, 2049, "stress", 0.0)])
# records of each hash size's sample store (9 samples per record: enough for the largest n drawn from it)
RECORDS = {9: 120, 3000: 120, 100000: 600, MAXH: 300}


def _lib():
    return _capi.load_library()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _ok(rc, what):
    if rc != 0:
        raise AssertionError("%s failed (%d): %s" % (what, rc, (_lib().r4_last_error(None) or b"?").decode()))


_STORES, _WEIGHTS = {}, {}


def _store(H):
    if H not in _STORES:
        _STORES[H] = R.make_edge_samples(RECORDS[H], H, seed=H % 1000 + 1)
    return _STORES[H]


def _weights(kind, H):
    """The W-table at H; at the maximum H only its dense tensors are used (from H = 9)."""
    Hw = 9 if H == MAXH else H
    if (kind, Hw) not in _WEIGHTS:
        cfg = {"category_hash_size": Hw}
        _WEIGHTS[(kind, Hw)] = (synth.make_weights(cfg, seed=21, bounded_scores=True) if kind == "default" else
                                synth.make_weights(cfg, seed=22, stress=2.0, bias_noise=0.1, bounded_scores=True))
    return _WEIGHTS[(kind, Hw)]


class _Data(object):
    """A sample store on the device and its r4_simtrain_data."""

    def __init__(self, samples):
        self.ts = [torch.from_numpy(np.ascontiguousarray(getattr(samples, k))).cuda() for k in simtrain.ItemSamples.FIELDS]
        self.d = _capi.SimTrainData(*[t.data_ptr() for t in self.ts])


def _offsets(H):
    out, o = {}, 0
    for name, shape in simtrain.layer_plan({"category_hash_size": H}):
        out[name] = (o, shape)
        o += int(np.prod(shape))
    return out


def _device_params(w, H, ids=None):
    """The kernel's f32 flat parameters at H on the device: w's tensors, or with ids, w's compact embedding tables (one row
    per id) written at rows ids of otherwise zero tables -- the maximum H without a host copy of its 10^9 parameters."""
    prm = torch.zeros(R.num_params(H), dtype=torch.float32, device="cuda")
    for name, (o, shape) in _offsets(H).items():
        v = torch.from_numpy(np.ascontiguousarray(w[name], dtype=np.float32)).cuda()
        k = int(np.prod(shape))
        if ids is not None and name.startswith("emb_"):
            prm[o:o + k].view(H, -1)[torch.from_numpy(ids).cuda()] = v
        else:
            prm[o:o + k] = v.reshape(-1)
    return prm


_MAXH_ROWS, _CLEAR = {}, {}
# A sample is clear when its float64 probabilities are at least CLEAR from 0 and 1, 100x the 1e-6 every row of a case must
# keep after dropout.  The stress weights make confident predictions: measured over each store, the filter leaves out
# 11 of 1080 samples at H = 9, 793 of 5400 at H = 100 000 and 21 of 2700 at the maximum H (none with the default weights).
CLEAR, MAX_DROP = 1e-4, 0.2


def _max_rows(s):
    """At the maximum H, the embedding rows of every id the store reads (ids ascending, emb_cat rows, emb_seq rows)."""
    if "rows" not in _MAXH_ROWS:
        ids = R.compact(s, np.arange(len(s)))[0]
        rs = np.random.RandomState(31)
        _MAXH_ROWS["rows"] = (ids, rs.uniform(-0.05, 0.05, (len(ids), R.E)).astype(np.float32),
                              rs.uniform(-0.05, 0.05, (len(ids), R.E)).astype(np.float32))
    return _MAXH_ROWS["rows"]


def _compact_w(H, kind, s, ids):
    w = _weights(kind, H)
    if H != MAXH:
        return R.compact_weights(w, ids)
    all_ids, ec, es = _max_rows(s)
    pos = np.searchsorted(all_ids, ids)
    return dict(w, emb_cat=ec[pos], emb_seq=es[pos])


def _clear(H, kind):
    """The store's samples whose float64 probabilities (no dropout) are at least CLEAR from 0 and 1: the loss clip is the
    gradient's one discrete decision, so rows near it are left out rather than absorbed into the bound."""
    if (H, kind) not in _CLEAR:
        s = _store(H)
        ids, sc, ic = R.compact(s, np.arange(len(s)))
        cfg = {"category_hash_size": len(ids)}
        p = R.ref_probs(cfg, simtrain.flatten(_compact_w(H, kind, s, ids), cfg), sc, ic, device="cuda")
        _CLEAR[(H, kind)] = np.minimum(p, 1 - p).min(1) > CLEAR
        assert (~_CLEAR[(H, kind)]).mean() <= MAX_DROP, (H, kind, "the clip filter left out %d of %d" % (
            int((~_CLEAR[(H, kind)]).sum()), len(s)))
    return _CLEAR[(H, kind)]


def _case(H, n, kind, rate=0.0):
    """-> (samples, idx, compact ids, samples', idx', the compact W-table, device params); idx are n clear samples in a
    seeded order.  With dropout, a sample the kernel's keep bits at its batch position (R.keep_bits) move within CLEAR of
    the clip is replaced by the next clear one."""
    s = _store(H)
    order = np.random.RandomState(n).permutation(len(s))
    pool = order[_clear(H, kind)[order]]
    assert len(pool) >= n, (H, kind, n)
    idx, spare = pool[:n].copy(), list(pool[n:])
    for _ in range(4 if rate > 0 else 0):
        ids, sc, ic = R.compact(s, idx)
        cfg = {"category_hash_size": len(ids)}
        p = R.ref_probs(cfg, simtrain.flatten(_compact_w(H, kind, s, ids), cfg), sc, ic, device="cuda",
                        keep=R.keep_bits(SEED, COUNTER, n, rate), rate=rate)
        near = np.flatnonzero(np.minimum(p, 1 - p).min(1) <= CLEAR)
        if not len(near):
            break
        assert len(near) <= len(spare), (H, kind, n, len(near))
        idx[near], spare = spare[:len(near)], spare[len(near):]
    ids, sc, ic = R.compact(s, idx)
    wc = _compact_w(H, kind, s, ids)
    prm = _device_params(wc, H, ids) if H == MAXH else _device_params(_weights(kind, H), H)
    return s, idx, ids, sc, ic, wc, prm


def _kernel_grad(H, prm, data, idx, rate, keep_in=None, seed=SEED, counter=COUNTER, grad=None, acc=None):
    """One r4_simtrain_grad into grad (default: a new zero buffer) -> (grad, stats, keep bits); the scratch is freed."""
    lib = _lib()
    n = len(idx)
    scratch = torch.empty(lib.r4_simtrain_scratch_size(n), dtype=torch.uint8, device="cuda")
    grad = torch.zeros_like(prm) if grad is None else grad
    keep_out = torch.zeros(n, 256, dtype=torch.uint8, device="cuda")
    stats = torch.zeros(2, dtype=torch.float32, device="cuda")
    ki = None if keep_in is None else torch.from_numpy(keep_in).cuda()
    it = torch.from_numpy(np.asarray(idx, np.int64)).cuda()
    _ok(lib.r4_simtrain_grad(H, _p(prm), C.byref(data.d), _p(it), n, seed, counter, rate, _p(ki), _p(keep_out), _p(scratch),
                             _p(grad), _p(stats), _p(acc), None), "r4_simtrain_grad")
    torch.cuda.synchronize()
    del scratch
    torch.cuda.empty_cache()
    return grad, stats.cpu().numpy(), keep_out.cpu().numpy()


def _check_grad(tag, H, grad, ids, ref):
    """The kernel's gradient (device, layout at H) against the compact reference ref (rows ids), per tensor; every
    embedding row outside ids exactly zero, checked on the device over the whole table."""
    rt = simtrain.unflatten(ref, {"category_hash_size": len(ids)})
    idt = torch.from_numpy(ids).cuda()
    bad = []
    for name, (o, shape) in _offsets(H).items():
        g = grad[o:o + int(np.prod(shape))]
        if name.startswith("emb_"):
            tab = g.view(H, -1)
            stray = (tab != 0).any(1)
            stray[idt] = False
            assert not bool(stray.any()), "%s: %d untouched %s rows are not zero" % (tag, int(stray.sum()), name)
            got = tab[idt].double().cpu().numpy()
        else:
            got = g.double().cpu().numpy().reshape(shape)
        scale = float(np.abs(rt[name]).max())
        err = float(np.abs(got - rt[name]).max())
        bound = (TOL_CANCEL if name.startswith(("att", "emb_cat")) else TOL) * scale
        record_margin("simtrain %s %s" % (name, tag), np.array([err]), np.array([bound + 1e-30]), np.array([scale]))
        if err > bound:
            bad.append((name, err, bound))
    assert not bad, "%s: tensors outside their bound (name, err, bound): %s" % (tag, bad)


def _check_clip(probs):
    assert np.all(np.minimum(probs, 1 - probs) > 1e-7 + 1e-6), "a row is within 1e-6 of the loss clip"


@pytest.mark.parametrize("H,n,kind,rate", GRID)
def test_gradient_parity_grid(H, n, kind, rate):
    s, idx, ids, sc, ic, wc, prm = _case(H, n, kind, rate)
    data = _Data(s)
    grad, stats, keep = _kernel_grad(H, prm, data, idx, rate)
    assert np.array_equal(keep, R.keep_bits(SEED, COUNTER, n, rate))
    cfg = {"category_hash_size": len(ids)}
    loss, ref, probs = R.ref_grad(cfg, simtrain.flatten(wc, cfg), sc, ic, keep if rate > 0 else None, rate, device="cuda")
    _check_clip(probs)
    assert abs(stats[0] - loss) <= 1e-5 * abs(loss) + 1e-6
    _check_grad("n%d H%d %s drop%g" % (n, H, kind, rate), H, grad, ids, ref)
    del grad, prm
    torch.cuda.empty_cache()


def _eval(H, prm, data, idx, acc):
    lib = _lib()
    n = len(idx)
    scratch = torch.empty(lib.r4_simtrain_scratch_size(n), dtype=torch.uint8, device="cuda")
    probs = torch.full((n, 2), -1.0, dtype=torch.float32, device="cuda")
    it = torch.from_numpy(np.asarray(idx, np.int64)).cuda()
    _ok(lib.r4_simtrain_eval(H, _p(prm), C.byref(data.d), _p(it), n, _p(scratch), _p(probs), _p(acc), None), "r4_simtrain_eval")
    torch.cuda.synchronize()
    del scratch
    torch.cuda.empty_cache()
    return probs.cpu().numpy()


def _loss_rows(p, y):
    """Keras's per-row loss from the kernel's float32 probabilities as k_st_loss forms it: 1 - p[c] is the other column."""
    p = np.asarray(p, np.float64)
    yy = np.eye(2)[np.asarray(y, np.int64)]
    pc, qc = np.clip(p, simtrain.CLIP, 1 - simtrain.CLIP), np.clip(p[:, ::-1], simtrain.CLIP, 1 - simtrain.CLIP)
    return -(yy * np.log(pc) + (1 - yy) * np.log(qc)).mean(1)


def _check_acc(tag, acc, m):
    """The device accumulator against Metrics: count, accuracy sum and both AUC histograms exactly, the loss sum (the
    kernel takes log(1 - p) from the other column's exponential) within 1e-6 relative."""
    a = acc.cpu().numpy()
    assert a[2] == m.acc[2] and a[1] == m.acc[1], (tag, a[:3], m.acc[:3])
    assert np.array_equal(a[3:], m.acc[3:]), (tag, np.flatnonzero(a[3:] != m.acc[3:]))
    assert abs(a[0] - m.acc[0]) <= 1e-6 * abs(m.acc[0]), (tag, a[0], m.acc[0])


@pytest.mark.parametrize("n", [1, 65, 4096])
def test_eval_probs_and_metrics(n):
    H = 100000
    s, w = _store(H), _weights("stress", H)
    prm, data = _device_params(w, H), _Data(s)
    idx = np.random.RandomState(n + 1).permutation(len(s))[:n]
    acc = torch.zeros(simtrain.Metrics().acc.size, dtype=torch.float64, device="cuda")
    probs = _eval(H, prm, data, idx, acc)
    ref = R.ref_probs({"category_hash_size": H}, simtrain.flatten(w, {"category_hash_size": H}), s, idx, device="cuda")
    assert_close_rel(probs, ref, what="simtrain eval probs n%d H%d" % (n, H))
    y = s.features(idx)[3]
    m = simtrain.Metrics()
    m.add(probs, y, _loss_rows(probs, y))
    _check_acc("eval n%d" % n, acc, m)
    # the training pass at drop rate 0 runs the same forward and adds the same accumulator
    acc_g = torch.zeros_like(acc)
    _kernel_grad(H, prm, data, idx, 0.0, acc=acc_g)
    assert torch.equal(acc_g, acc)


def test_eval_metrics_over_ragged_batches():
    H = 3000
    s, w = _store(H), _weights("default", H)
    prm, data = _device_params(w, H), _Data(s)
    acc = torch.zeros(simtrain.Metrics().acc.size, dtype=torch.float64, device="cuda")
    m = simtrain.Metrics()
    flat = simtrain.flatten(w, {"category_hash_size": H})
    order = np.random.RandomState(9).permutation(len(s))
    assert len(s) % 256
    for b in range(0, len(s), 256):                          # the last batch is ragged
        idx = order[b:b + 256]
        probs = _eval(H, prm, data, idx, acc)
        assert_close_rel(probs, R.ref_probs({"category_hash_size": H}, flat, s, idx, device="cuda"),
                         what="simtrain eval probs ragged H%d" % H)
        y = s.features(idx)[3]
        m.add(probs, y, _loss_rows(probs, y))
    assert m.acc[2] == len(s)
    _check_acc("ragged", acc, m)


def test_step_equals_grad_then_apply():
    """Three steps of different n: the fused step and the two calls leave the same params, m, v and gradient buffer."""
    lib = _lib()
    H = 3000
    s = _store(H)
    data = _Data(s)
    base = _device_params(_weights("default", H), H)
    A = [base.clone()] + [torch.zeros_like(base) for _ in range(3)]            # params, grad, m, v
    B = [base.clone()] + [torch.zeros_like(base) for _ in range(3)]
    sa, sb = torch.zeros(2, device="cuda"), torch.zeros(2, device="cuda")
    acc_a = torch.zeros(simtrain.Metrics().acc.size, dtype=torch.float64, device="cuda")
    acc_b = torch.zeros_like(acc_a)
    ad = simtrain.ADAM
    scratch = torch.empty(lib.r4_simtrain_scratch_size(65), dtype=torch.uint8, device="cuda")
    for step, n in enumerate((9, 64, 65), 1):
        it = torch.from_numpy(np.random.RandomState(step).permutation(len(s))[:n]).cuda()
        _ok(lib.r4_simtrain_step(H, *(_p(t) for t in A), C.byref(data.d), _p(it), n, SEED, step, 0.2, step, ad["lr"],
                                 ad["beta1"], ad["beta2"], ad["eps"], _p(scratch), _p(sa), _p(acc_a), None), "r4_simtrain_step")
        _ok(lib.r4_simtrain_grad(H, _p(B[0]), C.byref(data.d), _p(it), n, SEED, step, 0.2, None, None, _p(scratch), _p(B[1]),
                                 _p(sb), _p(acc_b), None), "r4_simtrain_grad")
        _ok(lib.r4_simtrain_apply(H, *(_p(t) for t in B), step, ad["lr"], ad["beta1"], ad["beta2"], ad["eps"], None),
            "r4_simtrain_apply")
        torch.cuda.synchronize()
        for what, a, b in zip(("params", "grad", "m", "v", "stats", "acc"), A + [sa, acc_a], B + [sb, acc_b]):
            assert torch.equal(a, b), (step, what)
    assert not torch.equal(A[0], base)


def test_next_gradient_after_a_step_holds_no_stale_rows():
    """A step on a batch whose ids all lie in [1, H/2), then the gradient of a batch whose ids lie in [H/2, H) into the
    same buffer: it matches the reference at the stepped parameters, and the rows of the first batch are exactly zero
    (k_keras_adam cleared what the step wrote; the second pass writes only its own rows)."""
    lib = _lib()
    H = 3000
    lo, hi = R.make_range_samples(40, H, 1, H // 2, seed=6), R.make_range_samples(40, H, H // 2, H, seed=7)
    prm = _device_params(_weights("stress", H), H)
    grad, m, v = (torch.zeros_like(prm) for _ in range(3))
    dlo, dhi = _Data(lo), _Data(hi)
    i_lo = np.random.RandomState(1).permutation(len(lo))[:65]
    i_hi = np.random.RandomState(2).permutation(len(hi))[:64]
    scratch = torch.empty(lib.r4_simtrain_scratch_size(65), dtype=torch.uint8, device="cuda")
    stats = torch.zeros(2, device="cuda")
    ad = simtrain.ADAM
    _ok(lib.r4_simtrain_step(H, _p(prm), _p(grad), _p(m), _p(v), C.byref(dlo.d), _p(torch.from_numpy(i_lo).cuda()), 65, SEED,
                             1, 0.2, 1, ad["lr"], ad["beta1"], ad["beta2"], ad["eps"], _p(scratch), _p(stats), None, None),
        "r4_simtrain_step")
    torch.cuda.synchronize()
    emb = _offsets(H)
    for name in ("emb_cat", "emb_seq"):
        o = emb[name][0]
        assert not grad[o:o + H * R.E].any(), name                 # the step's apply cleared its rows
    _kernel_grad(H, prm, dhi, i_hi, 0.0, grad=grad)
    for name in ("emb_cat", "emb_seq"):
        o = emb[name][0]
        assert not grad[o:o + H // 2 * R.E].any(), name
    ids, sc, ic = R.compact(hi, i_hi)
    assert ids.min() >= H // 2
    wc = R.compact_weights(simtrain.unflatten(prm.cpu().numpy(), {"category_hash_size": H}), ids)
    cfg = {"category_hash_size": len(ids)}
    _, ref, probs = R.ref_grad(cfg, simtrain.flatten(wc, cfg), sc, ic, None, 0.0, device="cuda")
    _check_clip(probs)
    _check_grad("n64 H%d after a step" % H, H, grad, ids, ref)


@pytest.mark.parametrize("seed,counter", [(0, 0), (0, 1), (0, 2 ** 32), (2 ** 64 - 59, 1), (0x9E3779B97F4A7C15, 2 ** 40 + 3)])
def test_keep_out_is_the_counter_draw(seed, counter):
    H = 9
    s = _store(H)
    prm, data = _device_params(_weights("default", H), H), _Data(s)
    idx = np.arange(65)
    for rate in (0.2, 0.5):
        _, _, keep = _kernel_grad(H, prm, data, idx, rate, seed=seed, counter=counter)
        assert np.array_equal(keep, R.keep_bits(seed, counter, 65, rate)), (seed, counter, rate)


def test_keep_in_is_used_and_returned():
    H, n, rate = 9, 65, 0.2
    s, idx, ids, sc, ic, wc, prm = _case(H, n, "stress")
    data = _Data(s)
    keep_in = (np.random.RandomState(4).random_sample((n, 256)) < 0.6).astype(np.uint8)
    grad, _, keep = _kernel_grad(H, prm, data, idx, rate, keep_in=keep_in)
    assert np.array_equal(keep, keep_in)
    cfg = {"category_hash_size": len(ids)}
    _, ref, _ = R.ref_grad(cfg, simtrain.flatten(wc, cfg), sc, ic, keep_in, rate, device="cuda")
    _check_grad("n%d H%d keep_in" % (n, H), H, grad, ids, ref)
    drawn, _, _ = _kernel_grad(H, prm, data, idx, rate)
    o, shape = _offsets(H)["dense_w1"]
    assert not torch.equal(grad[o:o + int(np.prod(shape))], drawn[o:o + int(np.prod(shape))])


class _Sentinels(object):
    """Output buffers filled with sentinels, sized for what a launch over n samples would write."""

    def __init__(self, n, nparams):
        self.grad = torch.full((nparams,), -1234.5, device="cuda")
        self.stats = torch.full((2,), -1234.5, device="cuda")
        self.acc = torch.full((simtrain.Metrics().acc.size,), -1234.5, dtype=torch.float64, device="cuda")
        self.keep = torch.full((max(n, 1), 256), 0xAB, dtype=torch.uint8, device="cuda")
        self.probs = torch.full((max(n, 1), 2), -1234.5, device="cuda")
        self.copy = [t.clone() for t in (self.stats, self.acc, self.keep, self.probs)]

    def untouched(self):
        torch.cuda.synchronize()
        return bool((self.grad == -1234.5).all()) and all(
            torch.equal(a, b) for a, b in zip((self.stats, self.acc, self.keep, self.probs), self.copy))


def _calls(H, n, rate, step, prm, data, out, scratch, it, m, v):
    """The entry points a shape reaches: name -> a call returning the status."""
    lib, ad = _lib(), simtrain.ADAM
    d = C.byref(data)
    return {
        "grad": lambda: lib.r4_simtrain_grad(H, _p(prm), d, _p(it), n, SEED, COUNTER, rate, None, _p(out.keep), _p(scratch),
                                             _p(out.grad), _p(out.stats), _p(out.acc), None),
        "eval": lambda: lib.r4_simtrain_eval(H, _p(prm), d, _p(it), n, _p(scratch), _p(out.probs), _p(out.acc), None),
        "step": lambda: lib.r4_simtrain_step(H, _p(prm), _p(out.grad), _p(m), _p(v), d, _p(it), n, SEED, COUNTER, rate, step,
                                             ad["lr"], ad["beta1"], ad["beta2"], ad["eps"], _p(scratch), _p(out.stats),
                                             _p(out.acc), None),
        "apply": lambda: lib.r4_simtrain_apply(H, _p(prm), _p(out.grad), _p(m), _p(v), step, ad["lr"], ad["beta1"],
                                               ad["beta2"], ad["eps"], None),
    }


def _reject(what, H, n, rate=0.2, step=1, entries=("grad", "eval", "step"), data=None, prm_h=None):
    """Each entry point at this argument set returns R4_ERR_ARG and leaves every output and the parameters as they were.
    The buffers are sized for what a launch at that shape would touch (the layout restatement of simtrain_ref), so even a
    missing check could not write outside them."""
    H_buf = prm_h if prm_h is not None else H
    s = _store(9)
    dd = _Data(s)
    data = data if data is not None else dd.d
    nb = max(n, 1)
    prm = _device_params(_weights("default", 9), 9) if H_buf == 9 else torch.zeros(R.num_params(H_buf), device="cuda")
    p0 = prm.clone() if H_buf < MAXH else None
    out = _Sentinels(n, R.num_params(H_buf))
    scratch = torch.empty(R.scratch_bytes(nb), dtype=torch.uint8, device="cuda")
    it = torch.from_numpy(np.arange(nb) % len(s)).cuda()
    # m and v share the parameters' storage: only the outputs are compared, and one buffer of the maximum H is 4 GB
    calls = _calls(H, n, rate, step, prm, data, out, scratch, it, prm, prm)
    for e in entries:
        assert calls[e]() == ERR_ARG, (what, e)
        assert out.untouched(), (what, e)
        if p0 is not None:
            assert torch.equal(prm, p0), (what, e)
    del prm, out, scratch, p0
    torch.cuda.empty_cache()


def test_rejected_batch_sizes():
    assert R.scratch_bytes(MAXN + 1) > R.scratch_bytes(MAXN)
    _reject("n = 0", 9, 0)
    _reject("n = 4097", 9, MAXN + 1)


def test_rejected_hash_sizes():
    _reject("H = 4000001", MAXH + 1, 65, entries=("grad", "eval", "step", "apply"))
    # at H = 0 the kernels' id clamp has no row to clamp to, so no buffer stands in for what a gather would read; the
    # apply, which touches the flat layout only, is the entry point whose launch there is bounded
    _reject("H = 0", 0, 65, entries=("apply",))


def test_rejected_drop_rates_and_steps():
    for rate in (1.0, float("nan"), -0.1):
        _reject("drop_rate %r" % rate, 9, 65, rate=rate, entries=("grad", "step"))
    _reject("step 0", 9, 65, step=0, entries=("step", "apply"))


def test_rejected_null_data_fields():
    s = _store(9)
    dd = _Data(s)
    for k in simtrain.ItemSamples.FIELDS:
        d = _capi.SimTrainData(*[0 if f == k else t.data_ptr() for f, t in zip(simtrain.ItemSamples.FIELDS, dd.ts)])
        _reject("null %s" % k, 9, 65, data=d)
