"""GPU: the dnn, widedeep and lstm backbones and adversarial_slate on the simulator-training kernels (r4_simtrain_net_*)
against the float64 twins of tests/simtrain_nets_ref.py.

  gradient grid   every valid (net, head) pair: n = 1, 7, 64, 65, 257 at H = 3000 (drop rate 0.2 and 0, default and stress
                  weights), edge samples at H = 9, n = 65 at H = 4 000 000 over the compacted reference.  Every tensor within
                  1e-4 of its largest reference element; every embedding row the batch does not read exactly zero.  lstm:
                  the reference's kink margin above simtrain_nets_ref.KINK_MARGIN in every case, one saturation-heavy
                  case, and the exact-kink case (z-bias 2.5)
  eval / metrics  probabilities against the twin; the accumulator against the host metrics on the kernel's probabilities
  env             the item head's probabilities equal r4_dien_forward's on an env of that algo and the float32 oracle; a
                  checkpoint trained a few steps and saved through the net's plan restores in the env through model_file
  steps           step == grad + apply bit for bit; twenty steps bit-identical; launches per step pinned per pair; net 0
                  equal to the r4_simtrain_head_* entry points bit for bit; rejected pairs write nothing
  learning        teacher-student fits on the GPU
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import simtrain_ref as R  # noqa: E402
import simtrain_nets_ref as NR  # noqa: E402
import simtrain_slate_ref as SR  # noqa: E402
from golden_util import assert_close_rel, record_margin  # noqa: E402

from rl4rs_b200 import _capi, simtrain, synth  # noqa: E402

pytestmark = pytest.mark.gpu

H = 3000
MAXH = 4000000
TOL = 1e-4
SEED, COUNTER = 5, 77
ERR_ARG = -1
NACC = {0: 3 + 2 * 201, 1: simtrain.SlateMetrics.SIZE, 2: simtrain.MulticlassMetrics.SIZE, 3: simtrain.SlateMetrics.SIZE}
# launches per step (grad + apply) and per eval, the radix sort counted once
LAUNCHES = {1: (18, 7), 2: (17, 6), 3: (34, 12), 4: (14, 5)}
_STORES = {}


def _lib():
    return _capi.load_library()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _ok(rc, what):
    if rc != 0:
        raise AssertionError("%s failed (%d): %s" % (what, rc, (_lib().r4_last_error(None) or b"?").decode()))


def _store(Hs, head, records=300, edge=False):
    key = (Hs, bool(head), records, edge)
    if key not in _STORES:
        _STORES[key] = NR.make_samples(records, Hs, head, seed=Hs % 1000 + 3, edge=edge)
    return _STORES[key]


class _Data(object):
    def __init__(self, samples):
        self.ts = [torch.from_numpy(np.ascontiguousarray(getattr(samples, k))).cuda() for k in simtrain.ItemSamples.FIELDS]
        self.d = _capi.SimTrainData(*[t.data_ptr() for t in self.ts])


def _offsets(net, Hs, head):
    out, o = {}, 0
    for name, shape in simtrain.layer_plan(NR.cfg(Hs, head), net):
        out[name] = (o, shape)
        o += int(np.prod(shape))
    return out


def _device_params(net, w, Hs, head, ids=None):
    prm = torch.zeros(NR.num_params(net, Hs, head), dtype=torch.float32, device="cuda")
    for name, (o, shape) in _offsets(net, Hs, head).items():
        v = torch.from_numpy(np.ascontiguousarray(w[name], dtype=np.float32)).cuda()
        k = int(np.prod(shape))
        if ids is not None and name.startswith("emb_"):
            prm[o:o + k].view(Hs, -1)[torch.from_numpy(ids).cuda()] = v
        else:
            prm[o:o + k] = v.reshape(-1)
    return prm


def _grad(net, head, Hs, prm, data, idx, rate, acc=None):
    lib = _lib()
    n = len(idx)
    scratch = torch.empty(lib.r4_simtrain_net_scratch_size(net, head, n), dtype=torch.uint8, device="cuda")
    grad = torch.zeros_like(prm)
    keep = torch.zeros(n, 256, dtype=torch.uint8, device="cuda")
    stats = torch.zeros(2, dtype=torch.float32, device="cuda")
    it = torch.from_numpy(np.asarray(idx, np.int64)).cuda()
    _ok(lib.r4_simtrain_net_grad(net, head, Hs, _p(prm), C.byref(data.d), _p(it), n, SEED, COUNTER, rate, None, _p(keep),
                                 _p(scratch), _p(grad), _p(stats), _p(acc), None), "r4_simtrain_net_grad")
    torch.cuda.synchronize()
    return grad, stats.cpu().numpy(), keep.cpu().numpy()


def _eval(net, head, Hs, prm, data, idx, acc=None):
    lib = _lib()
    n = len(idx)
    scratch = torch.empty(lib.r4_simtrain_net_scratch_size(net, head, n), dtype=torch.uint8, device="cuda")
    probs = torch.full((n, simtrain.CLASSES[head]), -1.0, dtype=torch.float32, device="cuda")
    it = torch.from_numpy(np.asarray(idx, np.int64)).cuda()
    _ok(lib.r4_simtrain_net_eval(net, head, Hs, _p(prm), C.byref(data.d), _p(it), n, _p(scratch), _p(probs), _p(acc), None),
        "r4_simtrain_net_eval")
    torch.cuda.synchronize()
    return probs.cpu().numpy()


def _check_grad(tag, net, head, Hs, grad, ids, ref):
    rt = simtrain.unflatten(ref, NR.cfg(len(ids), head), net)
    idt = torch.from_numpy(ids).cuda()
    bad = []
    for name, (o, shape) in _offsets(net, Hs, head).items():
        g = grad[o:o + int(np.prod(shape))]
        if name.startswith("emb_"):
            tab = g.view(Hs, -1)
            stray = (tab != 0).any(1)
            stray[idt] = False
            assert not bool(stray.any()), "%s: %d untouched %s rows are not zero" % (tag, int(stray.sum()), name)
            got = tab[idt].double().cpu().numpy()
        else:
            got = g.double().cpu().numpy().reshape(shape)
        scale = float(np.abs(rt[name]).max())
        err = float(np.abs(got - rt[name]).max())
        bound = TOL * scale
        record_margin("simtrain net%d head%d %s %s" % (net, head, name, tag), np.array([err]), np.array([bound + 1e-30]),
                      np.array([scale]))
        if err > bound:
            bad.append((name, err, bound))
    assert not bad, "%s: tensors outside their bound (name, err, bound): %s" % (tag, bad)


def _parity(net, head, Hs, s, idx, kind, rate, tag, w=None):
    ids, sc, ic = NR.compact(s, idx, head)
    if w is None:
        w = NR.make_weights(net, 9 if Hs == MAXH else Hs, head, kind)
    if Hs == MAXH:
        rs = np.random.RandomState(31)
        wc = dict(w, **{k: rs.uniform(-0.05, 0.05, (len(ids), 128)).astype(np.float32) for k in ("emb_cat", "emb_seq") if k in w})
        prm = _device_params(net, wc, Hs, head, ids)
    else:
        wc = NR.compact_weights(w, ids)
        prm = _device_params(net, w, Hs, head)
    grad, stats, keep = _grad(net, head, Hs, prm, _Data(s), idx, rate)
    assert np.array_equal(keep, R.keep_bits(SEED, COUNTER, len(idx), rate))
    c = NR.cfg(len(ids), head)
    loss, ref, _, margin = NR.ref_grad(net, head, c, simtrain.flatten(wc, c, net), sc, ic, keep if rate > 0 else None, rate,
                                       device="cuda")
    assert margin > NR.KINK_MARGIN, "%s: a hard-sigmoid argument lies %.3g from a kink" % (tag, margin)
    assert abs(stats[0] - loss) <= 1e-5 * abs(loss) + 1e-6, (stats[0], loss)
    _check_grad(tag, net, head, Hs, grad, ids, ref)
    del grad, prm
    torch.cuda.empty_cache()
    return margin


def _idx(s, head, n, seed):
    return np.random.RandomState(seed).choice(len(s), n, replace=n > len(s)).astype(np.int64)


@pytest.mark.parametrize("net,head", NR.PAIRS)
@pytest.mark.parametrize("n", [1, 7, 64, 65, 257])
def test_gradient_parity(net, head, n):
    s = _store(H, head)
    _parity(net, head, H, s, _idx(s, head, n, n), "default", 0.2, "n%d" % n)
    _parity(net, head, H, s, _idx(s, head, n, n + 1), "stress", 0.0, "n%d stress" % n)


@pytest.mark.parametrize("net,head", NR.PAIRS)
def test_gradient_parity_edges_and_max_hash(net, head):
    s = _store(9, head, records=40, edge=True)
    _parity(net, head, 9, s, _idx(s, head, 30, 2), "default", 0.2, "H9 edge")
    s = _store(MAXH, head, records=80)
    _parity(net, head, MAXH, s, _idx(s, head, 65, 3), "default", 0.2, "H4M")


@pytest.mark.parametrize("head", [0, 1])
def test_lstm_saturated_gates(head):
    s = _store(H, head)
    w = NR.make_weights(3, H, head, "saturate")
    idx = np.random.RandomState((6, 7)[head]).choice(len(s), 4, replace=False)     # seeds whose kink margin is 1.9e-5
    cat, dense, seq, _ = s.features(idx)
    for i in range(2):                                   # the input projection alone clips 5 % of the gate arguments or more
        a = 0.2 * (w["emb_seq"][seq[:, i]].astype(np.float64) @ w["sgru%d_k" % i] + w["sgru%d_b" % i])[..., :256] + 0.5
        assert np.mean((a < 0) | (a > 1)) > 0.05
    _parity(3, head, H, s, idx, None, 0.0, "saturated", w=w)


def test_lstm_exact_kink():
    """Zero GRU kernels, a nonzero candidate bias and every z-bias at 2.5: the z gate's argument is exactly 1 in float32
    (with or without FMA) and float64, z = 1, and the z-bias gradient takes the slope 0.2 (both ends of the clip included)."""
    head = 1
    s = _store(H, head)
    w = NR.make_weights(3, H, head, "default")
    for g in ("cgru", "sgru0", "sgru1"):
        w[g + "_k"] = np.zeros_like(w[g + "_k"])
        w[g + "_rk"] = np.zeros_like(w[g + "_rk"])
        b = np.zeros(384, np.float32)
        b[:128] = 2.5
        b[256:] = 0.3
        w[g + "_b"] = b
    idx = _idx(s, head, 9, 4)
    ids, sc, ic = NR.compact(s, idx, head)
    prm = _device_params(3, w, H, head)
    grad, _, _ = _grad(3, head, H, prm, _Data(s), idx, 0.0)
    c = NR.cfg(len(ids), head)
    _, ref, _, margin = NR.ref_grad(3, head, c, simtrain.flatten(NR.compact_weights(w, ids), c, 3), sc, ic, None, 0.0,
                                    device="cuda")
    assert margin == 0.0
    o = _offsets(3, H, head)
    for g in ("cgru", "sgru0", "sgru1"):
        off = o[g + "_b"][0]
        rb = simtrain.unflatten(ref, c, 3)[g + "_b"]
        kb = grad[off:off + 384].double().cpu().numpy()
        assert np.abs(rb[:128]).max() > 0 and np.abs(kb[:128]).max() > 0, g
        assert np.abs(kb - rb).max() <= TOL * np.abs(rb).max(), g
    # at 2.6 the argument is past the kink: no slope, the z-bias gradient is exactly zero
    for g in ("cgru", "sgru0", "sgru1"):
        w[g + "_b"][:128] = 2.6
    prm = _device_params(3, w, H, head)
    grad, _, _ = _grad(3, head, H, prm, _Data(s), idx, 0.0)
    for g in ("cgru", "sgru0", "sgru1"):
        off = o[g + "_b"][0]
        assert not bool(grad[off:off + 128].any()), g


@pytest.mark.parametrize("net,head", NR.PAIRS)
def test_eval_probs_and_metrics(net, head):
    s = _store(H, head)
    idx = _idx(s, head, 300, 11)
    w = NR.make_weights(net, H, head, "stress")
    prm = _device_params(net, w, H, head)
    acc = torch.zeros(NACC[head], dtype=torch.float64, device="cuda")
    probs = _eval(net, head, H, prm, _Data(s), idx, acc)
    c = NR.cfg(H, head)
    ref = NR.ref_probs(net, head, c, simtrain.flatten(w, c, net), s, idx, device="cuda")
    assert np.abs(probs - ref).max() <= 1e-4, np.abs(probs - ref).max()
    labels = s.features(idx)[3]
    loss = NR.ref_grad(net, head, c, simtrain.flatten(w, c, net), s, idx, None, 0.0, device="cuda")[0]
    m = simtrain.METRICS[head]()
    m.add(probs, labels, np.zeros(len(idx)))
    got = acc.cpu().numpy()
    assert got[2] == len(idx) and abs(got[1] - m.acc[1]) <= 1e-6 * len(idx)
    np.testing.assert_array_equal(got[3:], m.acc[3:])             # histograms and TP / FP / FN (empty for head 2)
    assert abs(got[0] / len(idx) - loss) <= 1e-5 * abs(loss) + 1e-6, (got[0] / len(idx), loss)


def _env_case(net, seq=False, B=8):
    from test_gpu_parity_regimes import _cfg
    algo = simtrain.NET_NAMES[net]
    cfg = dict(_cfg(B, seq), algo=algo, category_hash_size=5000)
    cat = synth.make_catalog()
    log = synth.make_log(4 * B, pages=1, catalog=cat, hash_size=5000)
    return cfg, cat, log


_ORACLES = {1: ("oracle.dnn_np", "DnnOracle"), 2: ("oracle.widedeep_np", "WideDeepOracle"), 3: ("oracle.lstm_np", "LstmOracle")}


def _oracle(net, w, dt):
    import importlib
    mod, cls = _ORACLES[net]
    return getattr(importlib.import_module(mod), cls)(w, dt)


@pytest.mark.parametrize("net", [1, 2, 3])
def test_item_head_matches_env_forward_and_oracle(net):
    from test_gpu_parity import make_env
    Hs = 5000
    cfg, cat, log = _env_case(net)
    w = NR.make_weights(net, Hs, 0, "stress")
    env = make_env(cfg, False, cat, log, w, output_format="numpy")
    s = NR.make_samples(60, Hs, 0, seed=12)
    idx = np.arange(len(s))[:300]
    cf, dense, seq, _ = s.features(idx)
    _, pe = env.sim.engine.dien_forward(seq.astype(np.int32), dense, cf.astype(np.int32))
    prm = _device_params(net, w, Hs, 0)
    pk = _eval(net, 0, Hs, prm, _Data(s), idx)
    po = _oracle(net, w, np.float32).forward(seq, dense, cf)[1]
    assert_close_rel(pk, pe.cpu().numpy(), what="net %d item probs vs env" % net)
    assert_close_rel(pk, po, what="net %d item probs vs f32 oracle" % net)


@pytest.mark.parametrize("net", [1, 2, 3])
def test_trained_checkpoint_restores_in_env(net, tmp_path):
    from test_gpu_parity import make_env
    Hs = 5000
    cfg, cat, log = _env_case(net)
    lib = _lib()
    w = NR.make_weights(net, Hs, 0, "default")
    prm = _device_params(net, w, Hs, 0)
    gr, m, v = torch.zeros_like(prm), torch.zeros_like(prm), torch.zeros_like(prm)
    s = NR.make_samples(60, Hs, 0, seed=13)
    d = _Data(s)
    n = 128
    scratch = torch.empty(lib.r4_simtrain_net_scratch_size(net, 0, n), dtype=torch.uint8, device="cuda")
    for step in range(1, 6):
        idx = torch.from_numpy(_idx(s, 0, n, step)).cuda()
        _ok(lib.r4_simtrain_net_step(net, 0, Hs, _p(prm), _p(gr), _p(m), _p(v), C.byref(d.d), _p(idx), n, SEED, step, 0.2, step,
                                     1e-3, 0.9, 0.999, 1e-7, _p(scratch), None, None, None), "r4_simtrain_net_step")
    torch.cuda.synchronize()
    trained = simtrain.unflatten(prm.cpu().numpy(), NR.cfg(Hs, 0), net)
    assert any(not np.array_equal(trained[k], w[k]) for k in w)
    prefix = str(tmp_path / "model")
    simtrain.SAVERS[net](prefix, trained, NR.cfg(Hs, 0))
    env = make_env(dict(cfg, model_file=prefix), False, cat, log, None, output_format="numpy")
    idx = np.arange(len(s))[:200]
    cf, dense, seq, _ = s.features(idx)
    _, pe = env.sim.engine.dien_forward(seq.astype(np.int32), dense, cf.astype(np.int32))
    po = _oracle(net, trained, np.float32).forward(seq, dense, cf)[1]
    assert_close_rel(pe.cpu().numpy(), po, what="net %d restored env probs vs oracle" % net)


@pytest.mark.parametrize("net,head", NR.PAIRS)
def test_step_is_grad_then_apply_deterministic_and_launches_pinned(net, head):
    lib = _lib()
    s = _store(H, head)
    d = _Data(s)
    w = NR.make_weights(net, H, head, "default")
    base = _device_params(net, w, H, head)
    n = 96
    nacc = NACC[head]

    def run(steps, split):
        prm, g, m, v = base.clone(), torch.zeros_like(base), torch.zeros_like(base), torch.zeros_like(base)
        scratch = torch.empty(lib.r4_simtrain_net_scratch_size(net, head, n), dtype=torch.uint8, device="cuda")
        acc = torch.zeros(nacc, dtype=torch.float64, device="cuda")
        for step in range(1, steps + 1):
            idx = torch.from_numpy(_idx(s, head, n, 100 + step)).cuda()
            if split:
                _ok(lib.r4_simtrain_net_grad(net, head, H, _p(prm), C.byref(d.d), _p(idx), n, SEED, step, 0.2, None, None,
                                             _p(scratch), _p(g), None, _p(acc), None), "grad")
                _ok(lib.r4_simtrain_net_apply(net, head, H, _p(prm), _p(g), _p(m), _p(v), step, 1e-3, 0.9, 0.999, 1e-7, None),
                    "apply")
            else:
                l0 = lib.r4_simtrain_launch_count()
                _ok(lib.r4_simtrain_net_step(net, head, H, _p(prm), _p(g), _p(m), _p(v), C.byref(d.d), _p(idx), n, SEED, step,
                                             0.2, step, 1e-3, 0.9, 0.999, 1e-7, _p(scratch), None, _p(acc), None), "step")
                assert lib.r4_simtrain_launch_count() - l0 == LAUNCHES[net][0]
        l0 = lib.r4_simtrain_launch_count()
        _eval(net, head, H, prm, d, _idx(s, head, 20, 1))
        assert lib.r4_simtrain_launch_count() - l0 == LAUNCHES[net][1]
        torch.cuda.synchronize()
        assert not bool(g[:H * 128].any())                  # apply leaves the category table's gradient rows zero
        return prm, m, v, acc

    a = run(20, False)
    b = run(20, False)
    c = run(20, True)
    for x, y, z in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x, z)


@pytest.mark.parametrize("head", [0, 1, 2])
def test_net_dien_equals_head_entry_points(head):
    lib = _lib()
    s = SR.make_samples(40, H, seed=2) if head else R.make_samples(40, H, seed=2)
    d = _Data(s)
    c = SR.cfg(H, head) if head else {"category_hash_size": H}
    w = simtrain.head_weights(c, head, seed=3, bounded_scores=True)
    base = torch.from_numpy(simtrain.flatten(w, c)).cuda()
    n = 33
    idx = torch.from_numpy(np.arange(n) % len(s)).cuda()
    scratch = torch.empty(lib.r4_simtrain_head_scratch_size(head, n), dtype=torch.uint8, device="cuda")
    assert lib.r4_simtrain_net_scratch_size(0, head, n) == lib.r4_simtrain_head_scratch_size(head, n)
    assert lib.r4_simtrain_net_num_params(0, head, H) == lib.r4_simtrain_head_num_params(head, H) == base.numel()
    out = []
    for new in (False, True):
        prm, g, m, v = base.clone(), torch.zeros_like(base), torch.zeros_like(base), torch.zeros_like(base)
        probs = torch.zeros(n, simtrain.CLASSES[head], device="cuda")
        for step in (1, 2, 3):
            args = (H, _p(prm), _p(g), _p(m), _p(v), C.byref(d.d), _p(idx), n, SEED, step, 0.2, step, 1e-3, 0.9, 0.999, 1e-7,
                    _p(scratch), None, None, None)
            _ok(lib.r4_simtrain_net_step(0, head, *args) if new else lib.r4_simtrain_head_step(head, *args), "step")
        eargs = (H, _p(prm), C.byref(d.d), _p(idx), n, _p(scratch), _p(probs), None, None)
        _ok(lib.r4_simtrain_net_eval(0, head, *eargs) if new else lib.r4_simtrain_head_eval(head, *eargs), "eval")
        torch.cuda.synchronize()
        out.append((prm, m, v, probs))
    for x, y in zip(*out):
        assert torch.equal(x, y)


def test_rejected_pairs_write_nothing():
    lib = _lib()
    s = _store(H, 1)
    d = _Data(s)
    prm = torch.zeros(NR.num_params(1, H, 1), device="cuda")
    g = torch.full_like(prm, 7.0)
    idx = torch.zeros(4, dtype=torch.int64, device="cuda")
    scratch = torch.zeros(lib.r4_simtrain_net_scratch_size(1, 1, 4), dtype=torch.uint8, device="cuda")
    probs = torch.full((4, 22), 5.0, device="cuda")
    for net, head in [(0, 3), (1, 3), (3, 3), (4, 0), (4, 1), (4, 2), (5, 1), (-1, 0), (2, -1)]:
        assert lib.r4_simtrain_net_num_params(net, head, H) == -1 and lib.r4_simtrain_net_scratch_size(net, head, 4) == -1
        assert lib.r4_simtrain_net_grad(net, head, H, _p(prm), C.byref(d.d), _p(idx), 4, 1, 1, 0.0, None, None, _p(scratch),
                                        _p(g), None, None, None) == ERR_ARG
        assert lib.r4_simtrain_net_eval(net, head, H, _p(prm), C.byref(d.d), _p(idx), 4, _p(scratch), _p(probs), None,
                                        None) == ERR_ARG
        assert lib.r4_simtrain_net_apply(net, head, H, _p(prm), _p(g), _p(g), _p(g), 1, 1e-3, 0.9, 0.999, 1e-7, None) == ERR_ARG
    for bad in ((1, 1, 0, 4), (1, 1, MAXH + 1, 4), (1, 1, H, 0), (1, 1, H, 4097)):
        net, head, Hs, n = bad
        assert lib.r4_simtrain_net_grad(net, head, Hs, _p(prm), C.byref(d.d), _p(idx), n, 1, 1, 0.0, None, None, _p(scratch),
                                        _p(g), None, None, None) == ERR_ARG
    torch.cuda.synchronize()
    assert bool((g == 7.0).all()) and not bool(prm.any()) and bool((probs == 5.0).all()) and not bool(scratch.any())


def _teacher(net, head, samples, Hs):
    """Slate labels from a float64 twin of the same net (a teacher drawn with stronger weights): the 9 columns drawn from
    its sigmoid outputs, or for the 22-way nets its decisions p > 0.5."""
    hd = 3 if net == 4 else 1
    w = simtrain.net_weights(NR.cfg(Hs, hd), net, hd, seed=7, stress=3.0, bias_noise=0.2)
    p = NR.ref_probs(net, hd, NR.cfg(Hs, hd), simtrain.flatten(w, NR.cfg(Hs, hd), net), samples, np.arange(len(samples)),
                     device="cuda")
    u = np.random.RandomState(1).random_sample(p.shape) if head != 2 else np.full(p.shape, 0.5)
    samples.feedback = (u < p).astype(np.uint8)


@pytest.mark.parametrize("net,head", [p for p in NR.PAIRS if p[1]])
def test_teacher_student_fit_on_gpu(net, head):
    Hs = 200
    if head == 2:
        tr = NR.make_samples(3000, Hs, head, seed=1)
        _teacher(net, head, tr, Hs)
        te = simtrain.SlateSamples(Hs, **{k: getattr(tr, k)[:1000] for k in simtrain.ItemSamples.FIELDS})
    else:
        tr, te = NR.make_samples(3000, Hs, head, seed=1), NR.make_samples(600, Hs, head, seed=2)
        _teacher(net, head, tr, Hs)
        _teacher(net, head, te, Hs)
    m = simtrain.get_model({"category_hash_size": Hs}, NR.NAMES[(net, head)], device="cuda",
                           weights=NR.make_weights(net, Hs, head, "default"))
    init = m.evaluate(te)["loss"]
    h = m.fit(tr, te, epochs=8, steps_per_epoch=40, validation_steps=4, batch_size=128)
    best = min(h["val_loss"])
    if head == 2:
        f = np.bincount(simtrain.slate2label(te.feedback), minlength=22) / len(te)
        assert max(h["val_acc"]) > f.max(), (h["val_acc"], f.max())
        return
    assert max(h["val_auc"]) > 0.8, h["val_auc"]
    assert best < 0.85 * init, (init, h["val_loss"])
    if head == 1:
        assert best < R.constant_loss(te.feedback), (R.constant_loss(te.feedback), h["val_loss"])
