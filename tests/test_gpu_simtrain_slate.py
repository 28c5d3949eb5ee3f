"""GPU: the slate-label heads of the simulator trainer (r4_simtrain_head_*, heads 1 = dien_slate and 2 =
dien_slate_multiclass) against the float64 twin of tests/simtrain_slate_ref.py.

  gradient grid   both heads, n = 1, 7, 8, 9, 63, 64, 65, 256, 257 at H = 3000, drop rate 0 / 0.2, default / stress weights;
                  edge samples at H = 9; n = 65 and 2049 at H = 4 000 000 over the compacted reference.  Bound as in
                  test_gpu_simtrain.py: max |g - ref| <= 1e-4 max |ref| per tensor, 1e-3 for the attention MLPs and emb_cat;
                  every embedding row the batch does not read is exactly zero.
  eval / metrics  probabilities against the twin; the f64 accumulator against the host metrics on the kernel's own
                  probabilities; grad's accumulator at rate 0 equal to eval's bit for bit
  chained steps   head_step == head_grad + head_apply bit for bit; twenty steps bit-identical across two runs
  head 0          the head entry points at head 0 equal the r4_simtrain_* ones bit for bit
  launches        59 per step for every head
  rejections      bad head, hash size or n: R4_ERR_ARG, nothing written
  learning        teacher-student fit for both heads; the saved checkpoint reloads bit-exact
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import simtrain_ref as R  # noqa: E402
import simtrain_slate_ref as SR  # noqa: E402
from golden_util import assert_close_rel, record_margin  # noqa: E402

from rl4rs_b200 import _capi, simtrain, synth  # noqa: E402
from rl4rs_b200.utils import tf_checkpoint  # noqa: E402

pytestmark = pytest.mark.gpu

H = 3000
MAXH = 4000000
TOL, TOL_CANCEL = 1e-4, 1e-3          # test_gpu_simtrain.py states why the attention MLPs and emb_cat get 1e-3
ERR_ARG = -1
SEED, COUNTER = 5, 77
_STORES = {}


def _lib():
    return _capi.load_library()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _ok(rc, what):
    if rc != 0:
        raise AssertionError("%s failed (%d): %s" % (what, rc, (_lib().r4_last_error(None) or b"?").decode()))


def _store(Hs, records=300, edge=False):
    key = (Hs, records, edge)
    if key not in _STORES:
        _STORES[key] = SR.make_samples(records, Hs, seed=Hs % 1000 + 3, edge=edge)
    return _STORES[key]


class _Data(object):
    def __init__(self, samples):
        self.ts = [torch.from_numpy(np.ascontiguousarray(getattr(samples, k))).cuda() for k in simtrain.ItemSamples.FIELDS]
        self.d = _capi.SimTrainData(*[t.data_ptr() for t in self.ts])


def _offsets(Hs, head):
    out, o = {}, 0
    for name, shape in simtrain.layer_plan(SR.cfg(Hs, head)):
        out[name] = (o, shape)
        o += int(np.prod(shape))
    return out


def _device_params(w, Hs, head, ids=None):
    """The flat parameters at Hs on the device; with ids, w's compact embedding rows at rows ids of zero tables."""
    prm = torch.zeros(SR.num_params(Hs, head), dtype=torch.float32, device="cuda")
    for name, (o, shape) in _offsets(Hs, head).items():
        v = torch.from_numpy(np.ascontiguousarray(w[name], dtype=np.float32)).cuda()
        k = int(np.prod(shape))
        if ids is not None and name.startswith("emb_"):
            prm[o:o + k].view(Hs, -1)[torch.from_numpy(ids).cuda()] = v
        else:
            prm[o:o + k] = v.reshape(-1)
    return prm


def _grad(head, Hs, prm, data, idx, rate, grad=None, acc=None):
    lib = _lib()
    n = len(idx)
    scratch = torch.empty(lib.r4_simtrain_head_scratch_size(head, n), dtype=torch.uint8, device="cuda")
    grad = torch.zeros_like(prm) if grad is None else grad
    keep = torch.zeros(n, 256, dtype=torch.uint8, device="cuda")
    stats = torch.zeros(2, dtype=torch.float32, device="cuda")
    it = torch.from_numpy(np.asarray(idx, np.int64)).cuda()
    _ok(lib.r4_simtrain_head_grad(head, Hs, _p(prm), C.byref(data.d), _p(it), n, SEED, COUNTER, rate, None, _p(keep),
                                  _p(scratch), _p(grad), _p(stats), _p(acc), None), "r4_simtrain_head_grad")
    torch.cuda.synchronize()
    return grad, stats.cpu().numpy(), keep.cpu().numpy()


def _eval(head, Hs, prm, data, idx, acc):
    lib = _lib()
    n = len(idx)
    scratch = torch.empty(lib.r4_simtrain_head_scratch_size(head, n), dtype=torch.uint8, device="cuda")
    probs = torch.full((n, simtrain.CLASSES[head]), -1.0, dtype=torch.float32, device="cuda")
    it = torch.from_numpy(np.asarray(idx, np.int64)).cuda()
    _ok(lib.r4_simtrain_head_eval(head, Hs, _p(prm), C.byref(data.d), _p(it), n, _p(scratch), _p(probs), _p(acc), None),
        "r4_simtrain_head_eval")
    torch.cuda.synchronize()
    return probs.cpu().numpy()


def _check_grad(tag, head, Hs, grad, ids, ref):
    """Per tensor against the reference over the rows ids; every other embedding row exactly zero."""
    rt = simtrain.unflatten(ref, SR.cfg(len(ids), head))
    idt = torch.from_numpy(ids).cuda()
    bad = []
    for name, (o, shape) in _offsets(Hs, head).items():
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
        bound = (TOL_CANCEL if name.startswith(("att", "emb_cat")) else TOL) * scale
        record_margin("simtrain slate%d %s %s" % (head, name, tag), np.array([err]), np.array([bound + 1e-30]), np.array([scale]))
        if err > bound:
            bad.append((name, err, bound))
    assert not bad, "%s: tensors outside their bound (name, err, bound): %s" % (tag, bad)


def _parity(head, Hs, s, idx, kind, rate, tag):
    ids, sc, ic = SR.compact(s, idx)
    w = SR.make_weights(9 if Hs == MAXH else Hs, head, kind)
    if Hs == MAXH:
        rs = np.random.RandomState(31)
        wc = dict(w, emb_cat=rs.uniform(-0.05, 0.05, (len(ids), 128)).astype(np.float32),
                  emb_seq=rs.uniform(-0.05, 0.05, (len(ids), 128)).astype(np.float32))
        prm = _device_params(wc, Hs, head, ids)
    else:
        wc = dict(w, emb_cat=w["emb_cat"][ids], emb_seq=w["emb_seq"][ids])
        prm = _device_params(w, Hs, head)
    grad, stats, keep = _grad(head, Hs, prm, _Data(s), idx, rate)
    assert np.array_equal(keep, R.keep_bits(SEED, COUNTER, len(idx), rate))
    c = SR.cfg(len(ids), head)
    loss, ref, _ = SR.ref_grad(head, c, simtrain.flatten(wc, c), sc, ic, keep if rate > 0 else None, rate, device="cuda")
    assert abs(stats[0] - loss) <= 1e-5 * abs(loss) + 1e-6, (stats[0], loss)
    _check_grad(tag, head, Hs, grad, ids, ref)
    del grad, prm
    torch.cuda.empty_cache()


@pytest.mark.parametrize("head", SR.HEADS)
@pytest.mark.parametrize("kind", ["default", "stress"])
@pytest.mark.parametrize("n", [1, 7, 8, 9, 63, 64, 65, 256, 257])
@pytest.mark.parametrize("rate", [0.0, 0.2])
def test_gradient_parity_per_tensor(head, kind, n, rate):
    s = _store(H)
    idx = np.random.RandomState(n).permutation(len(s))[:n]
    _parity(head, H, s, idx, kind, rate, "n%d H%d %s drop%g" % (n, H, kind, rate))


@pytest.mark.parametrize("head", SR.HEADS)
@pytest.mark.parametrize("n,kind,rate", [(1, "stress", 0.0), (64, "default", 0.2), (65, "stress", 0.2)])
def test_gradient_parity_edge_samples(head, n, kind, rate):
    s = _store(9, 120, edge=True)
    idx = np.random.RandomState(n + 5).permutation(len(s))[:n]
    _parity(head, 9, s, idx, kind, rate, "edge n%d H9 %s drop%g" % (n, kind, rate))


@pytest.mark.parametrize("head", SR.HEADS)
@pytest.mark.parametrize("n,kind,rate", [(65, "stress", 0.2), (2049, "default", 0.0)])
def test_gradient_parity_max_hash(head, n, kind, rate):
    s = _store(MAXH, 2100)
    idx = np.random.RandomState(n + 7).permutation(len(s))[:n]
    _parity(head, MAXH, s, idx, kind, rate, "n%d H%d %s drop%g" % (n, MAXH, kind, rate))


def _check_acc(head, acc, probs, y, loss):
    """The device accumulator against the host metrics of the kernel's own probabilities: every count exactly, the binary
    accuracy sum (f32 per-sample means) to 1e-6, the loss sum against the float64 twin's to 1e-5."""
    a = acc.cpu().numpy()
    m = SR.host_metrics(head, probs, y, np.zeros(len(y)))
    assert a.shape == m.acc.shape
    assert a[2] == m.acc[2] == len(y)
    if head == 1:
        assert abs(a[1] - m.acc[1]) <= 1e-6 * m.acc[1]
        assert np.array_equal(a[3:], m.acc[3:]), np.flatnonzero(a[3:] != m.acc[3:])
    else:
        assert a[1] == m.acc[1]
    assert abs(a[0] - loss) <= 1e-5 * abs(loss), (a[0], loss)


@pytest.mark.parametrize("head", SR.HEADS)
@pytest.mark.parametrize("n", [1, 257])
def test_eval_probs_and_metrics(head, n):
    s = _store(H)
    w = SR.make_weights(H, head, "stress")
    prm, data = _device_params(w, H, head), _Data(s)
    idx = np.random.RandomState(n + 1).permutation(len(s))[:n]
    acc = torch.zeros(simtrain.METRICS[head].SIZE, dtype=torch.float64, device="cuda")
    probs = _eval(head, H, prm, data, idx, acc)
    c = SR.cfg(H, head)
    flat = simtrain.flatten(w, c)
    assert_close_rel(probs, SR.ref_probs(head, c, flat, s, idx, device="cuda"), what="slate%d eval probs n%d" % (head, n))
    loss = SR.ref_grad(head, c, flat, s, idx, None, 0.0, device="cuda")[0] * n
    _check_acc(head, acc, probs, s.features(idx)[3], loss)
    acc_g = torch.zeros_like(acc)
    _grad(head, H, prm, data, idx, 0.0, acc=acc_g)
    assert torch.equal(acc_g, acc)


@pytest.mark.parametrize("head", SR.HEADS)
def test_step_equals_grad_then_apply(head):
    lib = _lib()
    s = _store(H)
    data = _Data(s)
    base = _device_params(SR.make_weights(H, head), H, head)
    A = [base.clone()] + [torch.zeros_like(base) for _ in range(3)]
    B = [base.clone()] + [torch.zeros_like(base) for _ in range(3)]
    acc_a = torch.zeros(simtrain.METRICS[head].SIZE, dtype=torch.float64, device="cuda")
    acc_b = torch.zeros_like(acc_a)
    sa, sb = torch.zeros(2, device="cuda"), torch.zeros(2, device="cuda")
    for step, n in enumerate((64, 9, 200), 1):
        idx = torch.from_numpy(np.random.RandomState(step).permutation(len(s))[:n].astype(np.int64)).cuda()
        scratch = torch.empty(lib.r4_simtrain_head_scratch_size(head, n), dtype=torch.uint8, device="cuda")
        _ok(lib.r4_simtrain_head_step(head, H, _p(A[0]), _p(A[1]), _p(A[2]), _p(A[3]), C.byref(data.d), _p(idx), n, SEED, step,
                                      0.2, step, 1e-3, 0.9, 0.999, 1e-7, _p(scratch), _p(sa), _p(acc_a), None), "step")
        _ok(lib.r4_simtrain_head_grad(head, H, _p(B[0]), C.byref(data.d), _p(idx), n, SEED, step, 0.2, None, None, _p(scratch),
                                      _p(B[1]), _p(sb), _p(acc_b), None), "grad")
        _ok(lib.r4_simtrain_head_apply(head, H, _p(B[0]), _p(B[1]), _p(B[2]), _p(B[3]), step, 1e-3, 0.9, 0.999, 1e-7, None),
            "apply")
    torch.cuda.synchronize()
    for a, b in zip(A, B):
        assert torch.equal(a, b)
    assert torch.equal(sa, sb) and torch.equal(acc_a, acc_b)
    assert not bool(A[1][:H * 128].any())                 # the embedding gradient rows cleared by the apply


@pytest.mark.parametrize("head", SR.HEADS)
def test_twenty_steps_bit_identical(head):
    s = _store(H)
    outs = []
    for _ in range(2):
        tr = simtrain.get_model({"category_hash_size": H}, SR.NAMES[head], device="cuda",
                                weights=SR.make_weights(H, head), data_seed=3)
        st = simtrain._Stream(len(s), 64, 3, torch.device("cuda"))
        for _ in range(20):
            tr.train_step(s, st.next())
        torch.cuda.synchronize()
        outs.append((tr.params.cpu().numpy(), tr.m.cpu().numpy(), tr.acc.cpu().numpy()))
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


def test_head0_entry_points_equal_the_item_ones():
    lib = _lib()
    s = R.make_samples(60, H, seed=4)
    data = _Data(s)
    w = synth.make_weights({"category_hash_size": H}, seed=21, bounded_scores=True)
    base = _device_params(w, H, 0)
    assert lib.r4_simtrain_head_num_params(0, H) == lib.r4_simtrain_num_params(H) == base.numel()
    n = 100
    assert lib.r4_simtrain_head_scratch_size(0, n) == lib.r4_simtrain_scratch_size(n)
    idx = torch.from_numpy(np.random.RandomState(2).permutation(len(s))[:n].astype(np.int64)).cuda()
    scratch = torch.empty(lib.r4_simtrain_scratch_size(n), dtype=torch.uint8, device="cuda")
    out = []
    for new in (False, True):
        P = [base.clone()] + [torch.zeros_like(base) for _ in range(3)]
        acc = torch.zeros(405, dtype=torch.float64, device="cuda")
        stats = torch.zeros(2, device="cuda")
        probs = torch.zeros(n, 2, device="cuda")
        for step in (1, 2):
            args = (H, _p(P[0]), _p(P[1]), _p(P[2]), _p(P[3]), C.byref(data.d), _p(idx), n, SEED, step, 0.2, step, 1e-3, 0.9,
                    0.999, 1e-7, _p(scratch), _p(stats), _p(acc), None)
            _ok(lib.r4_simtrain_head_step(0, *args) if new else lib.r4_simtrain_step(*args), "step")
        g = torch.zeros_like(base)
        gargs = (H, _p(P[0]), C.byref(data.d), _p(idx), n, SEED, 9, 0.2, None, None, _p(scratch), _p(g), _p(stats), _p(acc), None)
        _ok(lib.r4_simtrain_head_grad(0, *gargs) if new else lib.r4_simtrain_grad(*gargs), "grad")
        eargs = (H, _p(P[0]), C.byref(data.d), _p(idx), n, _p(scratch), _p(probs), _p(acc), None)
        _ok(lib.r4_simtrain_head_eval(0, *eargs) if new else lib.r4_simtrain_eval(*eargs), "eval")
        torch.cuda.synchronize()
        out.append([t.cpu().numpy() for t in P + [g, acc, stats, probs]])
    for a, b in zip(*out):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("head", [0, 1, 2])
def test_step_launches(head):
    lib = _lib()
    s = _store(H) if head else R.make_samples(40, H, seed=1)
    tr = simtrain.SimulatorTrainer({"category_hash_size": H}, device="cuda", head=head)
    idx = torch.arange(32, device="cuda")
    tr.train_step(s, idx)
    torch.cuda.synchronize()
    l0 = lib.r4_simtrain_launch_count()
    tr.train_step(s, idx)
    assert lib.r4_simtrain_launch_count() - l0 == 59


@pytest.mark.parametrize("head", SR.HEADS)
def test_rejections_write_nothing(head):
    lib = _lib()
    s = _store(H)
    data = _Data(s)
    prm = _device_params(SR.make_weights(H, head), H, head)
    grad = torch.full_like(prm, 7.0)
    m, v = torch.zeros_like(prm), torch.zeros_like(prm)
    n = 16
    idx = torch.arange(n, device="cuda")
    scratch = torch.empty(lib.r4_simtrain_head_scratch_size(head, 4096), dtype=torch.uint8, device="cuda")
    probs = torch.full((n, 22), -1.0, device="cuda")
    acc = torch.zeros(simtrain.METRICS[head].SIZE, dtype=torch.float64, device="cuda")
    p0 = prm.clone()
    for hd, Hs, nn in ((-1, H, n), (3, H, n), (head, 0, n), (head, MAXH + 1, n), (head, H, 0), (head, H, 4097)):
        assert lib.r4_simtrain_head_grad(hd, Hs, _p(prm), C.byref(data.d), _p(idx), nn, 1, 1, 0.0, None, None, _p(scratch),
                                         _p(grad), None, _p(acc), None) == ERR_ARG
        assert lib.r4_simtrain_head_eval(hd, Hs, _p(prm), C.byref(data.d), _p(idx), nn, _p(scratch), _p(probs), _p(acc),
                                         None) == ERR_ARG
        assert lib.r4_simtrain_head_step(hd, Hs, _p(prm), _p(grad), _p(m), _p(v), C.byref(data.d), _p(idx), nn, 1, 1, 0.0, 1,
                                         1e-3, 0.9, 0.999, 1e-7, _p(scratch), None, _p(acc), None) == ERR_ARG
        if nn == n:
            assert lib.r4_simtrain_head_apply(hd, Hs, _p(prm), _p(grad), _p(m), _p(v), 1, 1e-3, 0.9, 0.999, 1e-7,
                                              None) == ERR_ARG
    assert lib.r4_simtrain_head_grad(head, H, _p(prm), C.byref(data.d), _p(idx), n, 1, 1, 1.0, None, None, _p(scratch),
                                     _p(grad), None, _p(acc), None) == ERR_ARG
    torch.cuda.synchronize()
    assert torch.equal(prm, p0) and bool((grad == 7.0).all()) and not bool(acc.any()) and bool((probs == -1.0).all())
    assert not bool(m.any()) and not bool(v.any())


@pytest.mark.parametrize("head", SR.HEADS)
def test_teacher_student_on_gpu_and_checkpoint(head, tmp_path):
    Hs = 60
    if head == 1:
        tr_s, te_s = SR.make_samples(1500, Hs, seed=1), SR.make_samples(300, Hs, seed=2)
        SR.teacher_labels(tr_s, Hs)
        SR.teacher_labels(te_s, Hs, label_seed=3)
    else:                      # test_simtrain_slate_cpu.py's _fit_patterns: why the 22-way check validates on training records
        tr_s = SR.make_samples(900, Hs, seed=1)
        SR.teacher_labels(tr_s, Hs, draw=False)
        te_s = simtrain.SlateSamples(Hs, **{k: getattr(tr_s, k)[:300] for k in simtrain.ItemSamples.FIELDS})
    cfg = {"category_hash_size": Hs}
    w = simtrain.head_weights(SR.cfg(Hs, head), head, seed=123, bounded_scores=True)
    m = simtrain.get_model(cfg, SR.NAMES[head], device="cuda", weights=w)
    init = m.evaluate(te_s)["loss"]
    h = m.fit(tr_s, te_s, epochs=6, steps_per_epoch=30, validation_steps=5, batch_size=64)
    keys = ("loss", "auc", "precision", "recall") if head == 1 else ("loss", "acc")
    assert set(h) == set(keys) | {"val_" + k for k in keys}
    best = min(h["val_loss"])
    y = te_s.feedback
    if head == 1:
        const = R.constant_loss(y)
        assert max(h["val_auc"]) > 0.8, h["val_auc"]
    else:
        cls = simtrain.slate2label(y)
        f = np.bincount(cls, minlength=22) / len(cls)
        const = -float(np.sum(f[f > 0] * np.log(f[f > 0])))
        assert max(h["val_acc"]) > f.max(), (h["val_acc"], f.max())
    assert best < 0.85 * init and best < const, (init, const, h["val_loss"])
    prefix = str(tmp_path / "model")
    m.save(prefix)
    back = tf_checkpoint.load_dien_checkpoint(prefix, SR.cfg(Hs, head))
    ref = m.weights()
    assert set(back) == set(ref) and back["rew_w"].shape == (256, simtrain.CLASSES[head])
    for k in ref:
        assert np.array_equal(back[k], ref[k]), k
