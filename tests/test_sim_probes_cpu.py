"""CPU: the probe channel of tests/sim_probes.py is exact, and the weight regimes the GPU stage tests use are well
conditioned.

* Under every probe and regime the f32 oracle's full forward, decoded, equals the f32 stage output bit for bit, and the
  f64 forward equals the f64 stage output within 1e-12: the observation carries the stage unchanged, so a GPU
  observation decoded the same way can be held to the float64 stage itself.
* A probe changes only the tensors it lists, and it sees its stage: a small perturbation of the stage (Probe.perturb)
  moves the decoded float64 block past the probe's bar.
* f32 and f64 oracles agree within 1e-5 of the row rms on every stage of every regime.  (make_weights(stress=2) without
  bounded scores fails this -- its AUGRU outputs reach ~1e3 and f32 leaves f64 far behind -- so it is not a regime here.)
"""
import functools

import numpy as np
import pytest

import sim_probes as sp

ROWS = 40


@functools.lru_cache(maxsize=None)
def _regime(sim, regime):
    return sp.regime_weights(sim, regime)


@functools.lru_cache(maxsize=None)
def _rows(hash_size):
    return sp.feature_rows(ROWS, 17, hash_size)


def _cases():
    return [pytest.param(p.sim, p.name, r, id="%s-%s-%s" % (p.sim, p.name, r)) for p in sp.all_probes() for r in sp.regimes_of(p)]


def _probe(sim, name):
    return next(p for p in sp.all_probes() if p.sim == sim and p.name == name)


@pytest.mark.parametrize("sim,name,regime", _cases())
def test_probe_passes_the_stage_through_the_observation(sim, name, regime):
    probe = _probe(sim, name)
    cfg, w = _regime(sim, regime)
    seq, dense, cat = _rows(cfg["category_hash_size"])
    pw = probe.build(w)
    changed = sorted(k for k in w if not (w[k] is pw[k] or np.array_equal(w[k], pw[k])))
    assert changed and set(changed) <= set(probe.changed), (probe, changed)
    assert set(pw) == set(w)
    for dt, exact in ((np.float32, True), (np.float64, False)):
        o = sp.oracle(probe, pw, dt)
        obs = o.forward(seq, dense, cat)[0]
        got = sp.decode(obs)
        ref = probe.stage(o, seq, dense, cat)
        assert got.shape == ref.shape == (ROWS, 128)
        assert np.isfinite(ref).all()
        if exact:
            np.testing.assert_array_equal(got, ref, err_msg="%r %s f32" % (probe, regime))
        else:
            err = np.abs(got - ref).max()
            assert err <= 1e-12, (probe, regime, err)


@pytest.mark.parametrize("sim,name,regime", _cases())
def test_probe_sees_a_perturbation_of_its_stage(sim, name, regime):
    """The decoded float64 block of a probe moves past the probe's own bar when the stage it exposes is perturbed a
    little (`Probe.perturb`: 1e-3 of one 64-column chunk of a recurrent weight, 1 % of the lstm input kernels and of
    the DIN read-out, 1e-4 or 1e-5 of a GEMM-only stage's weights or embeddings, one ulp of the embedding table for
    Flatten).  A probe whose output did not
    depend on its stage -- a saturated gate, a product that underflows -- would fail here."""
    probe = _probe(sim, name)
    cfg, w = _regime(sim, regime)
    seq, dense, cat = _rows(cfg["category_hash_size"])
    o = sp.oracle(probe, probe.build(w), np.float64)
    ref = sp.decode(o.forward(seq, dense, cat)[0])
    moved = sp.decode(sp.oracle(probe, probe.build(probe.perturb(w)), np.float64).forward(seq, dense, cat)[0])
    mag = probe.mag(o, seq, dense, cat) if probe.mag else None
    shift = np.abs(moved - ref)
    if probe.kind == "exact":
        assert (shift > 0).mean() > 0.5, (probe, regime)
    else:
        worst = float((shift / sp.bound(probe, regime, ref, mag)).max())
        print("%r %s: perturbation moves the block %.3g x the bar" % (probe, regime, worst))
        assert worst > 2.0, (probe, regime, worst)


@pytest.mark.parametrize("regime", sp.BOUNDED)
def test_scores_probe_sees_the_scores_themselves(regime):
    """The scores probe holds the DIN scores of the last ~20 steps linearly: scaling every score by 1.01, or reading
    each step's score one step late, moves its decoded block past the bar, with the GRU-1 states unchanged."""
    cfg, w = _regime("dien", regime)
    seq, dense, cat = _rows(cfg["category_hash_size"])
    for i in range(2):
        probe = _probe("dien", "scores%d" % i)
        o = sp.oracle(probe, probe.build(w), np.float64)
        es = o.w["emb_seq"]
        q = es[cat[:, -10:].astype(np.int64)].mean(axis=1)
        H = o.gru(i, es[seq[:, i, :].astype(np.int64)])
        a = o.att_scores(i, q, H)
        ref = o.augru(i, H, a)[:, :128]
        late = np.concatenate([a[:, :1], a[:, :-1]], axis=1)
        # (the bounded regime's scores are nearly flat along the sequence, 0.539 .. 0.542 for sequence 0 on these rows, so
        # a one-step shift is the smaller change of the two)
        for what, a2, need in (("x1.01", a * 1.01, 2.0), ("one step late", late, 1.0)):
            moved = o.augru(i, H, a2)[:, :128]
            worst = float((np.abs(moved - ref) / sp.bound(probe, regime, ref, None)).max())
            print("scores%d %s, scores %s: the block moves %.3g x the bar" % (i, regime, what, worst))
            assert worst > need, (regime, i, what, worst)


def _stages(sim, o, seq, dense, cat):
    if sim == "dien":
        out = {"augru%d" % i: sp.dien_augru_stage(o, i, seq, cat) for i in range(2)}
        es = o.w["emb_seq"]
        q = es[cat[:, -10:].astype(np.int64)].mean(axis=1).astype(o.dt)
        for i in range(2):
            H = o.gru(i, es[seq[:, i, :].astype(np.int64)])
            out["gru%d" % i] = H[:, -1]
            out["scores%d" % i] = o.att_scores(i, q, H)
        out["dense"] = o.dense_feature(dense)
        out["catattn"] = o.category_feature(cat)[:, :128]
        return out
    names = {"lstm": list(sp.LSTM_OFF), "dnn": ["catpool", "dense"], "widedeep": ["pool0", "pool1"]}[sim]
    return {p.name: p.stage(o, seq, dense, cat) for p in sp.all_probes() if p.sim == sim and p.name in names}


@pytest.mark.parametrize("sim,regime", [("dien", r) for r in sp.DIEN_REGIMES] + [("lstm", r) for r in sp.LSTM_REGIMES]
                         + [("dnn", "default"), ("widedeep", "default")])
def test_regime_is_well_conditioned(sim, regime):
    cfg, w = _regime(sim, regime)
    seq, dense, cat = _rows(cfg["category_hash_size"])
    s32 = _stages(sim, sp.oracle(sim, w, np.float32), seq, dense, cat)
    s64 = _stages(sim, sp.oracle(sim, w, np.float64), seq, dense, cat)
    for k in s64:
        a, b = np.asarray(s32[k], np.float64), s64[k]
        rms = np.sqrt((b ** 2).mean(axis=-1, keepdims=True))
        worst = float((np.abs(a - b) / rms).max())
        assert worst <= 1e-5, (sim, regime, k, worst)


@pytest.mark.parametrize("regime", sp.DIEN_REGIMES)
def test_torch_float64_port_matches_the_oracle(regime):
    """The torch float64 port of GRU-1 -> scores -> AUGRU (run on the device by the GPU stage tests) against the NumPy
    oracle in float64, on the base weights and under the probes that change the AUGRU."""
    cfg, w = _regime("dien", regime)
    seq, dense, cat = _rows(cfg["category_hash_size"])
    for name in ("augru0a", "gru1_last1") + (("scores0",) if regime in sp.BOUNDED else ()):
        pw = _probe("dien", name).build(w)
        o = sp.oracle("dien", pw, np.float64)
        for i in range(2):
            ref = sp.dien_augru_stage(o, i, seq, cat)
            got = sp.dien_augru_stage_torch(pw, i, seq, cat)
            assert np.abs(got - ref).max() <= 1e-12, (regime, name, i, np.abs(got - ref).max())


def test_unbounded_stress_regime_is_ill_conditioned():
    """The regime left out on purpose: stress 2 with raw DIN scores.  Its AUGRU outputs grow far past 1 and the f32
    recurrence departs from f64 by more than the bar of the probes, so no float64 comparison could hold a kernel to it."""
    from rl4rs_b200 import synth
    cfg = sp.sim_cfg("dien", 5000)
    w = synth.make_weights(cfg, stress=2.0)
    seq, dense, cat = _rows(5000)
    a = sp.dien_augru_stage(sp.oracle("dien", w, np.float32), 0, seq, cat).astype(np.float64)
    b = sp.dien_augru_stage(sp.oracle("dien", w, np.float64), 0, seq, cat)
    rms = np.sqrt((b ** 2).mean(axis=-1, keepdims=True))
    assert np.abs(b).max() > 10.0
    assert (np.abs(a - b) / rms).max() > 1e-4


def test_decode_and_sample_rows():
    x = np.array([[-2.0, 0.0, 3.5] + [1.0] * 125], np.float32)
    el = lambda v: np.where(v > 0, v, np.expm1(np.minimum(v, 0)))
    obs = np.concatenate([el(x), el(-x)], axis=1).astype(np.float32)
    np.testing.assert_array_equal(sp.decode(obs), x)
    np.testing.assert_array_equal(sp.sample_rows(129), np.arange(129))
    idx = sp.sample_rows(4160)
    assert {0, 32, 63, 64, 4096, 4128, 4159} <= set(idx.tolist())
    assert len(idx) == 3 * 65
    seq, dense, cat = sp.feature_rows(12, 1, 5000)
    lens = (seq != 0).sum(axis=2)
    np.testing.assert_array_equal(lens[:5], np.repeat(np.array(sp.EDGE_LENGTHS)[:, None], 2, axis=1))
    assert (dense[10] == 1e4).all() and (dense[5:10] == 0).any()
