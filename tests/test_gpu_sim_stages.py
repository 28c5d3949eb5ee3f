"""GPU: each stage of the simulator forward held to float64, one stage at a time.

The observation is a dense head over the whole feature vector, so an error inside a recurrence reaches it diluted
(dien: 3456 inputs per output).  Here the head is replaced by a probe (tests/sim_probes.py): a +-I pass-through of one
128-column block of the feature vector, decoded back from the observation, which carries the block unchanged.  The
decoded block is compared with the oracle's own stage computation in float64 on the same probe weights.

* Stages: dien AUGRU halves (GRU-1 -> DIN scores -> AUGRU as deployed), GRU-1's last state through a pass-through AUGRU,
  the last ~20 DIN scores through an AUGRU whose only gate they are (linear in each score), dense tower, pooled category attention, three Flatten slots of
  the head's gathered half; lstm's two sequence GRUs (64 steps), category GRU (21 steps, hard sigmoid) and dense tower;
  dnn's category mean-pool and dense tower; widedeep's two sequence mean-pools.
* Row counts 1, 63, 64, 65, 127, 128, 129 (every row) and 4160 (first, middle and last row of every 64-row CTA); sequence
  lengths 0, 1, 2, 63, 64, ids 0 and hash - 1, dense rows of magnitudes 1e-6 .. 1e4 and a row of 1e4 (sim_probes.feature_rows).
* Chunked passes: 2500 rows at max_rows_per_pass 1000 and 129, so later chunks read the sequence caches at a row0 that
  is not a multiple of the 128-row tile.
* The env path: Slate (constant second sequence, read shared by every row) and SeqSlate-36 (second sequence rebuilt
  per page) at B = 65, the observation at reset and after every step -- the paying steps' from the reward pass -- held
  to float64 over the feature rows r4_features returns; and the Slate observations unchanged bit for bit by
  scores_shared_pct, which only changes the scores kernel's grid split.

Bars (sim_probes.TOL, per stage family): recurrences and scores |got - ref| <= tol * max(|ref|, rms(ref row)); GEMM-only stages
(dense tower, pools, category attention) |got - ref| <= tol * M, M the float64 magnitude pass (the same layers over
|x|, |W|, |b|); Flatten bit-exact.  Every comparison is recorded as a `stage ...` row of the margin report.
"""
import functools
import time

import numpy as np
import pytest

import golden_util
import sim_probes as sp

pytestmark = pytest.mark.gpu

ROW_COUNTS = (1, 63, 64, 65, 127, 128, 129, 4160)
R_MAX = ROW_COUNTS[-1]
CHUNKED_R = 2500
RECUR_PROBES = ("augru0a", "augru0b", "augru1a", "augru1b", "gru1_last0", "gru1_last1", "scores0", "scores1")

_USAGE = {"t0": None, "peak_gb": 0.0}
_RMS_WORST = {}          # (sim, family) -> worst |got - ref| / rms(ref row) of the recurrences


@pytest.fixture(scope="module", autouse=True)
def _runtime_and_memory():
    import torch
    _USAGE["t0"] = time.time()
    yield
    print("\n[sim stages] module runtime %.1f s, peak device memory in use %.1f GB"
          % (time.time() - _USAGE["t0"], _USAGE["peak_gb"]))
    for (sim, fam), v in sorted(_RMS_WORST.items()):
        print("[sim stages] %s %s: worst |err| / rms(row) %.3g" % (sim, fam, v))
    torch.cuda.empty_cache()


def _note_memory():
    import torch
    free, total = torch.cuda.mem_get_info()
    _USAGE["peak_gb"] = max(_USAGE["peak_gb"], (total - free) / 2.0 ** 30)


@functools.lru_cache(maxsize=None)
def _regime(sim, regime):
    return sp.regime_weights(sim, regime)


@functools.lru_cache(maxsize=None)
def _rows(hash_size, R=R_MAX, seed=29):
    return sp.feature_rows(R, seed, hash_size)


@functools.lru_cache(maxsize=None)
def _catalog_log(hash_size, seq=False, B=8):
    from rl4rs_b200 import synth
    cat = synth.make_catalog()
    return cat, synth.make_log(4 * B, pages=4 if seq else 1, catalog=cat, hash_size=hash_size, corrupt_frac=0.1)


def _engine(cfg, w):
    from rl4rs_b200.engine import Engine
    cat, log = _catalog_log(cfg["category_hash_size"])
    eng = Engine(dict(cfg), False, cat, w, log)
    _note_memory()
    return eng


def _probe(sim, name):
    return next(p for p in sp.all_probes() if p.sim == sim and p.name == name)


_STAGE_CACHE = {}


def _stage_ref(probe, regime, pw, seq, dense, cat, rows, tag):
    """float64 stage output (and magnitude pass) of `rows`; the two halves of one AUGRU share one computation."""
    key = (probe.sim, regime, probe.name[:-1] if probe.name.startswith("augru") else probe.name, tag)
    if key not in _STAGE_CACHE:
        s, d, c = seq[rows], dense[rows], cat[rows]
        if probe.sim == "dien" and probe.kind == "recur":
            # GRU-1 -> scores -> AUGRU in float64 on the device: the oracle's stage methods ported to torch
            # (held to them within 1e-12 by test_sim_probes_cpu.py); probes other than augru* read columns 0..127
            i = int(probe.name[5]) if probe.name.startswith("augru") else int(probe.name[-1])
            full = sp.dien_augru_stage_torch(pw, i, s, c, "cuda")
            if not probe.name.startswith("augru"):
                full = full[:, :128]
            mag = None
        else:
            o = sp.oracle(probe, pw, np.float64)
            full = probe.stage(o, s, d, c)
            mag = probe.mag(o, s, d, c) if probe.mag else None
        _STAGE_CACHE[key] = (full, mag)
    full, mag = _STAGE_CACHE[key]
    if probe.name.startswith("augru"):
        h = probe.name.endswith("b")
        return full[:, h * 128:(h + 1) * 128], mag
    return full, mag


def _check(probe, regime, what, got, ref, mag):
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert np.isfinite(got).all(), what
    if probe.kind == "exact":
        golden_util.record_margin(what, np.abs(got - ref), np.full(ref.shape, 1e-30), ref)
        np.testing.assert_array_equal(got, ref, err_msg=what)
        return
    tol = sp.tol(probe, regime)
    err = np.abs(got - ref)
    bound = sp.bound(probe, regime, ref, mag) + 1e-30
    if probe.kind == "recur":
        rms = np.sqrt((ref ** 2).mean(axis=-1, keepdims=True))
        key = (probe.sim, sp.family(probe))
        _RMS_WORST[key] = max(_RMS_WORST.get(key, 0.0), float((err / rms).max()))
    golden_util.record_margin(what, err, bound, ref)
    bad = err > bound
    assert not bad.any(), "%s: %d/%d outside tol %g (worst err/bound %.3g at row %d)" % (
        what, int(bad.sum()), bad.size, tol, float((err / bound).max()),
        int(np.unravel_index(np.argmax(err / bound), err.shape)[0]))


def _row_count_cases():
    return [pytest.param(p.sim, p.name, r, id="%s-%s-%s" % (p.sim, p.name, r)) for p in sp.all_probes() for r in sp.regimes_of(p)]


@pytest.mark.parametrize("sim,name,regime", _row_count_cases())
def test_stage_at_every_row_count(sim, name, regime):
    probe = _probe(sim, name)
    cfg, w = _regime(sim, regime)
    pw = probe.build(w)
    seq, dense, cat = _rows(cfg["category_hash_size"])
    rows = np.unique(np.concatenate([np.arange(129), sp.sample_rows(R_MAX)]))
    ref_all, mag_all = _stage_ref(probe, regime, pw, seq, dense, cat, rows, "rows")
    pos = {r: k for k, r in enumerate(rows.tolist())}
    eng = _engine(cfg, pw)
    try:
        for R in ROW_COUNTS:
            obs, _ = eng.dien_forward(seq[:R], dense[:R], cat[:R])
            obs = obs.cpu().numpy()
            _note_memory()
            idx = sp.sample_rows(R)
            k = np.asarray([pos[i] for i in idx.tolist()])
            _check(probe, regime, "stage %s %s %s R%d" % (sim, name, regime, R), sp.decode(obs[idx]), ref_all[k],
                   None if mag_all is None else mag_all[k])
    finally:
        eng.close()


@pytest.mark.parametrize("per_pass", [1000, 129])
@pytest.mark.parametrize("name", RECUR_PROBES)
def test_recurrent_stage_over_chunked_passes(name, per_pass):
    """2500 rows in passes of `per_pass`: the later passes read the sequence caches from row0 = 1000, 2000 or k * 129."""
    probe = _probe("dien", name)
    regime = "bounded"
    cfg, w = _regime("dien", regime)
    cfg = dict(cfg, max_rows_per_pass=per_pass)
    pw = probe.build(w)
    seq, dense, cat = _rows(cfg["category_hash_size"], CHUNKED_R, 31)
    starts = np.arange(0, CHUNKED_R, per_pass)
    idx = sp.sample_rows(CHUNKED_R, extra=np.concatenate([starts, starts - 1, starts + per_pass // 2]))
    ref, _ = _stage_ref(probe, regime, pw, seq, dense, cat, idx, "chunk%d" % per_pass)
    eng = _engine(cfg, pw)
    try:
        obs, _ = eng.dien_forward(seq, dense, cat)
        obs = obs.cpu().numpy()
        _note_memory()
    finally:
        eng.close()
    _check(probe, regime, "stage dien %s %s R%d pass%d" % (name, regime, CHUNKED_R, per_pass), sp.decode(obs[idx]), ref, None)


# ---- the env path --------------------------------------------------------------------------------------------------------
ENV_B = 65


def _run_env(seq_env, probe, pct=None):
    """One episode of a probe env (bounded regime, B = 65, 80 % logged actions): per state (reset, then every step) the
    decoded observation and the feature rows r4_features returns."""
    from rl4rs_b200 import _capi
    from test_gpu_parity import make_env, obs_arrays
    T = 36 if seq_env else 9
    cfg, w = _regime("dien", "bounded")
    cfg = dict(cfg, batch_size=ENV_B, cache_size=ENV_B, max_steps=T, support_rllib_mask=True)
    cat, log = _catalog_log(cfg["category_hash_size"], seq_env, ENV_B)
    states = []
    if pct is not None:
        _capi.set_option("scores_shared_pct", pct)
    try:
        env = make_env(cfg, seq_env, cat, log, probe.build(w), output_format="numpy")
        eng = env.sim.engine
        rs = np.random.RandomState(7)

        def grab(o):
            c, d, s = eng.features()
            states.append((np.asarray(obs_arrays(o)["obs"]).copy(), s.cpu().numpy(), d.cpu().numpy(), c.cpu().numpy()))
        grab(env.reset())
        for t in range(T):
            a = np.where(rs.rand(ENV_B) < 0.8, np.asarray(env.offline_action), rs.randint(0, 284, ENV_B))
            o, _, _, _ = env.step(a)
            grab(o)
        _note_memory()
        eng.close()
    finally:
        if pct is not None:
            _capi.set_option("scores_shared_pct", 85)
    return states


@pytest.mark.parametrize("name", ["augru0a", "augru0b", "augru1a", "augru1b"])
@pytest.mark.parametrize("kind", ["slate", "seqslate36"])
def test_env_observation_stage(kind, name):
    probe = _probe("dien", name)
    _, w = _regime("dien", "bounded")
    pw = probe.build(w)
    i, h = int(name[5]), name.endswith("b")
    for t, (obs, seq, dense, cat) in enumerate(_run_env(kind == "seqslate36", probe)):
        ref = sp.dien_augru_stage_torch(pw, i, seq, cat, "cuda")[:, h * 128:(h + 1) * 128]
        _check(probe, "bounded", "stage dien %s env %s B%d" % (name, kind, ENV_B), sp.decode(obs), ref, None)


def test_scores_shared_pct_changes_no_bit():
    """k_scores_tc2 splits its CTAs between the shared (constant) second sequence and the per-row first one by
    scores_shared_pct; each row's scores are computed the same way whichever CTA computes them."""
    probe = _probe("dien", "augru1a")
    base = _run_env(False, probe, 85)
    for pct in (10, 50, 100):
        other = _run_env(False, probe, pct)
        for t, (a, b) in enumerate(zip(base, other)):
            np.testing.assert_array_equal(a[0].view(np.uint32), b[0].view(np.uint32),
                                          err_msg="scores_shared_pct %d, state %d" % (pct, t))
