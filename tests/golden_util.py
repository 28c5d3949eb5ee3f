"""Helpers shared by the oracle (CPU) and CUDA (GPU) parity tests over tests/golden/*.npz."""
import glob
import json
import os

import numpy as np

from rl4rs_b200 import synth
from rl4rs_b200.utils.datautil import FeatureUtil

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden_names():
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "*.npz")))


class Golden(object):
    def __init__(self, name):
        z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
        self.name = name
        self.meta = json.loads(bytes(z["meta"]).decode())
        self.arr = {k: z[k] for k in z.files if k != "meta"}
        self.config = self.meta["config"]
        self.seq = self.meta["seq"]
        self.catalog = synth.Catalog.from_text(self.meta["catalog_text"])
        self.log = FeatureUtil.parse_log(self.meta["records"], self.config.get("maxlen", 64))
        self._weights = None

    @property
    def weights(self):
        if self._weights is None:
            self._weights = synth.make_weights(self.config, **self.meta["weights"])
        return self._weights

    @property
    def n_episodes(self):
        return self.arr["reward"].shape[0] // self.config["max_steps"]


# tolerance of the floating-point half (north_star: 1e-4 relative on rewards / observations).
# Observations are 256 ELU outputs of one 3456-long dot product each, some of them ~0, so the
# relative bound is taken against max(|ref|, rms(ref row)) -- an element-wise relative test on a
# value that happens to be 1e-7 would test nothing but cancellation.
RTOL = 1e-4

# Every comparison is recorded: worst error/bound under the rms-floored rule the assertion uses, and next to it the
# PLAIN element-wise worst relative error |got-ref|/|ref| (over elements with ref != 0) with the |ref| it occurred
# at, so a reader can see what the floor forgives.  conftest.py prints the table and writes
# gpurun_out/parity_margins.json at the end of a GPU session.
MARGINS = {}


def _record(what, err, bound, ref):
    key = what.split(" step ")[0]
    _record_key("".join(c for c in key if not c.isdigit()).strip() or "?", err, bound, ref)


def record_margin(key, err, bound, ref):
    """Record one comparison under `key` as given: digits are kept, so a key can name the shape it was measured at
    (the learner grid's `learner rainbow A284 Z8 ... sb2` rows)."""
    _record_key(key, np.asarray(err, dtype=np.float64), np.asarray(bound, dtype=np.float64), np.asarray(ref, dtype=np.float64))


def _record_key(key, err, bound, ref):
    nz = np.abs(ref) > 0
    plain = np.zeros_like(err)
    plain[nz] = err[nz] / np.abs(ref[nz])
    i = int(np.argmax(plain)) if plain.size else 0
    m = MARGINS.setdefault(key, {"n": 0, "floored_err_over_bound": 0.0, "plain_rel_max": 0.0, "plain_rel_at_abs_ref": 0.0,
                                 "row_rms_there": 0.0})
    m["n"] += int(err.size)
    if err.size:
        m["floored_err_over_bound"] = max(m["floored_err_over_bound"], float((err / bound).max()))
        if float(plain.flat[i]) > m["plain_rel_max"]:
            m["plain_rel_max"] = float(plain.flat[i])
            m["plain_rel_at_abs_ref"] = float(np.abs(ref).flat[i])
            if ref.ndim >= 2:
                row = np.unravel_index(i, ref.shape)[:-1]
                m["row_rms_there"] = float(np.sqrt((ref[row] ** 2).mean()))


def assert_close_rel(got, ref, rtol=RTOL, what=""):
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    if ref.ndim >= 2:
        scale = np.sqrt((ref ** 2).mean(axis=-1, keepdims=True))
    else:
        scale = np.abs(ref)
    bound = rtol * np.maximum(np.abs(ref), scale) + 1e-12
    err = np.abs(got - ref)
    _record(what, err, bound, ref)
    bad = err > bound
    assert not bad.any(), "%s: %d/%d outside rtol=%g (worst err/bound %.3g)" % (
        what, int(bad.sum()), bad.size, rtol, float((err / bound).max()))


REFERENCE_GOLDEN_DIR = os.path.join(GOLDEN_DIR, "reference")


def reference_result(key, compute):
    """What the reference's own code computes for one test case, stored under tests/golden/reference/<key>.npz.

    `compute()` runs the reference (oracle/ref_harness.py, oracle/tf_eager_stub.py) and returns a dict of NumPy arrays and
    JSON values.  It runs only to (re)write the stored result -- `RL4RS_WRITE_GOLDEN=1` with the reference tree present
    (tests/golden/make_reference_golden.py) -- so the comparison itself needs nothing outside the repository."""
    path = os.path.join(REFERENCE_GOLDEN_DIR, key + ".npz")
    if os.environ.get("RL4RS_WRITE_GOLDEN"):
        from oracle import ref_harness
        assert ref_harness.reference_available(), "RL4RS_WRITE_GOLDEN needs the reference tree (RL4RS_REFERENCE_ROOT)"
        out = compute()
        arrays = {k: np.asarray(v) for k, v in out.items() if isinstance(v, np.ndarray)}
        rest = {k: v for k, v in out.items() if not isinstance(v, np.ndarray)}
        os.makedirs(REFERENCE_GOLDEN_DIR, exist_ok=True)
        np.savez_compressed(path, __json__=np.frombuffer(json.dumps(rest).encode(), dtype=np.uint8), **arrays)
    assert os.path.exists(path), "stored reference result missing: %s" % path
    z = np.load(path)
    out = json.loads(bytes(z["__json__"]).decode())
    out.update({k: z[k] for k in z.files if k != "__json__"})
    return out
