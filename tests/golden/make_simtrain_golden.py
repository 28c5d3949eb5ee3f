"""Fixture generator (run in the build container only): the reference's OWN ``script/data_preprocess.py`` stage
``tfrecord_item`` on synthetic multi-page sessions -> tests/golden/simtrain/item_samples.npz (a directory of its own:
the env fixtures are every .npz directly under tests/golden).

``FeatureUtil.to_tfrecord`` is replaced by a capture that runs the reference's own ``FeatureUtil.feature_extraction`` on the
records it is handed (what to_tfrecord serialises), and ``random.shuffle`` runs on a seeded ``random``; the fixture keeps the
seed so a test can undo the shuffle.

    python tests/golden/make_simtrain_golden.py
"""
import os
import random
import runpy
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_harness  # noqa: E402
from rl4rs_b200 import synth  # noqa: E402

SHUFFLE_SEED = 11


def pages():
    """Sessions of 4, 1, 3, 4, 2 and 4 pages; history lengths from the synthetic log (several above 64)."""
    cat = synth.make_catalog()
    log = synth.make_log(24, pages=1, catalog=cat, keep_hist=True, seed=91)
    recs = synth.render_records(log, cat)
    out, r = [], 0
    for s, npage in enumerate((4, 1, 3, 4, 2, 4)):
        base = recs[r].split("@")
        for p in range(npage):
            f = recs[r + p].split("@")
            out.append("@".join([str(100 * s + p), base[1], str(p + 1), f[3], f[4], base[5], base[6], f[7], base[8]]))
        r += npage
    return out, log


def main():
    mods = ref_harness.install_stubs()
    del mods
    from rl4rs.utils import datautil as ref_datautil
    captured = {}

    def capture(self, data, filename):
        (seq, dense, catf, _), labels = self.feature_extraction(data)
        captured.update(seq=np.asarray(seq, np.int64), dense=np.asarray(dense, np.float32),
                        cat=np.asarray(catf, np.int64), label=np.asarray(labels, np.int64))
    ref_datautil.FeatureUtil.to_tfrecord = capture
    script = os.path.join(ref_harness.REFERENCE_ROOT, "script", "data_preprocess.py")
    lines, log = pages()
    assert (log.seq_len > 64).any()
    header = "timestamp@session_id@sequence_id@exposed_items@user_feedback@user_seqfeature@user_protrait@item_feature@behavior_policy_id"
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.csv"), os.path.join(d, "out.tfrecord")
        open(src, "w").write("\n".join([header] + lines + [""]))
        argv = sys.argv
        sys.argv = [script, src, dst, "tfrecord_item"]
        random.seed(SHUFFLE_SEED)
        try:
            runpy.run_path(script, run_name="__main__")
        finally:
            sys.argv = argv
    out = os.path.join(ROOT, "tests", "golden", "simtrain")
    os.makedirs(out, exist_ok=True)
    np.savez_compressed(os.path.join(out, "item_samples.npz"),
                        lines=np.array(lines), shuffle_seed=np.int64(SHUFFLE_SEED), **captured)
    print("samples:", captured["cat"].shape[0], "records:", len(lines))


if __name__ == "__main__":
    main()
