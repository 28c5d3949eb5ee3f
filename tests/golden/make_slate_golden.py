"""Fixture generator (run in the build container only): the reference's OWN ``script/data_preprocess.py`` stage
``tfrecord_slate`` on the synthetic multi-page sessions of make_simtrain_golden.py -> tests/golden/simtrain/slate_samples.npz.

As for the item samples, ``FeatureUtil.to_tfrecord`` is replaced by a capture that runs the reference's own
``FeatureUtil.feature_extraction`` on the records it is handed, and ``random.shuffle`` runs on a seeded ``random``; the
fixture keeps the seed so a test can undo the shuffle.  item_samples.npz is not touched.

    python tests/golden/make_slate_golden.py
"""
import os
import random
import runpy
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from oracle import ref_harness  # noqa: E402
import make_simtrain_golden  # noqa: E402

SHUFFLE_SEED = 13


def main():
    ref_harness.install_stubs()
    from rl4rs.utils import datautil as ref_datautil
    captured = {}

    def capture(self, data, filename):
        (seq, dense, catf, slate_label), _ = self.feature_extraction(data)
        captured.update(seq=np.asarray(seq, np.int64), dense=np.asarray(dense, np.float32),
                        cat=np.asarray(catf, np.int64), slate_label=np.asarray(slate_label, np.int64))
    ref_datautil.FeatureUtil.to_tfrecord = capture
    script = os.path.join(ref_harness.REFERENCE_ROOT, "script", "data_preprocess.py")
    lines, _ = make_simtrain_golden.pages()
    header = "timestamp@session_id@sequence_id@exposed_items@user_feedback@user_seqfeature@user_protrait@item_feature@behavior_policy_id"
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.csv"), os.path.join(d, "out.tfrecord")
        open(src, "w").write("\n".join([header] + lines + [""]))
        argv = sys.argv
        sys.argv = [script, src, dst, "tfrecord_slate"]
        random.seed(SHUFFLE_SEED)
        try:
            runpy.run_path(script, run_name="__main__")
        finally:
            sys.argv = argv
    out = os.path.join(HERE, "simtrain")
    os.makedirs(out, exist_ok=True)
    np.savez_compressed(os.path.join(out, "slate_samples.npz"),
                        lines=np.array(lines), shuffle_seed=np.int64(SHUFFLE_SEED), **captured)
    print("samples:", captured["cat"].shape[0], "records:", len(lines))


if __name__ == "__main__":
    main()
