"""Write tests/golden/mdpcheck/search.npz: the reference's own rl4rs/mdpchecker/decoder.py (under stand-ins for
bottleneck -- np.argpartition / np.partition -- and for np.int, which NumPy 2 dropped) run over the CPU torch twin of a
seeded model, for the GPU search tests.  Stored: the model's config and float32 weights, 2048 source rows, and the
reference's beam_search outputs for beam 1 and for beam 20 with 20 candidates over all 2048 rows, beam 100 over the first
128 rows, decode_step (beam 10) and token_probs over the first 256 rows after a 3-token prefix.

    python tests/golden/make_mdpcheck_golden.py      (needs the reference tree; RL4RS_REFERENCE_ROOT)
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_harness  # noqa: E402
from rl4rs_b200.mdpchecker import transformer as tf  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "mdpcheck", "search.npz")
CFG = dict(token_num=[120, 120], embed_dim=32, encoder_num=1, decoder_num=1, head_num=2, hidden_dim=64)
ROWS, TS = 2048, 18


def model():
    return tf.get_model(use_same_embed=False, device="cpu", seed=21, **CFG)


def inputs():
    rs = np.random.RandomState(21)
    enc = rs.randint(3, 120, (ROWS, TS))
    enc[:, 0] = 1
    for r in range(ROWS):
        e = rs.randint(6, TS + 1)
        enc[r, e - 1] = 2
        enc[r, e:] = 0
    dec = np.concatenate([np.ones((256, 1), int), rs.randint(3, 120, (256, 2))], 1)
    return enc, dec


class _Stub(object):
    def __init__(self, m):
        self.m = m

    def predict(self, x):
        return self.m.predict(x)


def main():
    bn = types.ModuleType("bottleneck")
    bn.argpartition = lambda a, k, axis=-1: np.argpartition(a, k, axis=axis)
    bn.partition = lambda a, k, axis=-1: np.partition(a, k, axis=axis)
    sys.modules["bottleneck"] = bn
    if not hasattr(np, "int"):
        np.int = int
    g = {"__name__": "ref_decoder", "print": lambda *a: None}
    src = os.path.join(ref_harness.REFERENCE_ROOT, "rl4rs", "mdpchecker", "decoder.py")
    exec(compile(open(src).read(), "decoder.py", "exec"), g)
    m = model()
    stub = _Stub(m)
    enc, dec = inputs()
    out = {"flat": m.flat.numpy(), "enc": enc.astype(np.uint8), "dec": dec.astype(np.uint8)}
    for beam, cand, rows in ((1, 0, ROWS), (20, 20, ROWS), (100, 0, 128)):
        p, s = g["beam_search"](stub, list(enc[:rows]), beam, 5, use_candidates=cand > 0, candidates_size=cand)
        out["path_%d_%d" % (beam, cand)] = np.asarray(p).astype(np.uint8)
        out["score_%d_%d" % (beam, cand)] = np.asarray(s, np.float32)
    out["step"] = np.asarray(g["decode_step"](stub, list(enc[:256]), dec, beam_size=10))
    out["probs"] = np.asarray(g["token_probs"](stub, list(enc[:256]), dec), np.float32)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
