"""Time the MDP checker's kernels on one GPU (rl4rs_b200.mdpchecker, csrc/r4_seq2seq.cuh) at the script's model size
(embed_dim 256, FFN 128, one head, one encoder and one decoder block, dropout 0.05) on a synthetic rl4rs-sized sequence
set: ms per training step at batch 256 and 1024, one epoch, the three beam searches over 2048 rows, the Experiment I
scoring, launches per train and search step, peak device memory, and the torch twin's step for comparison.

    python tools/mdpcheck_time.py [--rows 40000] [--vocab 286]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from rl4rs_b200 import _capi  # noqa: E402
from rl4rs_b200.mdpchecker import decoder as dc  # noqa: E402
from rl4rs_b200.mdpchecker import transformer as tf  # noqa: E402


def timed(fn, reps=1):
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / reps * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=40000)
    ap.add_argument("--vocab", type=int, default=286)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    rs = np.random.RandomState(0)
    V, N = a.vocab, a.rows
    enc = np.concatenate([np.ones((N, 1), int), rs.randint(3, V, (N, 16)), np.full((N, 1), 2)], 1)
    tgt = rs.randint(3, V, (N, 5))
    dec = np.concatenate([np.ones((N, 1), int), tgt, np.full((N, 1), 2)], 1)
    out = np.concatenate([tgt, np.full((N, 1), 2), np.zeros((N, 1), int)], 1)
    lib = _capi.load_library()
    m = tf.get_model([V, V], 256, 1, 1, 1, 128, dropout_rate=0.05, use_same_embed=False, device="cuda")
    m.compile("adam", "sparse_categorical_crossentropy")
    res = {"device": torch.cuda.get_device_name(0)}
    for b in (256, 1024):
        m.grad(enc[:b], dec[:b], out[:b])
        n0 = lib.r4_s2s_launch_count()
        ms, _ = timed(lambda: m.apply(m.grad(enc[:b], dec[:b], out[:b])[1]), reps=20)
        res["train_step_ms_b%d" % b] = round(ms, 3)
        res["launches_per_train_step_b%d" % b] = (lib.r4_s2s_launch_count() - n0) // 20
    torch.cuda.reset_peak_memory_stats()
    np.random.seed(1)
    ms, _ = timed(lambda: m.fit([enc, dec], out, epochs=1, batch_size=256, verbose=0))
    res["epoch_s_%d_rows_b256" % N] = round(ms / 1e3, 3)
    ev = enc[:2048]
    for beam, cand in ((1, 0), (20, 20), (100, 0)):
        dc.beam_search(m, ev[:64], beam, 5, use_candidates=cand > 0, candidates_size=cand)
        torch.cuda.reset_peak_memory_stats()
        n0 = lib.r4_s2s_launch_count()
        ms, (path, _) = timed(lambda: dc.beam_search(m, ev, beam, 5, use_candidates=cand > 0, candidates_size=cand))
        res["search_ms_beam%d_cand%d" % (beam, cand)] = round(ms, 1)
        res["search_launches_beam%d_cand%d" % (beam, cand)] = lib.r4_s2s_launch_count() - n0
        res["search_peak_gb_beam%d" % beam] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    ms, _ = timed(lambda: dc.path_probs(m, ev, path))
    res["experiment_i_scoring_ms_beam100"] = round(ms, 1)
    cpu = tf.get_model([V, V], 256, 1, 1, 1, 128, dropout_rate=0.05, use_same_embed=False, device="cpu")
    cpu.compile("adam", "sparse_categorical_crossentropy")
    t = time.perf_counter()
    cpu.apply(cpu.grad(enc[:256], dec[:256], out[:256])[1])
    res["twin_cpu_train_step_ms_b256"] = round((time.perf_counter() - t) * 1e3, 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
