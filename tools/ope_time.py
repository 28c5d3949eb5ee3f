"""Time one `ope` epoch (rl4rs_b200.offline_evaluation.ope_eval) on one GPU at the scripts' batch of 2048, on Slate (T = 9)
and SeqSlate (T = 36), for a batch-RL model (BC) and a PPO trainer with seeded weights, over a synthetic log ingested
from text.  The epoch is split into the env rollout, the policy act, the host parsing per reset, the behaviour forward
per page, the step gathers and the host estimators (each part ends in a device synchronise, so the parts add up to more
than an unsynchronised epoch).  Prints the card name and power limit read in the same run, then one JSON line.

    python tools/ope_time.py [--batch 2048] [--reps 3]
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from rl4rs_b200 import batchrl, offline_evaluation as oe, synth, trainer  # noqa: E402
from rl4rs_b200.utils.datautil import FeatureUtil  # noqa: E402
from test_gpu_parity import make_env  # noqa: E402


def _env(seq, B, rllib, d3rl):
    cfg = {"maxlen": 64, "batch_size": B, "action_size": 284, "class_num": 2, "dense_feature_num": 432,
           "category_feature_num": 21, "category_hash_size": 5000, "seq_num": 2, "emb_size": 128, "hidden_units": 128,
           "max_steps": 36 if seq else 9, "page_items": 9, "action_emb_size": 32, "is_eval": True, "cache_size": B,
           "support_rllib_mask": rllib, "support_d3rl_mask": d3rl, "epoch": 1}
    cat = synth.make_catalog()
    log = synth.make_log(B, pages=4 if seq else 1, catalog=cat, hash_size=5000, keep_hist=True)
    log = FeatureUtil.parse_log(synth.render_records(log, cat))
    w = synth.make_weights(cfg, stress=2.0, bias_noise=0.1, bounded_scores=True)
    return dict(cfg, catalog=cat), make_env(cfg, seq, cat, log, w, output_format="torch")


class Spans(object):
    def __init__(self):
        self.ms = {}

    @contextlib.contextmanager
    def __call__(self, name):
        torch.cuda.synchronize()
        t = time.perf_counter()
        yield
        torch.cuda.synchronize()
        self.ms[name] = self.ms.get(name, 0.0) + (time.perf_counter() - t) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    tmp = tempfile.mkdtemp()
    wfile = os.path.join(tmp, "logged_policy.npz")
    rs = np.random.RandomState(1)
    np.savez(wfile, **{n: (rs.standard_normal(s) / np.sqrt(s[0] if len(s) == 2 else 100)).astype(np.float32)
                       for n, _, s in oe.dnn_plan(100000, 284)})
    out = {"card": card, "batch": a.batch}
    for seq in (False, True):
        for algo in ("BC", "PPO"):
            cfg, env = _env(seq, a.batch, algo == "PPO", algo != "PPO")
            if algo == "BC":
                model = batchrl.get_model(cfg, "BC")
                model.create_impl(env.observation_space.shape[0])
            else:
                model = trainer.get_rl_model("PPO", {}, env, seed=0)
            bm = oe.behavior_model(cfg, wfile, device="cuda")
            with contextlib.redirect_stdout(io.StringIO()):
                oe.ope_eval(cfg, env, model, sample_model=bm)                 # warm-up: every shape of the timed epochs
            best = None
            for _ in range(a.reps):
                spans = Spans()
                torch.cuda.synchronize()
                t = time.perf_counter()
                with contextlib.redirect_stdout(io.StringIO()):
                    oe.ope_eval(cfg, env, model, sample_model=bm, timer=spans)
                spans.ms["epoch"] = (time.perf_counter() - t) * 1e3
                if best is None or spans.ms["epoch"] < best["epoch"]:
                    best = spans.ms
            key = "%s_%s_T%d" % ("seqslate" if seq else "slate", algo, cfg["max_steps"])
            out[key] = {k: round(v, 2) for k, v in best.items()}
            print(key, out[key])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
