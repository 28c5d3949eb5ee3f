"""Time the AUGRU recurrence kernel (k_augru_tc) alone at the two launch shapes of a Slate episode at B = 4096: an
observation pass (4096 rows, one CTA wave) and the reward pass (36 864 rows, several waves).  bench.py's synthetic
weights, `dien_forward` on random feature rows, the kernel timed by the engine's CUDA events (Engine.profile(1));
median of --reps launches after a warm-up.

    python tools/augru_time.py [--reps 7] [--rows 4096,36864]
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

IMAGE_BYTES = 786432          # recurrent weight image streamed per CTA and step (r4_recur.cuh: AU_IMAGE_BYTES)
STEPS = 64


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "%s, power limit unknown" % torch.cuda.get_device_name()


def rows(R, seed):
    rs = np.random.RandomState(seed)
    seq = rs.randint(1, 284, (R, 2, 64)).astype(np.int32)
    dense = rs.normal(0, 2, (R, 432)).astype(np.float32)
    cat = rs.randint(0, 100000, (R, 21)).astype(np.int32)
    return seq, dense, cat


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--rows", default="4096,36864")
    args = ap.parse_args()
    from rl4rs_b200 import synth, gymshim
    from rl4rs_b200.env.slate import SlateRecEnv, SlateState
    cfg = {"maxlen": 64, "batch_size": 8, "action_size": 284, "class_num": 2, "dense_feature_num": 432,
           "category_feature_num": 21, "category_hash_size": 100000, "seq_num": 2, "emb_size": 128,
           "hidden_units": 128, "max_steps": 9, "page_items": 9, "action_emb_size": 32, "is_eval": True,
           "cache_size": 8}
    cat = synth.make_catalog()
    log = synth.make_log(32, pages=1, catalog=cat, hash_size=100000)
    sim = SlateRecEnv(dict(cfg, catalog=cat, log=log, weights=synth.make_weights(cfg)), state_cls=SlateState)
    gymshim.make("SlateRecEnv-v0", recsim=sim)
    eng = sim.engine
    sms = torch.cuda.get_device_properties(eng.device).multi_processor_count
    name = card()
    for R in [int(r) for r in args.rows.split(",")]:
        seq, dense, catf = rows(R, R)
        eng.dien_forward(seq, dense, catf)                 # warm-up: workspaces, first launch
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.reps):
            eng.profile(1)
            eng.dien_forward(seq, dense, catf)
            torch.cuda.synchronize()
            k = [p for p in eng.profile_read() if p["name"].startswith("k_augru")]
            eng.profile(0)
            if not k:
                raise SystemExit("no k_augru_tc launch was timed")
            ms.append(k[0]["ms"] / k[0]["launches"])
            work = k[0]["work"] / k[0]["launches"]
        t = float(np.median(ms))
        ctas = 2 * ((R + 63) // 64)
        waves = (ctas + sms - 1) // sms
        print("k_augru_tc R=%d: %.3f ms/launch (min %.3f max %.3f, %d reps), %.2f us/step per wave (%d CTAs, %d waves), "
              "%.1f TFLOP/s, weight stream %.2f TB/s | %s"
              % (R, t, min(ms), max(ms), len(ms), t * 1e3 / (waves * STEPS), ctas, waves, work / (t / 1e3) / 1e12,
                 ctas * IMAGE_BYTES * STEPS / (t / 1e3) / 1e12, name), flush=True)


if __name__ == "__main__":
    main()
