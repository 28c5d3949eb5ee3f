"""Time the fp32-parity GEMM (k_gemm_tc) at its call sites over one env-only Slate episode at B = 4096: bench.py's
synthetic weights and log, the logged policy's actions, every kernel timed by the engine's CUDA events
(Engine.profile(2), one stream).  Per GEMM profile slot: ms per episode, launches, the algorithmic fp32 rate
(2 M N K per launch), the bf16 tensor rate it issues (x 6 products of the 3-way split) and the fraction of the floor.

Floor of a slot = the larger of its bf16 tensor work at --tflops (700 TFLOP/s by default, about 70 % of the data
sheet's dense 989) and, for the sequence-mode projections (K = 128), its output bytes at --hbm (3.35 TB/s).  Computed
from shapes, not measured.  Median over --reps episodes after one warm-up episode.

    python tools/gemm_time.py [--batch 4096] [--reps 3] [--simulator dien|dnn]
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PRODUCTS = 6                  # bf16 products per fp32 product (r4_gemm_tc.cuh)
PROJ_K = 128                  # K of the two sequence-mode input projections (emb_size)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "%s, power limit unknown" % torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--simulator", default="dien", choices=["dien", "dnn"])
    ap.add_argument("--tflops", type=float, default=700.0)
    ap.add_argument("--hbm", type=float, default=3.35)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from bench import base_config
    from rl4rs_b200 import synth, gymshim
    from rl4rs_b200.env.slate import SlateRecEnv, SlateState

    B = args.batch
    cfg = base_config(B, simulator=args.simulator)
    catalog = synth.make_catalog()
    log = synth.make_log(max(4 * B, 8192), pages=1, catalog=catalog, seed=synth.LOG_SEED)
    weights = synth.make_dnn_weights(cfg) if args.simulator == "dnn" else synth.make_weights(cfg)
    sim = SlateRecEnv(dict(cfg, catalog=catalog, log=log, weights=weights, output_format="torch"), state_cls=SlateState)
    env = gymshim.make("SlateRecEnv-v0", recsim=sim)
    env.seed(0)
    eng = sim.engine

    def episode():
        env.reset()
        for _ in range(cfg["max_steps"]):
            env.step(env.offline_action)
        torch.cuda.synchronize()

    episode()
    runs = []
    for _ in range(args.reps):
        eng.profile(2)
        episode()
        runs.append({p["name"]: p for p in eng.profile_read()})
        eng.profile(0)
    name = card()
    total = [sum(p["ms"] for p in r.values()) for r in runs]
    print("one env-only Slate episode, B=%d, %s simulator: %.2f ms of kernel time (median of %d) | %s"
          % (B, args.simulator, float(np.median(total)), len(runs), name))
    print("%-42s %9s %8s %9s %10s %9s %6s" % ("slot", "ms", "launches", "TFLOP/s", "bf16 TF/s", "floor ms", "floor"))
    for slot in sorted(runs[0]):
        if not slot.startswith("k_gemm_tc"):
            continue
        ms = float(np.median([r[slot]["ms"] for r in runs]))
        p = runs[0][slot]
        work = p["work"]
        floor = PRODUCTS * work / (args.tflops * 1e12) * 1e3
        if "input proj" in slot:          # M N fp32 outputs written once: work / (2 K) x 4 bytes
            floor = max(floor, work / (2 * PROJ_K) * 4 / (args.hbm * 1e12) * 1e3)
        print("%-42s %9.3f %8d %9.1f %10.1f %9.3f %6.2f"
              % (slot, ms, p["launches"], work / (ms / 1e3) / 1e12, PRODUCTS * work / (ms / 1e3) / 1e12, floor,
                 floor / ms), flush=True)


if __name__ == "__main__":
    main()
