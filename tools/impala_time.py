"""Time one PG and one IMPALA iteration on the device-resident path (rollout on the CUDA env + the learner kernels).

    python tools/impala_time.py [--algo PG IMPALA] [--batch 4096 8192] [--iters 3] [--warmup 1]

Prints one JSON line per algorithm and batch size with the rollout and learner times (CUDA events, median of the timed
iterations after warm-up iterations of the same shapes), the kernels one learner step launches as the library counts them,
transitions per second of the whole iteration, and the card name and power limit."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--algo", nargs="+", default=["PG", "IMPALA"])
    ap.add_argument("--batch", type=int, nargs="+", default=[4096, 8192])
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    from conti_time import card
    from test_gpu_parity import _synthetic, make_env
    from rl4rs_b200.trainer import get_rl_model
    for algo in args.algo:
        for B in args.batch:
            cfg, cat, log, w = _synthetic(B, False, support_rllib_mask=True, is_eval=False, cache_size=4 * B)
            env = make_env(cfg, False, cat, log, w, output_format="torch")
            tr = get_rl_model(algo, {}, env=env)
            ev = lambda: torch.cuda.Event(enable_timing=True)

            def one():
                e0, e1, e2 = ev(), ev(), ev()
                e0.record(); buf = tr.rollout(explore=True); e1.record()
                l0 = tr.ops.launches
                st = tr.learn(buf); e2.record()
                torch.cuda.synchronize()
                return e0.elapsed_time(e1), e1.elapsed_time(e2), (tr.ops.launches - l0) / st["sgd_steps"]
            for _ in range(args.warmup):
                one()
            rows = [one() for _ in range(args.iters)]
            med = lambda k: sorted(r[k] for r in rows)[len(rows) // 2]
            roll_ms, learn_ms = med(0), med(1)
            print(json.dumps({"workload": "%s iteration" % algo, "batch": B, "steps_per_episode": tr.T,
                              "rollout_ms": round(roll_ms, 2), "learner_ms": round(learn_ms, 3),
                              "learner_launches_per_step": rows[-1][2],
                              "transitions_per_s": round(tr.T * B / ((roll_ms + learn_ms) / 1e3)),
                              "learner_share": round(learn_ms / (roll_ms + learn_ms), 4), "card": card(),
                              "iters_timed": args.iters}), flush=True)
            del tr, env
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
