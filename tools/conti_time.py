"""Time one PPO_conti iteration on the device-resident path (rollout on the CUDA env + the Gaussian-policy learner) and,
in the same run, the env-only rollout of the same episode (one fixed action tensor, no policy).

    python tools/conti_time.py [--batch 8192 4096] [--iters 3] [--warmup 1]
    torchrun --nproc_per_node 4 tools/conti_time.py --batch 8192      (data-parallel learner over peer memory)

Prints one JSON line per batch size (rank 0) with the card name and power limit.  CUDA events around each phase, after
warm-up iterations of the same shapes."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else "?"
    except Exception as e:              # the timing stands without it; say why it is missing
        return "nvidia-smi unavailable: %s" % e


def main():
    import torch.distributed as dist
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[8192, 4096])
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if world > 1:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl")
    from test_gpu_parity import _synthetic, make_env
    from rl4rs_b200.trainer import get_rl_model
    for B in args.batch:
        cfg, cat, log, w = _synthetic(B, False, support_conti_env=True, is_eval=False, cache_size=4 * B)
        env = make_env(cfg, False, cat, log, w, output_format="torch")
        tr = get_rl_model("PPO_conti", {}, env=env)
        ev = lambda: torch.cuda.Event(enable_timing=True)

        a0 = torch.zeros(B, tr.D, device=tr.device)

        def env_only():
            env.reset()
            for _ in range(tr.T):
                env.step(a0)

        def one():
            e0, e1, e2, e3, e4 = ev(), ev(), ev(), ev(), ev()
            e0.record(); env_only(); e1.record()
            l0 = tr.ops.launches
            e2.record(); buf = tr.rollout(explore=True); e3.record()
            st = tr.learn(buf); e4.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1), e2.elapsed_time(e3), e3.elapsed_time(e4), st["sgd_steps"], tr.ops.launches - l0
        for _ in range(args.warmup):
            one()
        rows = [one() for _ in range(args.iters)]
        env_ms = sorted(r[0] for r in rows)[len(rows) // 2]
        roll_ms = sorted(r[1] for r in rows)[len(rows) // 2]
        learn_ms = sorted(r[2] for r in rows)[len(rows) // 2]
        steps, launches = rows[-1][3], rows[-1][4]
        act_launches = tr.T
        out = {"workload": "PPO_conti iteration", "batch_per_gpu": B, "world": world, "steps_per_episode": tr.T,
               "env_only_rollout_ms": round(env_ms, 2), "rollout_ms": round(roll_ms, 2), "learner_ms": round(learn_ms, 2),
               "sgd_steps": steps, "learner_launches_per_sgd_step": round((launches - act_launches - 1) / max(steps, 1), 2),
               "transitions_per_s": round(tr.T * B * world / ((roll_ms + learn_ms) / 1e3)),
               "learner_share": round(learn_ms / (roll_ms + learn_ms), 3), "card": card(), "iters_timed": args.iters}
        if rank == 0:
            print(json.dumps(out), flush=True)
        del tr, env
        torch.cuda.empty_cache()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
