"""Time RAINBOW on the device-resident path: one vector episode of rollout (act kernel + CUDA env), its n-step store into the
replay, the learner of one iteration, and back-to-back SGD steps on a filled buffer; in the same run, the env-only rollout
of the same episode (one fixed action tensor, no policy).

    python tools/rainbow_time.py [--batch 4096 8192] [--iters 3] [--warmup 1] [--steps 100]

Prints one JSON line per batch with the card name and power limit.  CUDA events around each phase, after warm-up calls of
the same shapes; medians over --iters."""
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
    from conti_time import card
    from test_gpu_parity import _synthetic, make_env
    from rl4rs_b200.trainer import get_rl_model
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[4096, 8192])
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--steps", type=int, default=100)
    args = ap.parse_args()
    name = card()
    med = lambda xs: sorted(xs)[len(xs) // 2]
    for B in args.batch:
        cfg, cat, log, w = _synthetic(B, False, support_rllib_mask=False, is_eval=False, cache_size=4 * B)
        env = make_env(cfg, False, cat, log, w, output_format="torch")
        # the default ring (100 000 transitions), learning from the first episode on
        tr = get_rl_model("RAINBOW", {"learning_starts": 0}, env=env)
        ev = lambda: torch.cuda.Event(enable_timing=True)
        a0 = torch.zeros(B, dtype=torch.int32, device=tr.device)

        def env_only():
            env.reset()
            for _ in range(tr.T):
                env.step(a0)

        def episode():
            e = [ev() for _ in range(6)]
            e[0].record(); env_only(); e[1].record()
            e[2].record(); tr.rollout(explore=True); e[3].record()
            tr.replay.store(tr.buf_obs, tr.final_obs, tr.buf_action, tr.buf_reward, tr.buf_done); e[4].record()
            tr.sgd_step(*tr.draws()); e[5].record()
            torch.cuda.synchronize()
            return [e[0].elapsed_time(e[1]), e[2].elapsed_time(e[3]), e[3].elapsed_time(e[4]), e[4].elapsed_time(e[5])]

        for _ in range(args.warmup):
            episode()
        rows = [episode() for _ in range(args.iters)]
        env_ms, roll_ms, store_ms, learn_ms = (med([r[k] for r in rows]) for k in range(4))
        l0 = tr.ops.launches
        s0, s1 = ev(), ev()
        s0.record()
        for _ in range(args.steps):
            tr.sgd_step(*tr.draws())
        s1.record()
        torch.cuda.synchronize()
        per_step = s0.elapsed_time(s1) / args.steps
        out = {"workload": "RAINBOW episode", "batch_per_gpu": B, "steps_per_episode": tr.T, "train_batch_size": tr.n_local,
               "env_only_rollout_ms": round(env_ms, 2), "rollout_ms": round(roll_ms, 2), "store_ms": round(store_ms, 3),
               "learner_ms_per_iteration": round(learn_ms, 3), "sgd_step_ms_back_to_back": round(per_step, 3),
               "launches_per_sgd_step": (tr.ops.launches - l0) / args.steps + 1,       # + the uniforms' draw
               "transitions_per_s": round(tr.T * B / ((roll_ms + store_ms + learn_ms) / 1e3)),
               "replay_size": tr.replay.size, "card": name, "iters_timed": args.iters}
        print(json.dumps(out), flush=True)
        del tr, env
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
