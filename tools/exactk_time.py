"""Time Exact-K's train and eval stages on the CUDA env (synthetic log and DIEN weights), per episode:

  rollout ms    the two sampled decodes and their 18 env steps and three resets
  decode ms     the two sampled decodes alone (CUDA events around r4_exactk_decode)
  critic ms     the critic's prediction, its step and its Adam
  gen ms        the generator's teacher-forced forward, backward and Adam
  launches      r4_exactk_launch_count per episode
  peak MB       torch's peak device memory (the env's and the learners' buffers)
and the greedy eval batch (one decode and nine env steps).  Needs a CUDA device.

    python tools/exactk_time.py [--batch 256 2048] [--episodes 5] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _gpu():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def run(B, episodes, warmup):
    from rl4rs_b200 import _capi
    from rl4rs_b200 import exactk as ek
    from test_gpu_parity import _synthetic, make_env
    lib = _capi.load_library()
    cfg, cat, log, w = _synthetic(B, False, is_eval=False, n_log=4 * B, cache_size=4 * B)
    env = make_env(cfg, False, cat, log, w, output_format="torch")
    gen, critic = ek.build_nets(dict(cfg, catalog=cat), torch.device("cuda"))
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(8)]
    rows = []
    torch.cuda.reset_peak_memory_stats()
    for ep in range(warmup + episodes):
        c0 = lib.r4_exactk_launch_count()
        ev[0].record()
        obs = env.reset()
        paths, dec = [], 0.0
        for _ in range(2):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            p, _ = gen.draw(obs, ek.SAMPLE)
            b.record()
            for s in range(9):
                _, reward, _, _ = env.step(p[:, s])
            env.reset()
            paths.append((p, reward, a, b))
        ev[1].record()
        (p0, r0, a0, b0), (p1, r1, a1, b1) = paths
        second = r1 > r0
        target, reward = torch.where(second.unsqueeze(1), p1, p0), torch.where(second, r1, r0)
        reward_ = critic.predict(obs)
        critic.train(obs, reward)
        ev[2].record()
        adv = reward - reward_
        adv = adv / adv.double().std(unbiased=False).float()
        ev[3].record()
        gen.train(obs, target, adv)
        ev[4].record()
        torch.cuda.synchronize()
        if ep >= warmup:
            rows.append({"rollout_ms": ev[0].elapsed_time(ev[1]), "decode_ms": a0.elapsed_time(b0) + a1.elapsed_time(b1),
                         "critic_ms": ev[1].elapsed_time(ev[2]), "gen_ms": ev[3].elapsed_time(ev[4]),
                         "launches": lib.r4_exactk_launch_count() - c0})
    evals = []
    for i in range(warmup + 3):
        ev[5].record()
        obs = env.reset()
        p, _ = gen.draw(obs, ek.GREEDY)
        for s in range(9):
            env.step(p[:, s])
        ev[6].record()
        torch.cuda.synchronize()
        if i >= warmup:
            evals.append(ev[5].elapsed_time(ev[6]))
    med = {k: sorted(r[k] for r in rows)[len(rows) // 2] for k in rows[0]}
    return dict(med, batch=B, episodes=episodes, eval_batch_ms=sorted(evals)[len(evals) // 2],
                peak_mb=torch.cuda.max_memory_allocated() / 2 ** 20,
                generator_scratch_mb=lib.r4_exactk_scratch_size(0, B, 284) / 2 ** 20)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[256, 2048])
    ap.add_argument("--episodes", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("exactk_time.py needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    print(json.dumps({"gpu": _gpu()}))
    for B in a.batch:
        print(json.dumps({k: (round(v, 3) if isinstance(v, float) else v) for k, v in run(B, a.episodes, a.warmup).items()}))
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
