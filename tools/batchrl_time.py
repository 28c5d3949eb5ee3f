"""Time the batch-RL learners (csrc/r4_batchrl.cuh) on the GPU: SGD steps/s at minibatch 256 over back-to-back steps and
launches per step (counted by the library), one epoch over a synthetic dataset of the a-size (10^7 entries), and one
evaluate episode at batch 2048 with its act time (CUDA events) and the env-only rollout of the same episode; the torch twin's step on the same device for comparison.  Prints the
card name and power limit read in the same run.

    python tools/batchrl_time.py [--steps 2000] [--entries 10000000] [--algos BC,BCQ,CQL]
    python tools/batchrl_time.py --algo BCQ-conti CQL-conti   (the continuous learners on a continuous dataset, D 32)
"""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:
        return "nvidia-smi unavailable (%s)" % exc


def synthetic(N, K=266, L=10, seed=0):
    """N entries (episodes of L) in the writer's layout, built in chunks to bound host memory."""
    import numpy as np
    rs = np.random.RandomState(seed)
    obs = np.empty((N, K), np.float32)
    for s in range(0, N, 1 << 20):
        e = min(N, s + (1 << 20))
        obs[s:e] = rs.standard_normal((e - s, K)).astype(np.float32)
    obs[:, K - 10:K - 1] = rs.randint(0, 284, (N, 9))
    obs[:, K - 1] = np.arange(N) % L
    term = ((np.arange(N) % L) == L - 1).astype(np.float32)
    return {"observations": obs, "actions": rs.randint(0, 284, (N, 1)).astype(np.float32),
            "rewards": rs.rand(N).astype(np.float32), "terminals": term}


def sync_time(fn):
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def launches_per_step(m, data, perm, steps=20):
    """Kernel launches per SGD step of r4_batchrl_epoch, as the library counts them (r4_batchrl_launch_count)."""
    n0 = m.lib.r4_batchrl_launch_count()
    m._epoch_kernels(data, perm[:256 * steps])
    return (m.lib.r4_batchrl_launch_count() - n0) / steps


def synthetic_conti(N, K=266, D=32, L=10, seed=0):
    """N entries (episodes of L) with continuous actions f32 [N, D] in [-1, 1), built in chunks."""
    import numpy as np
    rs = np.random.RandomState(seed)
    obs = np.empty((N, K), np.float32)
    for s in range(0, N, 1 << 20):
        e = min(N, s + (1 << 20))
        obs[s:e] = rs.standard_normal((e - s, K)).astype(np.float32)
    act = (rs.rand(N, D).astype(np.float32) * 2 - 1)
    term = ((np.arange(N) % L) == L - 1).astype(np.float32)
    return {"observations": obs, "actions": act, "rewards": rs.rand(N).astype(np.float32), "terminals": term,
            "discrete_action": np.asarray(False)}


def eval_episode(ecfg, env, pol):
    """One evaluate episode (after a warm-up one): (episode s, act s by CUDA events, act calls, env-only rollout s)."""
    import torch
    for rep in range(2):
        events, actions = [], []
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        obs = env.reset()
        for _ in range(ecfg["max_steps"]):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            a = pol.predict_with_mask(obs)
            e1.record()
            events.append((e0, e1))
            actions.append(a)
            obs, _, _, _ = env.step(a)
        torch.cuda.synchronize()
        t_ep = time.perf_counter() - t0
    t_act = sum(e0.elapsed_time(e1) for e0, e1 in events) / 1e3
    t0 = time.perf_counter()
    env.reset()
    for a in actions:
        env.step(a)
    torch.cuda.synchronize()
    return t_ep, t_act, len(events), time.perf_counter() - t0


def conti(args):
    import torch
    from rl4rs_b200 import batchrl
    from test_gpu_parity import _synthetic
    print("card:", card())
    small = synthetic_conti(args.steps * 256 * 10 // 9 + 256 * 20)
    big = synthetic_conti(args.entries) if args.entries else None
    for algo in args.algo:
        cfg = {"action_size": 284, "action_emb_size": 32, "support_conti_env": True, "CQL_alpha": 1}
        m = batchrl.get_model(cfg, algo)
        m.build_with_dataset(small)
        data = m._device_data(small)
        perm = torch.randperm(data.n, device="cuda")[:256 * args.steps]
        m._epoch_kernels(data, perm[:256 * 20])                        # warm-up
        n0, s0 = m.lib.r4_batchrl_launch_count(), m.step
        t, _ = sync_time(lambda: m._epoch_kernels(data, perm))
        steps = m.step - s0
        print("%-9s kernel  %d steps of 256: %.1f steps/s (%.1f us/step), %.0f launches/step"
              % (algo, steps, steps / t, 1e6 * t / steps, (m.lib.r4_batchrl_launch_count() - n0) / steps))
        if big is not None:
            mb = batchrl.get_model(cfg, algo)
            t_up, _ = sync_time(lambda: mb.build_with_dataset(big) or mb._device_data(big))
            dn = mb._data.n
            t3, _ = sync_time(lambda: mb.fit(big, 1))
            print("%-9s epoch   %d entries, D 32 (%d transitions, %d steps): %.1f s (upload %.1f s)"
                  % (algo, args.entries, dn, dn // 256, t3, t_up))
            del mb
            torch.cuda.empty_cache()
        B = args.eval_batch
        ecfg, ecat, elog, w = _synthetic(B, False)
        ecfg = dict(ecfg, catalog=ecat, log=elog, weights=w, support_conti_env=True)
        env = batchrl.make_eval_env(ecfg, B)
        t_ep, t_act, k, t_env = eval_episode(ecfg, env, batchrl.policy_model(m, ecfg))
        print("%-9s evaluate one episode at B=%d: %.2f ms, act %.2f ms (CUDA events, %.3f ms/step), env-only rollout %.2f ms"
              % (algo, B, 1e3 * t_ep, 1e3 * t_act, 1e3 * t_act / k, 1e3 * t_env))
        del m
        torch.cuda.empty_cache()
    print("card:", card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--entries", type=int, default=10_000_000)
    ap.add_argument("--algos", default="BC,BCQ,CQL")
    ap.add_argument("--algo", nargs="+", choices=("BCQ-conti", "CQL-conti"),
                    help="time the continuous learners instead of the discrete ones")
    ap.add_argument("--eval-batch", type=int, default=2048)
    args = ap.parse_args()
    import numpy as np
    import torch
    import __graft_entry__ as g
    g.build()
    assert torch.cuda.is_available(), "tools/batchrl_time.py measures on a CUDA device"
    if args.algo:
        return conti(args)
    from rl4rs_b200 import batchrl, synth
    print("card:", card())
    cat = synth.make_catalog()
    small = synthetic(args.steps * 256 * 10 // 9 + 256 * 20)          # at least `steps` minibatches of transitions
    big = synthetic(args.entries) if args.entries else None
    for algo in args.algos.split(","):
        cfg = {"action_size": 284, "page_items": 9, "catalog": cat, "CQL_alpha": 1}
        m = batchrl.get_model(cfg, algo)
        m.build_with_dataset(small)
        data = m._device_data(small)
        perm = torch.randperm(data.n, device="cuda")[:256 * args.steps]
        m._epoch_kernels(data, perm[:256 * 20])                        # warm-up
        s0 = m.step
        t, _ = sync_time(lambda: m._epoch_kernels(data, perm))
        steps = m.step - s0
        print("%-4s kernel  %d steps of 256: %.1f steps/s (%.1f us/step), %.0f launches/step"
              % (algo, steps, steps / t, 1e6 * t / steps, launches_per_step(m, data, perm)))
        tw = batchrl.get_model(cfg, algo)
        tw.use_kernels = False
        tw.build_with_dataset(small)
        for k in range(5):
            tw.train_step_twin(data.batch(perm[k * 256:(k + 1) * 256]))
        nt = 200
        t2, _ = sync_time(lambda: [tw.train_step_twin(data.batch(perm[k * 256:(k + 1) * 256])) for k in range(nt)])
        print("%-4s twin    %d steps of 256: %.1f steps/s (%.1f us/step)" % (algo, nt, nt / t2, 1e6 * t2 / nt))
        del tw
        if big is not None:
            mb = batchrl.get_model(cfg, algo)
            t_up, _ = sync_time(lambda: mb.build_with_dataset(big) or mb._device_data(big))
            dn = mb._data.n
            t3, _ = sync_time(lambda: mb.fit(big, 1))
            print("%-4s epoch   %d entries (%d transitions, %d steps): %.1f s (upload %.1f s)"
                  % (algo, args.entries, dn, dn // 256, t3, t_up))
            del mb
            torch.cuda.empty_cache()
        # one evaluate episode at the eval batch, run as evaluate runs it (one synchronise at the end); the act calls timed
        # inside it by CUDA events; then the env-only rollout of the same episode (the same users, its actions replayed)
        from test_gpu_parity import _synthetic
        B = args.eval_batch
        ecfg, ecat, elog, w = _synthetic(B, False)
        ecfg = dict(ecfg, catalog=ecat, log=elog, weights=w)
        env = batchrl.make_eval_env(ecfg, B)
        pol = batchrl.policy_model(m, ecfg)
        for rep in range(2):                                           # the first episode warms up
            events, actions = [], []
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            obs = env.reset()
            for _ in range(ecfg["max_steps"]):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                a = pol.predict_with_mask(obs)
                e1.record()
                events.append((e0, e1))
                actions.append(a)
                obs, _, _, _ = env.step(a)
            torch.cuda.synchronize()
            t_ep = time.perf_counter() - t0
        t_act = sum(e0.elapsed_time(e1) for e0, e1 in events) / 1e3
        t0 = time.perf_counter()
        env.reset()
        for a in actions:
            env.step(a)
        torch.cuda.synchronize()
        t_env = time.perf_counter() - t0
        print("%-4s evaluate one episode at B=%d: %.2f ms, act %.2f ms (CUDA events, %.3f ms/step), env-only rollout %.2f ms"
              % (algo, B, 1e3 * t_ep, 1e3 * t_act, 1e3 * t_act / len(events), 1e3 * t_env))
        del m
        torch.cuda.empty_cache()
    print("card:", card())


if __name__ == "__main__":
    main()
