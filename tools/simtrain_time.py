"""Time simulator training (csrc/r4_simtrain.cuh) on the GPU at the reference's sizes (category_hash_size 100000):
ms per optimiser step at batch 256 and 1024 over back-to-back steps, with the launches per step (counted by the library)
and samples/s; one steps_per_epoch epoch (2343 steps of 256) plus its validation (1562 batches); the torch twin's step on
the same card; and peak device memory.  Prints the card name and power limit read in the same run.  --model dien_slate /
dien_slate_multiclass times the slate-label nets instead (one sample per record, so samples/s reads records/s; no twin).

    python tools/simtrain_time.py [--model dien] [--steps 50] [--epoch-steps 2343] [--val-steps 1562] [--records 20000]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="dien", choices=["dien", "dien_slate", "dien_slate_multiclass"])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--epoch-steps", type=int, default=600000 // 256)
    ap.add_argument("--val-steps", type=int, default=400000 // 256)
    ap.add_argument("--records", type=int, default=20000)
    ap.add_argument("--twin-steps", type=int, default=2)
    a = ap.parse_args()
    import numpy as np
    import torch
    import simtrain_ref as R
    from rl4rs_b200 import simtrain, _capi
    assert torch.cuda.is_available(), "simtrain_time.py needs a CUDA device"
    print("card:", card())
    cfg = {"category_hash_size": 100000}
    samples = R.make_samples(a.records, 100000, seed=0)
    slate = a.model != "dien"
    if slate:
        samples = simtrain.SlateSamples.view(samples)
        print("model:", a.model)
    unit = "records" if slate else "samples"
    lib = _capi.load_library()
    for B in (256, 1024):
        tr = simtrain.get_model(cfg, a.model, device="cuda")
        st = simtrain._Stream(len(samples), B, 0, torch.device("cuda"))
        for _ in range(3):
            tr.train_step(samples, st.next())
        batches = [st.next() for _ in range(a.steps)]
        torch.cuda.synchronize()
        l0 = lib.r4_simtrain_launch_count()
        t = time.perf_counter()
        for b in batches:
            tr.train_step(samples, b)
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t) / a.steps
        launches = (lib.r4_simtrain_launch_count() - l0) / a.steps
        print("batch %d: %.2f ms/step, %.0f launches/step, %.0f %s/s" % (B, dt * 1e3, launches, B / dt, unit))
        del tr
    torch.cuda.reset_peak_memory_stats()
    tr = simtrain.get_model(cfg, a.model, device="cuda")
    test = R.make_samples(max(a.records // 4, 100), 100000, seed=1)
    if slate:
        test = simtrain.SlateSamples.view(test)
    torch.cuda.synchronize()
    t = time.perf_counter()
    h = tr.fit(samples, test, epochs=1, steps_per_epoch=a.epoch_steps, validation_steps=a.val_steps)
    torch.cuda.synchronize()
    print("one epoch of %d steps + %d validation batches: %.1f s  (loss %.4f val_loss %.4f)"
          % (a.epoch_steps, a.val_steps, time.perf_counter() - t, h["loss"][0], h["val_loss"][0]))
    print("peak device memory: %.2f GB" % (torch.cuda.max_memory_allocated() / 1e9))
    del tr
    if slate:
        return
    net = simtrain.SimulatorNet(cfg).cuda()
    m, v = torch.zeros_like(net.flat.data), torch.zeros_like(net.flat.data)
    idx = np.arange(256)
    cat, dense, seq, y = samples.features(idx)
    times = []
    for s in range(1, a.twin_steps + 2):
        torch.cuda.synchronize()
        t = time.perf_counter()
        keep = (torch.rand(256, 256) >= 0.2).to(torch.uint8)
        probs, _ = net(torch.from_numpy(cat).cuda(), torch.from_numpy(dense).cuda(), torch.from_numpy(seq).cuda(),
                       keep.cuda(), 0.2)
        loss = simtrain.keras_bce(probs, torch.from_numpy(y).cuda())
        net.flat.grad = None
        loss.backward()
        simtrain.keras_adam_(net.flat.data, net.flat.grad, m, v, s)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t)
    print("torch twin on the same card, batch 256: %.1f ms/step" % (1e3 * float(np.median(times[1:]))))


if __name__ == "__main__":
    main()
