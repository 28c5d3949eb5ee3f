"""Multi-GPU check of the peer-memory gradient exchange (csrc/r4_comm.cuh), one rank per GPU:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29511 tools/dist_check.py

1. r4_grad_exchange on random partial gradients, 40 consecutive steps (both parities, varying G): the result must
   equal the fixed-order sum (partials in CTA order, then ranks in rank order) BIT FOR BIT on every rank.
2. Two PPO iterations over the real env (256 rows per rank) through r4_ppo_epoch_dist: parameters stay bit-identical
   across ranks, and agree with the NCCL all-reduce path (same seeds) to fp32 summation-order tolerance.
3. Timing: SGD pass of one iteration, peer-memory path against the NCCL path.
Prints one JSON line on rank 0; exit code 0 = all checks passed."""
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    import __graft_entry__ as g
    g.build()
    from rl4rs_b200 import synth, gymshim, _capi
    from rl4rs_b200.env.slate import SlateRecEnv, SlateState
    from rl4rs_b200._capi import ptr as _p
    from rl4rs_b200.trainer import PPOTrainer, PeerComm
    lib = _capi.load_library()
    out = {"world": world}

    # ---- 1. raw exchange -------------------------------------------------------------------------
    A = 284
    n = lib.r4_policy_num_params(A)
    comm = PeerComm(n, dev)
    out["peer_comm"] = comm.ok
    if not comm.ok:
        out["why"] = comm.why
    ok = True
    if comm.ok:
        gen = torch.Generator(device="cpu").manual_seed(100 + rank)
        flat = torch.zeros(n, device=dev)
        stats = torch.zeros(5, device=dev)
        for step in range(40):
            G = 1 + (step * 7) % 64
            scratch = torch.randn(G * (n + 5), generator=gen).to(dev)
            rc = lib.r4_grad_exchange(comm.h, _p(scratch), G, A, _p(flat), _p(stats), 1.0,
                                      C.c_void_p(torch.cuda.current_stream().cuda_stream))
            assert rc == 0, lib.r4_last_error(None)
            part = scratch[:G * n].view(G, n)
            mine = part[0].clone()
            for c in range(1, G):
                mine = mine + part[c]
            every = [torch.empty_like(mine) for _ in range(world)]
            dist.all_gather(every, mine)
            want = every[0].clone() * 0.0
            for r in range(world):
                want = want + every[r]
            same = torch.equal(want.view(torch.int32), flat.view(torch.int32))
            ok = ok and same
            if not same and rank == 0:
                print("exchange mismatch at step", step, float((want - flat).abs().max()), file=sys.stderr)
        out["exchange_bit_exact_40_steps"] = ok
        comm.close()

    # ---- 2./3. trainer: peer path vs NCCL path ------------------------------------------------------
    B = 256
    cfg = {"maxlen": 64, "batch_size": B, "action_size": 284, "class_num": 2, "dense_feature_num": 432,
           "category_feature_num": 21, "category_hash_size": 100000, "seq_num": 2, "emb_size": 128, "hidden_units": 128,
           "max_steps": 9, "page_items": 9, "action_emb_size": 32, "is_eval": False, "cache_size": 2048,
           "support_rllib_mask": True, "output_format": "torch", "device": local}
    cat = synth.make_catalog()
    log = synth.make_log(4096, pages=1, catalog=cat, seed=synth.LOG_SEED + rank)
    w = synth.make_weights(cfg)

    def make_trainer(no_peer):
        if no_peer:
            os.environ["R4_NO_PEER_COMM"] = "1"
        else:
            os.environ.pop("R4_NO_PEER_COMM", None)
        sim = SlateRecEnv(dict(cfg, catalog=cat, log=log, weights=w), state_cls=SlateState)
        env = gymshim.make("SlateRecEnv-v0", recsim=sim)
        env.seed(rank)
        np.random.seed(rank)
        return PPOTrainer({"sgd_minibatch_size": 64 * world}, env, seed=0)

    res = {}
    for name, no_peer in (("peer", False), ("nccl", True)):
        tr = make_trainer(no_peer)
        for _ in range(2):
            st = tr.train()
        torch.cuda.synchronize()
        flat = tr.policy.flat.detach().clone()
        every = [torch.empty_like(flat) for _ in range(world)]
        dist.all_gather(every, flat)
        ident = all(torch.equal(every[0].view(torch.int32), e.view(torch.int32)) for e in every)
        # timing of the SGD pass alone
        buf = tr.buf
        ts = []
        for _ in range(3):
            dist.barrier(); torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.learn(buf)
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        res[name] = {"flat": flat, "replicas_bit_identical": ident, "uses_peer": bool(tr.comm and tr.comm.ok),
                     "sgd_pass_ms": 1e3 * min(ts), "sgd_steps": st["sgd_steps"], "total_loss": st["total_loss"]}
    d = (res["peer"]["flat"] - res["nccl"]["flat"]).abs().max().item()
    out["trainer"] = {k: {kk: vv for kk, vv in v.items() if kk != "flat"} for k, v in res.items()}
    out["peer_vs_nccl_max_abs_param_diff"] = d
    ok = ok and res["peer"]["replicas_bit_identical"] and res["nccl"]["replicas_bit_identical"] and d < 5e-5
    ok = ok and abs(res["peer"]["total_loss"] - res["nccl"]["total_loss"]) <= 1e-3 * abs(res["nccl"]["total_loss"])
    if comm.ok:
        ok = ok and res["peer"]["uses_peer"] and not res["nccl"]["uses_peer"]
    out["ok"] = bool(ok)
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print(json.dumps(out))
    dist.destroy_process_group()
    sys.exit(0 if flag.item() else 1)


if __name__ == "__main__":
    main()
