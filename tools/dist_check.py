"""Timing of the data-parallel PPO learner, one rank per GPU:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29511 tools/dist_check.py

The SGD pass of one iteration (256 env rows per rank), the peer-memory path against the NCCL path.  Correctness lives in
tests/test_gpu_comm.py (the exchange, every learner's data-parallel step, and the trainers' peer path against NCCL).
Prints one JSON line on rank 0."""
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
    from rl4rs_b200.trainer import PPOTrainer, PeerComm
    out = {"world": world}

    lib = _capi.load_library()
    n = lib.r4_policy_num_params(284)
    comm = PeerComm(n, dev)           # whether this box maps its peers (the trainers build their own)
    out["peer_comm"] = comm.ok
    if not comm.ok:
        out["why"] = comm.why
    comm.close()

    # ---- 1./2. trainer: peer path vs NCCL path ------------------------------------------------------
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
        # timing of the SGD pass alone
        buf = tr.buf
        ts = []
        for _ in range(3):
            dist.barrier(); torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.learn(buf)
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        res[name] = {"uses_peer": bool(tr.comm and tr.comm.ok), "sgd_pass_ms": 1e3 * min(ts), "sgd_steps": st["sgd_steps"]}
    out["trainer"] = res
    if rank == 0:
        print(json.dumps(out))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
