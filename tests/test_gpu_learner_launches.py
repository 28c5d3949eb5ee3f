"""GPU: the library's learner launch count (r4_learner_launch_count) against the launch structure of each learner path --
the per-call kernel counts the trainers once re-derived by hand -- and no count for a call rejected on its arguments; the
shared-memory opt-in above 48 KB on every device a process drives."""
import ctypes as C

import pytest

pytestmark = pytest.mark.gpu


def _lib():
    from rl4rs_b200 import _capi
    return _capi.load_library()


def _launched(fn):
    """-> the learner kernels fn launched, as the library counts them."""
    import torch
    lib = _lib()
    n0 = lib.r4_learner_launch_count()
    fn()
    torch.cuda.synchronize()
    return lib.r4_learner_launch_count() - n0


def _rejected(fn):
    """fn must fail on its arguments (R4Error) and launch nothing."""
    from rl4rs_b200 import _capi

    def call():
        with pytest.raises(_capi.R4Error, match="bad argument"):
            fn()
    assert _launched(call) == 0


def _ppo_data(ops, pol, n, dev):
    import torch
    from test_gpu_trainer import _random_batch
    obs, mask = _random_batch(n, pol.A, dev)
    act = torch.empty(n, dtype=torch.int32, device=dev)
    lp, v, lg = torch.empty(n, device=dev), torch.empty(n, device=dev), torch.empty(n, pol.A, device=dev)
    assert _launched(lambda: ops.act(pol.flat, obs, mask, True, 1, act, lp, v, lg)) == 1
    g = torch.Generator().manual_seed(4)
    adv, tgt = torch.randn(n, generator=g).to(dev), torch.randn(n, generator=g).to(dev)
    return (obs, mask, act.long(), lp, lg, v, adv, tgt)


HP = {"clip": 0.3, "vf_clip": 500.0, "vf_coeff": 0.5, "kl_coeff": 0.2, "ent_coeff": 0.01}


def test_ppo_and_a2c_launches():
    import torch
    from rl4rs_b200.policy import MaskedPolicy
    from rl4rs_b200.trainer import KernelOps
    dev = torch.device("cuda")
    A, n, mb = 284, 300, 64
    pol = MaskedPolicy(A, dev, seed=3)
    ops = KernelOps(A, dev, pol.n_params)
    data = _ppo_data(ops, pol, n, dev)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(2)).to(dev)
    flat = pol.flat.detach().clone()
    for clip in (None, 0.5):      # fused: k_policy_grad + k_reduce_adam; clipped: + k_grad_reduce, k_sumsq_one, k_adam
        rc = []
        assert _launched(lambda: rc.append(ops.ppo_epoch(flat, data, perm, n, mb, HP, 1e-3, clip))) == \
            n // mb * (4 if clip else 2)
        assert rc == [n // mb]
    for clip in (None, 10.0):     # A2C: k_policy_grad + k_grad_reduce, then k_adam (after k_sumsq_one when clipping)
        def a2c():
            ops.policy_grad(1, flat, data, None, 0, n, HP, 1.0, 1.0 / n)
            ops.adam(flat, 1e-3, 1.0, clip)
        assert _launched(a2c) == 2 + (2 if clip else 1)
    assert _launched(lambda: ops.gae(torch.randn(9, 40, device=dev), torch.randn(9, 40, device=dev), 1.0, 1.0)) == 1
    _rejected(lambda: ops.ppo_epoch(flat, data, perm, n, 0, HP, 1e-3, None))
    _rejected(lambda: ops.policy_grad(0, flat, data, None, 0, 0, HP, 1.0, 1.0))


def test_gauss_ppo_launches_per_chunk():
    import torch
    from test_gpu_trainer_conti import D, _batch, _policy
    from rl4rs_b200.trainer import GaussKernelOps
    dev = torch.device("cuda")
    pol = _policy(dev)
    ops = GaussKernelOps(D, dev, pol.n_params)
    n = 2500                      # one minibatch of 2500 samples: two chunks of k_gauss_rows + k_dense_wgrad (CH = 2048)
    data = _batch(pol, n, dev)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(2)).to(dev)
    chunks = lambda k: 2 * -(-k // 2048)
    flat = pol.flat.detach().clone()
    for clip in (None, 0.5):
        assert _launched(lambda: ops.ppo_epoch(flat, data, perm, n, n, HP, 1e-3, clip)) == chunks(n) + (2 if clip else 1)
    assert _launched(lambda: ops.policy_grad(1, flat, data, None, 0, 300, HP, 1.0, 1.0)) == chunks(300)
    _rejected(lambda: ops.ppo_epoch(flat, data, perm, n, 0, HP, 1e-3, None))


@pytest.mark.parametrize("algo", ["DDPG", "TD3"])
@pytest.mark.parametrize("prio", [True, False])
def test_ddpg_train_step_launches(algo, prio):
    import torch
    from test_gpu_trainer_ddpg import _fill, _pair
    tk, _ = _pair(algo, prioritized_replay=prio, train_batch_size=64)
    _fill((tk,))
    assert (tk.replay.prio is not None) == prio
    draws = tk.draws()            # sample, rows, weight gradient, apply (+ priorities)
    assert _launched(lambda: tk.sgd_step(*draws)) == (5 if prio else 4)
    empty = torch.empty(0, device="cuda")
    _rejected(lambda: tk.ops.train_step(None, tk.policy, tk.replay, empty, draws[1], 1, 1, tk._hp()))


def test_rainbow_train_step_launches():
    import torch
    from test_gpu_trainer_rainbow import _fill, _pair
    tk, _ = _pair(train_batch_size=64)
    _fill((tk,))
    assert tk.replay.prio is not None
    draws = tk.draws()
    assert _launched(lambda: tk.sgd_step(*draws)) == 5
    _rejected(lambda: tk.ops.train_step(None, tk.policy, tk.replay, torch.empty(0, device="cuda"), 1, False, tk._hp()))


@pytest.mark.parametrize("algo", ["BC", "BCQ", "CQL"])
def test_batchrl_epoch_launches(algo):
    import torch
    from test_gpu_batchrl import _dataset, _model
    from rl4rs_b200 import batchrl
    lib = _lib()
    ds = _dataset(266, E=60, L=10)
    m = _model(algo, 266, ds, batch_size=25, target_update_interval=5)
    data = m._device_data(ds)
    perm = torch.randperm(data.n, generator=torch.Generator(device="cuda").manual_seed(2), device="cuda")[:100]
    b0 = lib.r4_batchrl_launch_count()
    per_step = 3 + (algo != "CQL")    # rows, weight gradient, apply, and the embedding gradient of BC's / BCQ's nets
    assert _launched(lambda: m._epoch_kernels(data, perm)) == 4 * per_step
    assert lib.r4_batchrl_launch_count() - b0 == 4 * per_step
    n0, b0 = lib.r4_learner_launch_count(), lib.r4_batchrl_launch_count()
    rc = lib.r4_batchrl_epoch(batchrl.ALGOS[algo], m.net.K, m.A, C.c_void_p(m.net.flat.data_ptr()),
                              C.c_void_p(m.net.target.data_ptr()), C.c_void_p(m.m.data_ptr()), C.c_void_p(m.v.data_ptr()),
                              C.byref(m._tables.data(data)), C.byref(m._hyper_c()), C.c_void_p(perm.data_ptr()),
                              perm.numel(), 0, m.step, 1e-4, 1e-8, 0, C.c_void_p(m.scratch.data_ptr()), None, m._stream())
    assert rc == -1 and lib.r4_learner_launch_count() == n0 and lib.r4_batchrl_launch_count() == b0


def test_simtrain_step_launches():
    import torch
    import simtrain_ref as R
    from rl4rs_b200 import simtrain
    lib = _lib()
    H = 3000
    samples = R.make_samples(300, H, seed=11)
    tr = simtrain.SimulatorTrainer({"category_hash_size": H}, device="cuda", data_seed=3)
    idx = torch.arange(64, dtype=torch.int64, device="cuda")
    s0 = lib.r4_simtrain_launch_count()
    assert _launched(lambda: tr.train_step(samples, idx)) == 59     # DESIGN.md: 59 launches per step, the sort counted once
    assert lib.r4_simtrain_launch_count() - s0 == 59
    n0 = lib.r4_learner_launch_count()
    rc = lib.r4_simtrain_step(H, C.c_void_p(tr.params.data_ptr()), C.c_void_p(tr.grad.data_ptr()), C.c_void_p(tr.m.data_ptr()),
                              C.c_void_p(tr.v.data_ptr()), C.byref(tr._data(samples)), C.c_void_p(idx.data_ptr()), 0, 3, 1,
                              0.2, 1, 1e-3, 0.9, 0.999, 1e-7, C.c_void_p(tr._scratch(64).data_ptr()), None, None, None)
    assert rc == -1 and lib.r4_learner_launch_count() == n0


def test_shared_memory_opt_in_on_every_device():
    """k_ddpg_rows asks for more than 48 KB of shared memory: the opt-in is per device, so a launch on the second device
    after one on the first must succeed too."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two devices")
    lib = _lib()
    D, n, rows = 8, 16, 32
    np_ = lib.r4_ddpg_num_params(D, 0)
    for d in range(2):
        dev = torch.device("cuda", d)
        with torch.cuda.device(dev):
            z = lambda *s: torch.zeros(*s, device=dev)
            prm, obs, act, new_obs = z(np_), z(rows, 256), z(rows, D), z(rows, 256)
            rew, done = z(rows), torch.zeros(rows, dtype=torch.uint8, device=dev)
            idx = torch.arange(n, dtype=torch.int64, device=dev)
            scratch, grad, td, stats = z(lib.r4_ddpg_scratch_size(D, 0, n)), z(np_), z(n), z(3)
            p = lambda t: C.c_void_p(t.data_ptr())
            rc = lib.r4_ddpg_grad(p(prm), p(prm), D, 0, p(obs), p(act), p(rew), p(new_obs), p(done), p(idx), None, None, n,
                                  0.99, 0.2, 0.5, 1.0 / n, p(scratch), p(grad), p(td), p(stats),
                                  C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
            torch.cuda.synchronize(dev)
            assert rc == 0, (d, (lib.r4_last_error(None) or b"?").decode())
