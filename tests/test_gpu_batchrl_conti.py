"""GPU: the continuous-action CQL kernels (csrc/r4_cqlconti.cuh) against the torch twin (policy.BatchRLContiNet) in float64
-- every group's gradient over the C-ABI's shape grid, chained epochs, determinism, argument checks, predict -- and the
train / eval stages end to end on the CUDA env."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LAUNCHES_PER_STEP = 56      # DESIGN.md section 4
BCQ_LAUNCHES_PER_STEP = 69


def _model(K, D, ds, algo="CQL-conti", **hp):
    from rl4rs_b200 import batchrl
    m = batchrl.get_model({"action_size": 284, "action_emb_size": D, "support_conti_env": True}, algo)
    m.hp.update(hp)
    m.batch_size = int(m.hp["batch_size"])
    m.build_with_dataset(ds)
    assert m.use_kernels and m.net.K == K
    return m


def _dataset(K, D, E=60, L=10, seed=0):
    from test_batchrl_conti_cpu import conti_dataset
    return conti_dataset(K, D, E, L, seed)


def _tensors(net):
    import math
    off, out = 0, []
    for name, shape in net._shapes:
        k = math.prod(shape)
        out.append((name, slice(off, off + k)))
        off += k
    return out


def _edge_rows(net, flat, batch, noise, S, tol=1e-5):
    """The minibatch rows whose gradient meets a discrete edge within float32 roundoff (DESIGN.md section 7): a relu
    pre-activation of the critics on the critic-phase or actor-phase rows, or of the actor on s, within tol times the
    layer's rms times sqrt(max(1, K_in / 256)) of zero (learner_ref64.RELU_TIE's unit); the two critics' Q at the actor's
    sample within 1e-4 of each other (relative); a raw logstd within 1e-5 of its clamp."""
    import torch
    p = net.params(flat)
    obs, act = batch[0].double(), batch[1].double()
    n = obs.shape[0]
    edge = torch.zeros(n, dtype=torch.bool, device=obs.device)

    def kinks(pre, x):
        h = x
        for layer in ("1", "2"):
            z = h @ p[pre + "w" + layer] + p[pre + "b" + layer]
            rms = z.pow(2).mean().sqrt() * max(1.0, h.shape[-1] / 256) ** 0.5
            bad = (z.abs() < tol * rms).flatten(1 if z.dim() == 2 else 1).any(-1)
            yield bad
            h = torch.relu(z)
    with torch.no_grad():
        mu, ls = net.actor(obs, p)
        for bad in kinks("a_", obs):
            edge |= bad
        edge |= ((ls + 20).abs() < 1e-5).any(-1) | ((ls - 2).abs() < 1e-5).any(-1)
        a_p, _ = net.sample(mu[:, None], ls[:, None], noise["critic_policy"])
        a_pi, _ = net.sample(mu, ls, noise["actor"])
        rows = [torch.cat([obs, act], -1)[:, None], torch.cat([obs[:, None].expand(n, S, obs.shape[1]), a_p], -1),
                torch.cat([obs[:, None].expand(n, S, obs.shape[1]), noise["critic_uniform"]], -1),
                torch.cat([obs, a_pi], -1)[:, None]]
        x = torch.cat(rows, 1)                                        # [n, 2 + 2 S, K + D]
        for k in (0, 1):
            for bad in kinks("q%d_" % k, x.reshape(-1, x.shape[-1])):
                edge |= bad.view(n, -1).any(-1)
        q0, q1 = net.critic(obs, a_pi, 0, p), net.critic(obs, a_pi, 1, p)
        edge |= (q0 - q1).abs() < 1e-4 * torch.maximum(q0.abs(), q1.abs()).clamp(min=1e-3)
    return edge


@pytest.mark.parametrize("n", [1, 8, 9, 255, 256, 257])
@pytest.mark.parametrize("D", [1, 2, 32, 33, 284])
@pytest.mark.parametrize("K", [266, 3082])
def test_gradient_matches_float64_autograd(K, D, n):
    """r4_cqlc_grad against the twin's float64 autograd on the same draws, tensor by tensor: max |g - ref| <= 1e-3 of
    max(the tensor's largest |ref|, 0.01) (the floor: the last-layer biases' gradient is a sum of the conservative
    term's +-alpha w / n per row, which cancel to far less than the terms).  Rows at a discrete edge (_edge_rows) are replaced by other transitions at the same minibatch
    position before the comparison; the share replaced is reported."""
    import torch
    ds = _dataset(K, D, E=max(8, 3 * n // 9 + 2))
    m = _model(K, D, ds, batch_size=n)
    with torch.no_grad():
        m.net.target.add_(0.01 * torch.randn(m.net.n_target, generator=torch.Generator().manual_seed(3)).cuda())
    data = m._device_data(ds)
    net, S = m.net, int(m.hp["n_action_samples"])
    noise = net.noise(m.seed, 5, n, S, dtype=torch.float64)
    flat64 = net.flat.detach().double()
    cand = torch.randperm(data.n, generator=torch.Generator(device="cuda").manual_seed(1), device="cuda")
    pos, nxt, replaced = cand[:n].clone(), n, 0
    for _ in range(20):
        edge = _edge_rows(net, flat64, data.batch(pos), noise, S)
        k = int(edge.sum())
        if k == 0 or nxt + k > data.n:
            break
        pos[edge] = cand[nxt:nxt + k]
        nxt, replaced = nxt + k, replaced + k
    assert not bool(_edge_rows(net, flat64, data.batch(pos), noise, S).any())
    m.grad_kernels(data, pos, step=5)
    torch.cuda.synchronize()
    ref, st = net.grads(data.batch(pos), noise, m._hyper(), flat64, net.target.double())
    worst = []
    for name, sl in _tensors(net):
        r, g = ref[sl], m.grad[sl].double()
        scale = max(float(r.abs().max()), 1e-2)
        err = float((g - r).abs().max()) / scale
        worst.append((err, name))
        assert err <= 1e-3, (K, D, n, name, err, scale)
    assert torch.allclose(m.stats.double(), st, rtol=1e-4, atol=1e-4), (m.stats, st)
    print("K %d D %d n %d worst %.2e (%s), edge rows replaced %d of %d drawn" % ((K, D, n) + max(worst) + (replaced, nxt)))


def _epoch_call(m, data, perm, mb, step0):
    stats = __import__("torch").zeros(5 * (perm.numel() // mb), device="cuda")
    rc = m.lib.r4_cqlc_epoch(m.net.K, m.D, C.c_void_p(m.net.flat.data_ptr()), C.c_void_p(m.net.target.data_ptr()),
                             C.c_void_p(m.m.data_ptr()), C.c_void_p(m.v.data_ptr()), C.byref(data.c_data()),
                             C.byref(m._hyper_c()), C.c_void_p(perm.data_ptr()), perm.numel(), mb, step0,
                             C.c_void_p(m.scratch.data_ptr()), C.c_void_p(stats.data_ptr()), None)
    assert rc == perm.numel() // mb
    return stats


def test_chained_epoch_matches_twin_steps():
    """20 steps of r4_cqlc_epoch (all four optimisers and the soft target) against 20 twin steps on the same minibatches
    and draws."""
    import torch
    K, D, mb = 266, 32, 64
    ds = _dataset(K, D, E=160)
    m = _model(K, D, ds, batch_size=mb)
    twin = _model(K, D, ds, batch_size=mb)
    twin.use_kernels = False
    data = m._device_data(ds)
    perm = torch.randperm(data.n, generator=torch.Generator(device="cuda").manual_seed(2), device="cuda")[:20 * mb]
    _epoch_call(m, data, perm, mb, 0)
    for k in range(20):
        twin.step = k
        twin.train_step_twin(data.batch(perm[k * mb:(k + 1) * mb]))
    torch.cuda.synchronize()
    assert m.step == 0 and twin.step == 20
    # Adam turns fp32 noise in near-zero gradients into full-size steps, so the drift is judged in norm
    init = _model(K, D, ds, batch_size=mb).net
    moved = float((twin.net.flat.detach() - init.flat.detach()).norm())
    d = float((m.net.flat.detach() - twin.net.flat.detach()).norm())
    assert d <= 0.05 * moved, (d, moved)
    t_moved = float((twin.net.target - init.target).norm())
    assert float((m.net.target - twin.net.target).norm()) <= 0.05 * t_moved


def test_two_runs_bit_identical_and_epoch_equals_its_steps():
    import torch
    K, D, mb = 266, 32, 128
    ds = _dataset(K, D, E=120)
    a, b, c = (_model(K, D, ds, batch_size=mb) for _ in range(3))
    data = a._device_data(ds)
    perm = torch.randperm(data.n, generator=torch.Generator(device="cuda").manual_seed(4), device="cuda")[:5 * mb]
    sa = _epoch_call(a, data, perm, mb, 0)
    sb = _epoch_call(b, data, perm, mb, 0)
    for k in range(5):
        _epoch_call(c, data, perm[k * mb:(k + 1) * mb].contiguous(), mb, k)
    torch.cuda.synchronize()
    for x in (b, c):
        assert torch.equal(a.net.flat, x.net.flat) and torch.equal(a.net.target, x.net.target)
        assert torch.equal(a.m, x.m) and torch.equal(a.v, x.v)
    assert torch.equal(sa, sb)


def test_out_of_range_arguments_write_nothing():
    import torch
    from rl4rs_b200 import _capi
    lib = _capi.load_library()
    assert lib.r4_cqlc_num_params(0, 32) == -1 and lib.r4_cqlc_num_params(4097, 32) == -1
    assert lib.r4_cqlc_num_params(266, 0) == -1 and lib.r4_cqlc_num_params(266, 513) == -1
    assert lib.r4_cqlc_scratch_size(266, 32, 0, 256) == -1 and lib.r4_cqlc_scratch_size(266, 32, 65, 256) == -1
    assert lib.r4_cqlc_scratch_size(266, 32, 10, 0) == -1 and lib.r4_cqlc_scratch_size(266, 32, 10, 4097) == -1
    K, D = 266, 32
    ds = _dataset(K, D, E=10)
    m = _model(K, D, ds, batch_size=16)
    data = m._device_data(ds)
    pos = torch.arange(16, device="cuda")
    before = lib.r4_batchrl_launch_count()
    g0 = m.grad.clone()
    v = C.c_void_p
    for K2, D2, n2, S2 in ((0, D, 16, 10), (4097, D, 16, 10), (K, 0, 16, 10), (K, 513, 16, 10), (K, D, 0, 10),
                           (K, D, 4097, 10), (K, D, 16, 0), (K, D, 16, 65)):
        h = m._hyper_c()
        h.n_action_samples = S2
        rc = lib.r4_cqlc_grad(K2, D2, v(m.net.flat.data_ptr()), v(m.net.target.data_ptr()), C.byref(data.c_data()),
                              C.byref(h), v(pos.data_ptr()), n2, 1, v(m.scratch.data_ptr()), v(m.grad.data_ptr()),
                              v(m.stats.data_ptr()), None)
        assert rc == -1                                   # R4_ERR_ARG
        rc = lib.r4_cqlc_epoch(K2, D2, v(m.net.flat.data_ptr()), v(m.net.target.data_ptr()), v(m.m.data_ptr()),
                               v(m.v.data_ptr()), C.byref(data.c_data()), C.byref(h), v(pos.data_ptr()), 16, max(n2, 0),
                               0, v(m.scratch.data_ptr()), None, None)
        assert rc == -1
    x = torch.zeros(4, K, device="cuda")
    for K2, D2, n2 in ((0, D, 4), (K, 0, 4), (K, D, 0)):
        assert lib.r4_cqlc_act(K2, D2, v(m.net.flat.data_ptr()), v(x.data_ptr()), 0, n2, None, v(m.grad.data_ptr()),
                               None, v(m.scratch.data_ptr()), None) == -1
    torch.cuda.synchronize()
    assert lib.r4_batchrl_launch_count() == before and torch.equal(m.grad, g0)


@pytest.mark.parametrize("D", [32, 284])
def test_predict_kernel_matches_the_twin(D):
    import torch
    K = 266
    ds = _dataset(K, D, E=10)
    m = _model(K, D, ds, batch_size=16)
    x = torch.randn(2048, K, dtype=torch.float64, device="cuda")
    a_in = torch.rand(2048, D, device="cuda") * 2 - 1
    a, q = m.act(x, want_q=True)
    _, q_in = m.act(x, a_in, want_q=True)
    flat = m.net.flat.detach().double()
    ra = m.net.predict(x, flat)
    assert float((a.double() - ra).abs().max()) < 1e-5
    assert torch.allclose(q.double(), m.net.predict_value(x, ra, flat), rtol=1e-4, atol=1e-5)
    assert torch.allclose(q_in.double(), m.net.predict_value(x, a_in.double(), flat), rtol=1e-4, atol=1e-5)


def test_device_draws_match_the_restatement():
    """The kernels' noise (the scratch's noise planes after r4_cqlc_grad) equals policy.cqlc_draws to float32 roundoff."""
    import torch
    from rl4rs_b200.policy import BatchRLContiNet
    K, D, n, S = 266, 33, 9, 10
    ds = _dataset(K, D, E=10)
    m = _model(K, D, ds, batch_size=n)
    data = m._device_data(ds)
    m.grad_kernels(data, torch.arange(n, device="cuda"), step=7)
    torch.cuda.synchronize()
    off = n * (2 * K + D + 2)
    dev = m.scratch[off:off + (2 + 4 * S) * n * D].double().cpu()
    nz = m.net.noise(m.seed, 7, n, S, dtype=torch.float64)
    ref = torch.cat([nz[s].reshape(-1).cpu() for s in BatchRLContiNet.STREAMS])
    assert float((dev - ref).abs().max()) < 1e-5


def test_launches_per_step_match_the_design_count():
    import torch
    K, D, mb = 266, 32, 64
    ds = _dataset(K, D, E=60)
    m = _model(K, D, ds, batch_size=mb)
    data = m._device_data(ds)
    perm = torch.arange(3 * mb, device="cuda")
    c0 = m.lib.r4_batchrl_launch_count()
    _epoch_call(m, data, perm, mb, 0)
    assert m.lib.r4_batchrl_launch_count() - c0 == 3 * LAUNCHES_PER_STEP


@pytest.mark.parametrize("algo", ["CQL-conti", "BCQ-conti"])
@pytest.mark.parametrize("seq,onehot", [(False, False), (True, False), (False, True)])
def test_train_and_eval_end_to_end_on_the_env(seq, onehot, algo, tmp_path):
    import torch
    from test_gpu_parity import _synthetic
    from rl4rs_b200 import batchrl, dataset
    B = 64
    cfg, cat, log, w = _synthetic(B, seq)
    cfg = dict(cfg, catalog=cat, log=log, weights=w, CQL_alpha=1, support_conti_env=True,
               support_onehot_action=onehot, env="SeqSlateRecEnv-v0" if seq else "SlateRecEnv-v0")
    np.random.seed(0)
    gen = dataset.data_generate_rl4rs_b_conti if seq else dataset.data_generate_rl4rs_a_conti
    gen(cfg, str(tmp_path / "ds.npz"), epochs=4)
    ds = batchrl.load_dataset(str(tmp_path / "ds.npz"))
    D = 284 if onehot else cfg["action_emb_size"]
    assert ds["actions"].shape[1] == D
    m = batchrl.get_model(cfg, algo)
    hist = m.fit(ds, n_epochs=1)
    assert m._data.n == 4 * B * cfg["max_steps"] and all(np.isfinite(v) for v in hist[-1][1].values())
    pol = batchrl.policy_model(m, cfg)
    avg = batchrl.evaluate(cfg, pol, batch_size=B, episodes=1)
    assert np.isfinite(avg)
    path = str(tmp_path / "cqlc.pt")
    m.save_model(path)
    m2 = batchrl.get_model(cfg, algo)
    m2.load_model(path)
    x = ds["observations"][:300]
    assert np.array_equal(m.predict(x), m2.predict(x))      # BCQ's draws follow the act counter, saved with the model
    avg = batchrl.evaluate(cfg, pol, batch_size=B, episodes=1)
    avg2 = batchrl.evaluate(cfg, batchrl.policy_model(m2, cfg), batch_size=B, episodes=1)
    print("evaluate %r after load %r, max |a| logged %.3f" % (avg, avg2, float(np.abs(ds["actions"]).max())))
    assert avg2 == avg
    torch.cuda.synchronize()


# ---- BCQ-conti ---------------------------------------------------------------------------------------------
def _bcq_edge_rows(net, flat, batch, noise, hp, tol=1e-5):
    """BCQ's rows at a discrete edge of its gradient: a relu pre-activation (learner_ref64.RELU_TIE's unit) of the
    encoder and decoder on the VAE rows, the critics on the data rows, the actor on its rows and critic 0 on the perturbed
    action; the perturbation within 1e-5 of its clamp; an encoder logstd within 1e-5 of its clamp."""
    import torch
    p = net.params(flat)
    obs, act = batch[0].double(), batch[1].double()
    n, L, flex = obs.shape[0], net.L, hp["action_flexibility"]
    edge = torch.zeros(n, dtype=torch.bool, device=obs.device)

    def kinks(pre, x):
        h = x
        for layer in ("1", "2"):
            z = h @ p[pre + "w" + layer] + p[pre + "b" + layer]
            rms = z.pow(2).mean().sqrt() * max(1.0, h.shape[-1] / 256) ** 0.5
            yield (z.abs() < tol * rms).any(-1)
            h = torch.relu(z)
    cat = lambda a, b: torch.cat([a, b], -1)
    with torch.no_grad():
        e = net._mlp(p, "e_", cat(obs, act))
        mu, lsr = e[:, :L], e[:, L:]
        edge |= ((lsr + 20).abs() < 1e-5).any(-1) | ((lsr - 2).abs() < 1e-5).any(-1)
        z = mu + lsr.clamp(-20, 2).exp() * noise["vae"]
        a_s = net.decode(p, obs, noise["actor"].clamp(-0.5, 0.5))
        f = net._mlp(p, "a_", cat(obs, a_s))
        v = a_s + flex * torch.tanh(f)
        edge |= ((v.abs() - 1).abs() < 1e-5).any(-1)
        a_pi = v.clamp(-1, 1)
        for pre, x in (("e_", cat(obs, act)), ("d_", cat(obs, z)), ("q0_", cat(obs, act)), ("q1_", cat(obs, act)),
                       ("a_", cat(obs, a_s)), ("q0_", cat(obs, a_pi))):
            for bad in kinks(pre, x):
                edge |= bad
    return edge


@pytest.mark.parametrize("n", [1, 8, 9, 255, 256, 257])
@pytest.mark.parametrize("D", [1, 2, 32, 33, 284])
@pytest.mark.parametrize("K", [266, 3082])
def test_bcq_gradient_matches_float64_autograd(K, D, n):
    """r4_bcqc_grad against the twin's float64 autograd on the same draws (100 target samples), tensor by tensor, with the
    bound of test_gradient_matches_float64_autograd; edge rows (_bcq_edge_rows) replaced and reported."""
    import torch
    ds = _dataset(K, D, E=max(8, 3 * n // 9 + 2))
    m = _model(K, D, ds, "BCQ-conti", batch_size=n)
    with torch.no_grad():
        m.net.target.add_(0.01 * torch.randn(m.net.n_target, generator=torch.Generator().manual_seed(3)).cuda())
    data = m._device_data(ds)
    net, S, hp = m.net, int(m.hp["n_action_samples"]), m._hyper()
    noise = net.noise(m.seed, 5, n, S, dtype=torch.float64)
    flat64 = net.flat.detach().double()
    cand = torch.randperm(data.n, generator=torch.Generator(device="cuda").manual_seed(1), device="cuda")
    pos, nxt, replaced = cand[:n].clone(), n, 0
    for _ in range(20):
        edge = _bcq_edge_rows(net, flat64, data.batch(pos), noise, hp)
        k = int(edge.sum())
        if k == 0 or nxt + k > data.n:
            break
        pos[edge] = cand[nxt:nxt + k]
        nxt, replaced = nxt + k, replaced + k
    assert not bool(_bcq_edge_rows(net, flat64, data.batch(pos), noise, hp).any())
    m.grad_kernels(data, pos, step=5)
    torch.cuda.synchronize()
    ref, st = net.grads(data.batch(pos), noise, hp, flat64, net.target.double())
    worst = []
    for name, sl in _tensors(net):
        r, g = ref[sl], m.grad[sl].double()
        scale = max(float(r.abs().max()), 1e-2)
        err = float((g - r).abs().max()) / scale
        worst.append((err, name))
        assert err <= 1e-3, (K, D, n, name, err, scale)
    assert torch.allclose(m.stats.double(), st, rtol=1e-4, atol=1e-4), (m.stats, st)
    print("BCQ K %d D %d n %d worst %.2e (%s), edge rows replaced %d of %d drawn"
          % ((K, D, n) + max(worst) + (replaced, nxt)))


def _bcq_epoch(m, data, perm, mb, step0):
    import torch
    stats = torch.zeros(5 * (perm.numel() // mb), device="cuda")
    rc = m.lib.r4_bcqc_epoch(m.net.K, m.D, C.c_void_p(m.net.flat.data_ptr()), C.c_void_p(m.net.target.data_ptr()),
                             C.c_void_p(m.m.data_ptr()), C.c_void_p(m.v.data_ptr()), C.byref(data.c_data()),
                             C.byref(m._hyper_c()), C.c_void_p(perm.data_ptr()), perm.numel(), mb, step0,
                             C.c_void_p(m.scratch.data_ptr()), C.c_void_p(stats.data_ptr()), None)
    assert rc == perm.numel() // mb
    return stats


def test_bcq_chained_epoch_matches_twin_and_is_deterministic():
    """20 steps of r4_bcqc_epoch against 20 twin steps (all three optimisers and the soft targets; drift judged in norm);
    a second run is bit-identical and one call per minibatch equals the chained call; 69 launches per step."""
    import torch
    K, D, mb = 266, 32, 64
    ds = _dataset(K, D, E=160)
    m, b, c = (_model(K, D, ds, "BCQ-conti", batch_size=mb) for _ in range(3))
    twin = _model(K, D, ds, "BCQ-conti", batch_size=mb)
    twin.use_kernels = False
    data = m._device_data(ds)
    perm = torch.randperm(data.n, generator=torch.Generator(device="cuda").manual_seed(2), device="cuda")[:20 * mb]
    c0 = m.lib.r4_batchrl_launch_count()
    sa = _bcq_epoch(m, data, perm, mb, 0)
    assert m.lib.r4_batchrl_launch_count() - c0 == 20 * BCQ_LAUNCHES_PER_STEP
    sb = _bcq_epoch(b, data, perm, mb, 0)
    for k in range(20):
        _bcq_epoch(c, data, perm[k * mb:(k + 1) * mb].contiguous(), mb, k)
        twin.step = k
        twin.train_step_twin(data.batch(perm[k * mb:(k + 1) * mb]))
    torch.cuda.synchronize()
    assert torch.equal(sa, sb)
    for x in (b, c):
        assert torch.equal(m.net.flat, x.net.flat) and torch.equal(m.net.target, x.net.target) and torch.equal(m.v, x.v)
    init = _model(K, D, ds, "BCQ-conti", batch_size=mb).net
    moved = float((twin.net.flat.detach() - init.flat.detach()).norm())
    assert float((m.net.flat.detach() - twin.net.flat.detach()).norm()) <= 0.05 * moved
    t_moved = float((twin.net.target - init.target).norm())
    assert float((m.net.target - twin.net.target).norm()) <= 0.05 * t_moved


@pytest.mark.parametrize("D", [32, 284])
def test_bcq_predict_kernel_matches_the_twin(D):
    """Batch 2048 x 100 candidates on the same latent draws: the kernel's action is the twin's best candidate except at
    recorded near-ties of Q_0 (top-two gap <= 1e-4 of the row's largest |Q_0|), and predict_value matches."""
    import torch
    K = 266
    ds = _dataset(K, D, E=10)
    m = _model(K, D, ds, "BCQ-conti", batch_size=16)
    x = torch.randn(2048, K, dtype=torch.float64, device="cuda")
    a, _ = m.act(x)
    net, hp, S = m.net, m._hyper(), int(m.hp["n_action_samples"])
    flat = net.flat.detach().double()
    p = net.params(flat)
    z = net.predict_noise(m.seed, m.act_counter, 2048, S, torch.float64)
    cand = net.candidates(p, x, z, hp["action_flexibility"])
    q = net.critic(x[:, None].expand(2048, S, K), cand, 0, p)
    best = cand[torch.arange(2048, device="cuda"), q.argmax(1)]
    top = q.topk(2, 1).values
    tie = (top[:, 0] - top[:, 1]) <= 1e-4 * q.abs().max(1).values.clamp(min=1e-3)
    match = (a.double() - best).abs().max(1).values < 1e-4
    assert bool((match | tie).all()), int((~match & ~tie).sum())
    print("BCQ predict D %d: %d of 2048 rows differ, all at near-ties (%d near-ties)" % (D, int((~match).sum()), int(tie.sum())))
    a_in = torch.rand(2048, D, device="cuda") * 2 - 1
    _, qv = m.act(x, a_in, want_q=True)
    assert torch.allclose(qv.double(), net.predict_value(x, a_in.double(), flat), rtol=1e-4, atol=1e-5)


def test_bcq_out_of_range_arguments_write_nothing():
    import torch
    from rl4rs_b200 import _capi
    lib = _capi.load_library()
    assert lib.r4_bcqc_num_params(0, 32, 32) == -1 and lib.r4_bcqc_num_params(266, 513, 32) == -1
    assert lib.r4_bcqc_num_params(266, 32, 0) == -1 and lib.r4_bcqc_num_params(266, 32, 513) == -1
    assert lib.r4_bcqc_scratch_size(266, 32, 32, 257, 256) == -1 and lib.r4_bcqc_scratch_size(266, 32, 32, 100, 4097) == -1
    assert lib.r4_bcqc_act_scratch_size(266, 32, 32, 100, 20000) == -1
    assert lib.r4_cqlc_act_scratch_size(266, 32, (1 << 20) + 1) == -1
    K, D = 266, 32
    ds = _dataset(K, D, E=10)
    m = _model(K, D, ds, "BCQ-conti", batch_size=16)
    data = m._device_data(ds)
    pos = torch.arange(16, device="cuda")
    before, g0 = lib.r4_batchrl_launch_count(), m.grad.clone()
    v = C.c_void_p
    for K2, D2, n2, S2, L2 in ((0, D, 16, 100, 32), (K, 0, 16, 100, 32), (K, D, 0, 100, 32), (K, D, 4097, 100, 32),
                               (K, D, 16, 0, 32), (K, D, 16, 257, 32), (K, D, 16, 100, 0)):
        h = m._hyper_c()
        h.n_action_samples, h.latent_size = S2, L2
        assert lib.r4_bcqc_grad(K2, D2, v(m.net.flat.data_ptr()), v(m.net.target.data_ptr()), C.byref(data.c_data()),
                                C.byref(h), v(pos.data_ptr()), n2, 1, v(m.scratch.data_ptr()), v(m.grad.data_ptr()),
                                v(m.stats.data_ptr()), None) == -1
        assert lib.r4_bcqc_epoch(K2, D2, v(m.net.flat.data_ptr()), v(m.net.target.data_ptr()), v(m.m.data_ptr()),
                                 v(m.v.data_ptr()), C.byref(data.c_data()), C.byref(h), v(pos.data_ptr()), 16, n2,
                                 0, v(m.scratch.data_ptr()), None, None) == -1
        if n2 <= 16:                # (n 4097 is a valid predict size)
            assert lib.r4_bcqc_act(K2, D2, v(m.net.flat.data_ptr()), v(data.obs.data_ptr()), 0, n2, C.byref(h), 1, None,
                                   v(m.grad.data_ptr()), None, v(m.scratch.data_ptr()), None) == -1
    torch.cuda.synchronize()
    assert lib.r4_batchrl_launch_count() == before and torch.equal(m.grad, g0)
