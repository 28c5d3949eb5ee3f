"""GPU: the batch-RL kernels (csrc/r4_batchrl.cuh) against the torch twin (policy.BatchRLNet) and autograd -- the gradient,
chained epochs with target copies, determinism, the act rule -- and the train / eval stages end to end on the CUDA env."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

A = 284


def _dataset(K, E=80, L=10, seed=0):
    from test_batchrl_cpu import synthetic_dataset
    return synthetic_dataset(K, E, L, seed)


def _model(algo, K, ds, **hp):
    import torch
    from rl4rs_b200 import batchrl, synth
    cfg = {"action_size": A, "page_items": 9, "catalog": synth.make_catalog(), "CQL_alpha": 1}
    m = batchrl.get_model(cfg, algo)
    m.hp.update(hp)
    m.batch_size = int(m.hp["batch_size"])
    m.build_with_dataset(ds)
    assert m.use_kernels and m.net.K == K
    if m.net.n_target:
        with torch.no_grad():
            g = torch.Generator().manual_seed(3)
            m.net.target.add_(0.05 * torch.randn(m.net.n_target, generator=g).cuda())
    return m


def _tensors(net):
    """(name, slice) of every tensor of the flat layout."""
    import math
    off, out = 0, []
    for name, shape in net._shapes:
        k = math.prod(shape)
        out.append((name, slice(off, off + k)))
        off += k
    return out


@pytest.mark.parametrize("K", [266, 3082])
@pytest.mark.parametrize("algo", ["BC", "BCQ", "CQL"])
def test_gradient_matches_autograd(algo, K):
    import torch
    ds = _dataset(K)
    m = _model(algo, K, ds, batch_size=256)
    data = m._device_data(ds)
    pos = torch.randperm(data.n, generator=torch.Generator(device="cuda").manual_seed(1), device="cuda")[:256]
    m.grad_kernels(data, pos)
    torch.cuda.synchronize()
    net = m.net
    if net.flat.grad is not None:
        net.flat.grad.zero_()
    loss, st = net.loss(*data.batch(pos), m._hyper())
    loss.backward()
    ref = net.flat.grad.detach()
    for name, sl in _tensors(net):
        r, g = ref[sl], m.grad[sl]
        scale = float(r.abs().max())
        assert float((g - r).abs().max()) <= 1e-4 * max(scale, 1e-6), (algo, K, name, float((g - r).abs().max()), scale)
    assert torch.allclose(m.stats, st.float(), rtol=1e-4, atol=1e-5), (m.stats, st)


@pytest.mark.parametrize("algo", ["BC", "BCQ", "CQL"])
def test_chained_epoch_matches_twin_steps(algo):
    """20 steps of r4_batchrl_epoch (target copies at steps 1, 6, 11, 16) against 20 twin steps on the same minibatches."""
    import torch
    ds = _dataset(266, E=60, L=10)
    mk = _model(algo, 266, ds, batch_size=25, target_update_interval=5, learning_rate=1e-4)
    mt = _model(algo, 266, ds, batch_size=25, target_update_interval=5, learning_rate=1e-4)
    mt.use_kernels = False
    data = mk._device_data(ds)
    assert data.n == 60 * 9
    perm = torch.randperm(data.n, generator=torch.Generator(device="cuda").manual_seed(2), device="cuda")[:500]
    with torch.no_grad():
        mt.net.flat.copy_(mk.net.flat)
        mt.net.target.copy_(mk.net.target)
    pre = mk.net.target.clone()
    mk._epoch_kernels(data, perm)
    for k in range(20):
        mt.train_step_twin(data.batch(perm[k * 25:(k + 1) * 25]))
    torch.cuda.synchronize()
    assert mk.step == mt.step == 20
    # Adam turns fp32 noise in near-zero gradients into full-size steps, so the drift is judged in norm
    init = _model(algo, 266, ds).net.flat.detach()
    moved = float((mt.net.flat.detach() - init).norm())
    d = float((mk.net.flat.detach() - mt.net.flat.detach()).norm())
    assert d <= 0.05 * moved, (d, moved)
    if mk.net.n_target:             # the last copy (step 16) holds the parameters of step 16 in both
        td = float((mk.net.target - mt.net.target).norm())
        q = mk.net.flat.detach()[:mk.net.n_target]
        assert td <= 0.05 * moved and float((mk.net.target - q).norm()) < float((pre - q).norm())


def test_two_runs_are_bit_identical():
    import torch
    ds = _dataset(266)
    outs = []
    for _ in range(2):
        m = _model("BCQ", 266, ds, batch_size=64, target_update_interval=3)
        m.fit(ds, 1)
        torch.cuda.synchronize()
        outs.append((m.net.flat.detach().clone(), m.net.target.clone(), m.m.clone(), m.v.clone()))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("algo", ["BC", "BCQ", "CQL"])
def test_act_kernel_matches_the_twin(algo):
    import torch
    ds = _dataset(266)
    m = _model(algo, 266, ds)
    obs = torch.as_tensor(ds["observations"][:400], device="cuda")
    for mode in (0, 1):
        for x in (obs, obs.double()):
            a, probs, vals = m.act(x, mode, want_probs=True, want_values=True)
            at, pt, vt = m.net.act(obs, mode, m._hyper()["log_flex"])
            assert float((vals - vt).abs().max()) <= 1e-4 * float(vt.abs().max())
            assert float((probs - pt).abs().max()) <= 1e-4 * max(1.0, float(pt.abs().max()))
            pick = torch.where(m.net.keep(obs), pt, torch.full_like(pt, -2.0 ** 15)) if mode == 0 else \
                (m.net.bcq_filtered(obs, m._hyper()["log_flex"]) if algo == "BCQ" else pt)
            top2 = pick.topk(2, 1).values
            clear = (top2[:, 0] - top2[:, 1]) > 1e-4 * max(1e-3, float(top2[:, 0].abs().max().detach()))
            assert int(clear.sum()) > 300
            assert torch.equal(a.long()[clear], at.long()[clear]), (algo, mode)
            # the rule never picks an excluded item in mode 0
            if mode == 0:
                assert bool(m.net.keep(obs)[torch.arange(400, device="cuda"), a.long()].all())


@pytest.mark.parametrize("seq", [False, True])
def test_train_and_eval_end_to_end_on_the_env(seq, tmp_path):
    import torch
    from test_gpu_parity import _synthetic
    from rl4rs_b200 import batchrl, dataset
    B = 64
    cfg, cat, log, w = _synthetic(B, seq)
    cfg = dict(cfg, catalog=cat, log=log, weights=w, CQL_alpha=1, env="SeqSlateRecEnv-v0" if seq else "SlateRecEnv-v0")
    np.random.seed(0)
    gen = dataset.data_generate_rl4rs_b if seq else dataset.data_generate_rl4rs_a
    ds = gen(cfg, str(tmp_path / "ds.npz"), epochs=4)
    ds = batchrl.load_dataset(str(tmp_path / "ds.npz"))
    T = cfg["max_steps"]
    for algo in ("BC", "BCQ", "CQL"):
        m = batchrl.get_model(cfg, algo)
        hist = m.fit(ds, n_epochs=1 if algo != "BC" else 30)
        assert m._data.n == 4 * B * T and all(np.isfinite(v) for v in hist[-1][1].values())
        pol = batchrl.policy_model(m, cfg)
        avg = batchrl.evaluate(cfg, pol, batch_size=B, episodes=1)
        assert np.isfinite(avg)
        path = str(tmp_path / ("%s.pt" % algo))
        m.save_model(path)
        m2 = batchrl.get_model(cfg, algo)
        m2.load_model(path)
        x = ds["observations"][:300]
        assert np.array_equal(m.predict(x), m2.predict(x))
        assert np.array_equal(pol.predict_with_mask(x), batchrl.policy_model(m2, cfg).predict_with_mask(x))
        if algo == "BC":
            data = m._data
            e = data.transitions
            got = m.act(data.obs[e], 0)[0].long()
            match = float((got == data.action[e].long()).float().mean())
            keep = m.net.keep(data.obs[e])
            chance = float((1.0 / keep.sum(1).clamp(min=1).double()).mean())
            assert match > chance, (match, chance)
    torch.cuda.synchronize()
