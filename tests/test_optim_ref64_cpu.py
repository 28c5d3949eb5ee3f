"""CPU: the float64 optimiser rules of tests/optim_ref64.py against torch.optim.Adam and clip_grad_norm_ in float64, their
bounds against an fp32 evaluation of the same rule, and the DDPG, batch-RL and continuous batch-RL layouts against the
twins' own slices and the C-ABI's r4_*_num_params / r4_*_target_size."""
import math

import numpy as np
import pytest
import torch

import optim_ref64 as O


def _lib():
    from rl4rs_b200 import _capi
    return _capi.load_library()


@pytest.mark.parametrize("step", [1, 2, 10, 10000])
def test_adam_matches_torch_optim_adam_in_float64(step):
    n = 4000
    g, m, v = O.carried(n, step)
    p = np.random.RandomState(7).randn(n).astype(np.float32)
    lr = 1e-3
    st = O.adam(p, g, m, v, step, lr)
    t = torch.tensor(p, dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([t], lr=O.f32(lr), betas=(O.B1, O.B2), eps=O.EPS)
    opt.state[t] = {"step": torch.tensor(float(step - 1), dtype=torch.float64),
                    "exp_avg": torch.tensor(m, dtype=torch.float64), "exp_avg_sq": torch.tensor(v, dtype=torch.float64)}
    t.grad = torch.tensor(g, dtype=torch.float64)
    opt.step()
    s = opt.state[t]
    np.testing.assert_allclose(st.m, s["exp_avg"].numpy(), rtol=1e-14, atol=0)
    np.testing.assert_allclose(st.v, s["exp_avg_sq"].numpy(), rtol=1e-14, atol=0)
    # the update itself within float64 reordering (torch divides by bc1 in another place)
    np.testing.assert_allclose(st.p - p, t.detach().numpy() - p, rtol=1e-12, atol=1e-30)


def _adam_f32(p, g, m, v, step, lr, eps=1e-8):
    """adam_update's operation order in float32 (what a correct kernel computes, up to the contractions it may make)."""
    f = np.float32
    b1, b2 = f(0.9), f(0.999)
    mi = b1 * m + (f(1) - b1) * g
    vi = b2 * v + (f(1) - b2) * g * g
    bc1, bc2 = f(1) - b1 ** f(step), f(1) - b2 ** f(step)
    den = np.sqrt(vi) / np.sqrt(bc2) + f(eps)
    return p - (f(lr) / bc1) * (mi / den), mi, vi


@pytest.mark.parametrize("step", [1, 2, 10, 10000])
def test_bounds_hold_an_fp32_adam_and_catch_the_wrong_rules(step):
    """An fp32 evaluation of the rule stays within the bounds; a step count off by one, TF1's eps, a dropped clip factor
    and a doubled one each land at >= 100x on some element."""
    n = 20000
    g, m, v = O.carried(n, 100 + step)
    p = np.random.RandomState(3).randn(n).astype(np.float32)
    st = O.adam(p, g, m, v, step, 1e-3)
    p32, m32, v32 = _adam_f32(p, g, m, v, step, 1e-3)
    for got, ref, b in ((p32, st.p, st.bp), (m32, st.m, st.bm), (v32, st.v, st.bv)):
        assert float((np.abs(got.astype(np.float64) - ref) / b).max()) <= 0.5
    wrong = []
    if step > 1:
        wrong.append(O.adam(p, g, m, v, step - 1, 1e-3).p)
    wrong.append(O.adam(p, g, m, v, step + 1, 1e-3).p)
    # TF1: lr_t = lr sqrt(1 - b2^t) / (1 - b1^t), p -= lr_t m / (sqrt(v) + eps), i.e. eps added before the bias correction
    bc1, bc2 = 1 - O.B1 ** step, 1 - O.B2 ** step
    wrong.append(p - O.f32(1e-3) * math.sqrt(bc2) / bc1 * st.m / (np.sqrt(st.v) + O.EPS))
    if step <= 10:
        assert all(float((np.abs(w - st.p) / st.bp).max()) > 100 for w in wrong), step
    # a clip factor of 0.5 dropped or applied twice moves m far beyond its bound
    g2, c, on = O.global_clip(g, 1.0, 0.5 * math.sqrt(float((g.astype(np.float64) ** 2).sum())))
    assert on and abs(c - 0.5) < 1e-6
    ref = O.adam(p, g2, m, v, step, 1e-3, rel_g=2 * O.U + O.sumsq_rel(n, 1024))
    for k in (1.0 / c, c):
        bad = O.adam(p, g2 * k, m, v, step, 1e-3)
        assert float((np.abs(bad.m - ref.m) / ref.bm).max()) > 100


@pytest.mark.parametrize("grad_scale", [1.0, 0.5])
@pytest.mark.parametrize("ratio", [0.0, 0.3, 3.0])
def test_global_clip_is_torch_clip_grad_norm_after_the_scale(grad_scale, ratio):
    g = np.random.RandomState(1).randn(1000).astype(np.float32)
    norm = float(np.sqrt((g.astype(np.float64) ** 2).sum())) * grad_scale
    clip = ratio * norm
    got, c, on = O.global_clip(g, grad_scale, clip)
    t = torch.tensor(g, dtype=torch.float64) * grad_scale
    t.grad = t.clone()
    if clip > 0:
        torch.nn.utils.clip_grad_norm_([t], O.f32(clip))
    np.testing.assert_allclose(got, t.grad.numpy(), rtol=1e-12)
    assert on == (0 < ratio < 1)


def test_clip_per_tensor_matches_the_rainbow_twin():
    from rl4rs_b200.policy import DistributionalQNetwork
    net = DistributionalQNetwork(6, torch.device("cpu"), seed=1, num_atoms=4)
    g = torch.randn(net.n_params, generator=torch.Generator().manual_seed(2)) * 0.3
    norms = sorted(float(g[lo:hi].norm()) for lo, hi in net.slices)
    clip = math.sqrt(norms[5] * norms[6])
    ref = g.clone()
    net.clip_per_tensor(ref, clip)
    got, which = O.clip_per_tensor(g.numpy(), net.slices, clip)
    np.testing.assert_allclose(got, ref.double().numpy(), rtol=1e-6, atol=0)      # the twin clips in float32
    assert 0 < sum(on for _, _, on in which) < len(which)


@pytest.mark.parametrize("D,twin", [(2, 0), (2, 1), (32, 0), (32, 1), (17, 1)])
def test_ddpg_layout_matches_the_twin_and_the_c_abi(D, twin):
    from rl4rs_b200.policy import DeterministicActorCritic
    net = DeterministicActorCritic(D, torch.device("cpu"), seed=0, twin=bool(twin))
    n, na, kern = O.ddpg_layout(D, twin)
    assert n == net.n_params == _lib().r4_ddpg_num_params(D, twin)
    assert na == net.n_actor
    assert np.array_equal(kern, net.kernel_mask.numpy())
    names = [t for _, ts in O.ddpg_nets(D, twin)[0] for t, _, _, _ in ts]
    assert names == [name for name, _ in net._shapes]


def test_ddpg_apply_rule():
    """l2 on the kernels only, each optimiser at its own lr and step, the actor frozen at actor_step 0 while its target still
    moves, and tau p + (1 - tau) t."""
    D, twin = 2, 1
    n, na, kern = O.ddpg_layout(D, twin)
    rs = np.random.RandomState(0)
    p, t, g = (rs.randn(n).astype(np.float32) * s for s in (0.1, 0.1, 1e-3))
    m, v = np.zeros(n, np.float32), np.zeros(n, np.float32)
    st, a_end = O.ddpg_apply(p, t, g, m, v, D, twin, 0, 3, 1e-3, 3e-4, 1e-2, 0.005, 0.5)
    assert a_end == na
    assert np.array_equal(st.p[:na], p[:na]) and np.array_equal(st.m[:na], m[:na])
    geff = 0.5 * g.astype(np.float64) + np.where(kern, O.f32(1e-2) * p.astype(np.float64), 0.0)
    np.testing.assert_allclose(st.m[na:], (1 - O.B1) * geff[na:], rtol=1e-15)
    ref = O.adam(p[na:], geff[na:], m[na:], v[na:], 3, 3e-4)
    np.testing.assert_allclose(st.p[na:], ref.p, rtol=1e-15)
    tgt, _ = O.soft_target(st.p, t, 0.005)
    np.testing.assert_allclose(tgt, O.f32(0.005) * st.p + O.f32(1 - O.f32(0.005)) * t.astype(np.float64), rtol=1e-15)


def _algos():
    from rl4rs_b200.batchrl import ALGOS
    return ALGOS


@pytest.mark.parametrize("algo", ["BC", "BCQ", "CQL"])
@pytest.mark.parametrize("K,A", [(11, 2), (266, 284), (3082, 284), (4096, 284), (2998, 512), (266, 512)])
def test_batchrl_layout_matches_the_twin_and_the_c_abi(algo, K, A):
    from rl4rs_b200.policy import BatchRLNet
    lib = _lib()
    k = _algos()[algo]
    n, ntgt = O.bq_layout(algo, K, A)
    assert lib.r4_batchrl_num_params(k, K, A) == n
    assert lib.r4_batchrl_target_size(k, K, A) == ntgt
    if K <= 266:        # the twin allocates its parameters: the small shapes suffice for the slices
        net = BatchRLNet(algo, K, np.ones((4, A), np.float32), [0], A, torch.device("cpu"), seed=0)
        assert net.n_params == n and net.n_target == ntgt
    assert lib.r4_batchrl_target_size(k, K + (4097 - K), A) == -1


@pytest.mark.parametrize("K,D", [(1, 1), (266, 32), (3082, 284), (4096, 512)])
def test_cqlc_groups_match_the_twin_and_the_c_abi(K, D):
    from rl4rs_b200.policy import BatchRLContiNet
    lib = _lib()
    n, ntgt, t0 = O.cqlc_sizes(K, D)
    assert lib.r4_cqlc_num_params(K, D) == n and lib.r4_cqlc_target_size(K, D) == ntgt
    groups = O.cqlc_groups(K, D)
    assert [g[0] for g in groups] == ["temp", "alpha", "critic", "actor"]
    cover = sorted(g[1] for g in groups)
    assert cover[0][0] == 0 and cover[-1][1] == n and all(a[1] == b[0] for a, b in zip(cover, cover[1:]))
    if K * D <= 266 * 32:
        net = BatchRLContiNet(K, D, torch.device("cpu"), 0, 1.0, 1.0)
        assert net.n_params == n and net.n_target == ntgt and net.t0 == t0
        for name, (lo, hi), _, tr in groups:
            assert net.group(name) == slice(lo, hi), name
            if tr is not None:      # the soft update writes target[k] from params[t0 + k]
                assert (tr[0] + t0, tr[1] + t0) == (lo, hi)


@pytest.mark.parametrize("K,D,Lat", [(1, 1, 1), (266, 32, 64), (3082, 284, 512), (4096, 512, 512)])
def test_bcqc_groups_match_the_twin_and_the_c_abi(K, D, Lat):
    from rl4rs_b200.policy import BatchRLContiBCQNet
    lib = _lib()
    n, ntgt = O.bcqc_sizes(K, D, Lat)
    assert lib.r4_bcqc_num_params(K, D, Lat) == n and lib.r4_bcqc_target_size(K, D, Lat) == ntgt
    groups = O.bcqc_groups(K, D, Lat)
    assert [g[0] for g in groups] == ["imitator", "critic", "actor"]
    # the target ranges the two soft updates write tile [0, ntgt) and follow params at the same index
    tr = sorted(g[3] for g in groups if g[3] is not None)
    assert tr[0][0] == 0 and tr[-1][1] == ntgt and tr[0][1] == tr[1][0]
    assert all(g[3] is None or g[3] == g[1] for g in groups)
    if K * D <= 266 * 32:
        net = BatchRLContiBCQNet(K, D, torch.device("cpu"), 0, Lat)
        assert net.n_params == n and net.n_target == ntgt
        for name, (lo, hi), _, _ in groups:
            assert net.group(name) == slice(lo, hi), name
