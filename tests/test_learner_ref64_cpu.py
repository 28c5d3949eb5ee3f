"""CPU: the float64 learner reference (tests/learner_ref64.py) against the fp32 twins' autograd and the NumPy float64
restatements of test_trainer_rainbow_cpu.py and test_batchrl_cpu.py, across the GPU grid's shapes; and the C-ABI's size
functions at the last accepted and the first rejected shape of every learner (host calls: they need the library, not a
device).

The twin bound is per tensor, 1e-3 of the tensor's max |ref| on rows clear of every decision: a single bias gradient off
by 1 % fails it."""
import math

import numpy as np
import pytest
import torch

import learner_ref64 as R

TWIN_TOL = 1e-3


def _per_tensor(what, got, ref, twin, tol=TWIN_TOL):
    bad = []
    for name, sl in R.tensors(twin):
        r = ref[sl]
        err = float((got[sl].double() - r).abs().max())
        if err > tol * max(float(r.abs().max()), 1e-30):
            bad.append((name, err / (tol * float(r.abs().max()))))
    assert not bad, (what, bad)


def _clear(ref, n):
    keep = torch.nonzero(ref.clear()).reshape(-1)
    assert keep.numel() >= 0.92 * len(ref.clear()), "the tie filter dropped too many rows"
    return keep[:n]


# ---- mask policy and Gaussian policy ---------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("A", [2, 31, 284, 512])
def test_policy_reference_matches_the_twin(A, mode):
    from rl4rs_b200.policy import MaskedPolicy
    from rl4rs_b200.trainer import A2CTrainer, PPOTrainer
    pol = MaskedPolicy(A, "cpu", seed=3)
    with torch.no_grad():
        pol.flat.add_(0.05 * torch.randn(pol.n_params, generator=torch.Generator().manual_seed(4)))
    pool = R.mask_batch(pol, 80, A, torch.device("cpu"), seed=A)
    hp = R.PG_HP[mode]
    sel = _clear(R.policy_grad(pol, pol.flat, mode, *pool, hp, 1.0), 64)
    data = tuple(x[sel] for x in pool)
    n = len(sel)
    ref = R.policy_grad(pol, pol.flat, mode, *data, hp, 1.0 / n if mode == 0 else 1.0)
    cfg = {"clip_param": hp["clip"], "vf_clip_param": hp["vf_clip"], "vf_loss_coeff": hp["vf_coeff"],
           "entropy_coeff": hp["ent_coeff"]}
    tr = type("T", (), {"config": cfg, "kl_coeff": hp["kl_coeff"], "policy": pol})()
    pol.flat.grad = None
    if mode == 0:
        total, st = PPOTrainer.loss(tr, *data)
    else:
        total, st = A2CTrainer.loss(tr, data[0], data[1], data[2], data[6], data[7])
    total.backward()
    _per_tensor("policy A%d" % A, pol.flat.grad, ref.grad, pol)
    assert abs(float(total.detach()) - float(ref.loss)) <= 1e-5 * max(1.0, abs(float(ref.loss)))


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("D", [2, 32, 64])
def test_gauss_reference_matches_the_twin(D, mode):
    from rl4rs_b200.policy import GaussianPolicy
    from rl4rs_b200.trainer import A2CTrainer, PPOTrainer
    pol = GaussianPolicy(D, "cpu", seed=3)
    with torch.no_grad():
        pol.flat.add_(0.02 * torch.randn(pol.n_params, generator=torch.Generator().manual_seed(3)))
    pool = R.gauss_batch(pol, 80, D, torch.device("cpu"), seed=D)
    hp = R.PG_HP[mode]
    sel = _clear(R.gauss_grad(pol, pol.flat, mode, *pool, hp, 1.0), 64)
    data = tuple(x[sel] for x in pool)
    n = len(sel)
    ref = R.gauss_grad(pol, pol.flat, mode, *data, hp, 1.0 / n if mode == 0 else 1.0)
    cfg = {"clip_param": hp["clip"], "vf_clip_param": hp["vf_clip"], "vf_loss_coeff": hp["vf_coeff"],
           "entropy_coeff": hp["ent_coeff"]}
    tr = type("T", (), {"config": cfg, "kl_coeff": hp["kl_coeff"], "policy": pol})()
    pol.flat.grad = None
    if mode == 0:
        total, _ = PPOTrainer.loss(tr, *data)
    else:
        total, _ = A2CTrainer.loss(tr, data[0], data[1], data[5], data[6])
    total.backward()
    _per_tensor("gauss D%d" % D, pol.flat.grad, ref.grad, pol)


# ---- DDPG / TD3 ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("twin", [False, True])
@pytest.mark.parametrize("D", [2, 7, 32])
def test_ddpg_reference_matches_the_twin(D, twin):
    from rl4rs_b200.policy import DeterministicActorCritic
    pol = DeterministicActorCritic(D, "cpu", seed=5, twin=twin)
    g = torch.Generator().manual_seed(D)
    with torch.no_grad():
        pol.flat.add_(0.01 * torch.randn(pol.n_params, generator=g))
        pol.target.copy_(pol.flat.detach() + 0.01 * torch.randn(pol.n_params, generator=g))
    P = 80
    obs, nobs = torch.randn(P, 256, generator=g), torch.randn(P, 256, generator=g)
    act = torch.rand(P, D, generator=g) * 2 - 1
    rew = torch.randn(P, generator=g)
    done = (torch.rand(P, generator=g) < 0.3).to(torch.uint8)
    w = None if twin else torch.rand(P, generator=g) + 0.5
    noise = torch.randn(P, D, generator=g) if twin else None
    sel = _clear(R.ddpg_grad(pol, pol.flat, pol.target, obs, act, rew, nobs, done, w, noise, 0.99, 0.2, 0.5, 1.0), 64)
    pick = lambda x: None if x is None else x[sel]
    b = tuple(map(pick, (obs, act, rew, nobs, done, w, noise)))
    n = len(sel)
    ref = R.ddpg_grad(pol, pol.flat, pol.target, *b, 0.99, 0.2, 0.5, 1.0 / n)
    pol.flat.grad = None
    cl, al, td = pol.losses(*b[:5], b[5], b[6], 0.99, 0.2, 0.5, 1.0 / n)
    (cl + al).backward()
    _per_tensor("ddpg D%d" % D, pol.flat.grad, ref.grad, pol)
    assert float((td.double() - ref.rows).abs().max()) <= 1e-4 * max(1.0, float(ref.rows.abs().max()))
    cl, al = cl.detach(), al.detach()
    assert abs(float(cl) - float(ref.stats[0])) <= 1e-5 * max(1.0, abs(float(ref.stats[0])))
    assert abs(float(al) - float(ref.stats[1])) <= 1e-5 * max(1.0, abs(float(ref.stats[1])))


# ---- RAINBOW ------------------------------------------------------------------------------------------------------
def _rainbow_case(A, Z, v_min, v_max, P=80, seed=0):
    from rl4rs_b200.policy import DistributionalQNetwork
    pol = DistributionalQNetwork(A, "cpu", seed=2, num_atoms=Z, v_min=v_min, v_max=v_max)
    g = torch.Generator().manual_seed(A * Z + seed)
    with torch.no_grad():
        pol.target.add_(0.3 * torch.randn(pol.n_params, generator=g))
    obs, nobs = torch.randn(P, 256, generator=g), torch.randn(P, 256, generator=g)
    act = torch.randint(0, A, (P,), generator=g, dtype=torch.int32)
    rew = R.rb_rewards(P, Z, v_min, v_max, g)
    done = (torch.arange(P) % 3 == 0).to(torch.uint8)
    w = torch.rand(P, generator=g) + 0.5
    return pol, (obs, act, rew, nobs, done, w)


@pytest.mark.parametrize("vrange", [(0.0, 1000.0), (-10.0, 10.0)])
@pytest.mark.parametrize("AZ", [(2, 2), (284, 8), (512, 8), (128, 32), (2, 32)])
def test_rainbow_reference_matches_the_twin(AZ, vrange):
    A, Z = AZ
    pol, pool = _rainbow_case(A, Z, *vrange)
    gamma_n = 1.0 if vrange[0] == 0.0 else 0.729
    sel = _clear(R.rainbow_grad(pol, pol.flat, pol.target, *pool, gamma_n, 1.0), 64)
    b = tuple(x[sel] for x in pool)
    n = len(sel)
    ref = R.rainbow_grad(pol, pol.flat, pol.target, *b, gamma_n, 1.0 / n)
    pol.flat.grad = None
    loss, td = pol.loss(*b[:5], b[5], gamma_n, 1.0 / n)
    loss.backward()
    _per_tensor("rainbow A%d Z%d" % (A, Z), pol.flat.grad, ref.grad, pol)
    assert float((td.double() - ref.rows).abs().max()) <= 1e-4 * max(1.0, float(ref.rows.abs().max()))


def test_rainbow_reference_matches_numpy():
    """At the trainer's shape (284 actions, 8 atoms): td and loss against test_trainer_rainbow_cpu's NumPy restatement."""
    from test_trainer_rainbow_cpu import _np_forward, _np_params, _np_project
    pol, pool = _rainbow_case(284, 8, 0.0, 10.0, P=24)
    obs, act, rew, nobs, done, w = pool
    n = len(rew)
    ref = R.rainbow_grad(pol, pol.flat, pol.target, *pool, 1.0, 1.0 / n)
    p, pt_ = _np_params(pol), _np_params(pol, pol.target)
    o, no = obs.double().numpy(), nobs.double().numpy()
    a_star = _np_forward(p, no, 0, 10)[1].argmax(1)
    lt = _np_forward(pt_, no, 0, 10)[0][np.arange(n), a_star]
    pt = np.exp(lt - lt.max(-1, keepdims=True))
    pt /= pt.sum(-1, keepdims=True)
    m = _np_project(rew.double().numpy(), done.numpy(), pt, 1.0, 0.0, 10.0)
    sel = _np_forward(p, o, 0, 10)[0][np.arange(n), act.numpy()]
    logp = sel - sel.max(-1, keepdims=True)
    logp -= np.log(np.exp(logp).sum(-1, keepdims=True))
    rtd = -(m * logp).sum(-1)
    # NumPy forms the support and the projected returns in float64, the reference in float32 (as the kernel): ~1e-7 apart
    np.testing.assert_allclose(ref.rows.numpy(), rtd, rtol=1e-6, atol=1e-9)
    assert float(ref.loss) == pytest.approx(float((w.double().numpy() * rtd).mean()), rel=1e-6)


# ---- BC / BCQ / CQL -----------------------------------------------------------------------------------------------
def _bq_cpu(algo, K, A, P=48):
    net = R.bq_net(algo, K, A, torch.device("cpu"))
    data = R.bq_data(K, A, P, "cpu", seed=K + A)
    return net, data, R.bq_hyper(algo)


@pytest.mark.parametrize("algo", ["BC", "BCQ", "CQL"])
@pytest.mark.parametrize("KA", [(11, 2), (266, 284), (3082, 284), (4096, 284), (2998, 512), (266, 512)])
def test_batchrl_reference_matches_the_twin(KA, algo):
    K, A = KA
    net, data, hp = _bq_cpu(algo, K, A)
    pool = torch.arange(min(data.n, 48))
    sel = pool[_clear(R.batchrl_grad(net, net.flat, net.target, *data.batch(pool), hp), 40)]
    ref = R.batchrl_grad(net, net.flat, net.target, *data.batch(sel), hp)
    net.flat.grad = None
    loss, st = net.loss(*data.batch(sel), hp)
    loss.backward()
    _per_tensor("batchrl %s K%d A%d" % (algo, K, A), net.flat.grad, ref.grad, net)
    assert torch.allclose(st.double(), ref.stats, rtol=1e-5, atol=1e-6), (st, ref.stats)


@pytest.mark.parametrize("algo", ["BC", "BCQ", "CQL"])
def test_batchrl_reference_matches_numpy(algo):
    """The loss against test_batchrl_cpu's NumPy float64 restatement of the masked net, the targets and the losses."""
    from test_batchrl_cpu import _huber, _lsm, _np_keep, _np_mnet, _np_params
    net, data, hp = _bq_cpu(algo, 266, 284)
    o, a, r, o2, t = data.batch(torch.arange(40))
    ref = R.batchrl_grad(net, net.flat, net.target, o, a, r, o2, t, hp)
    on, on2, an = o.numpy(), o2.numpy(), a.numpy().astype(np.int64)
    rn, tn = r.numpy().astype(np.float64), t.numpy().astype(np.float64)
    rows = np.arange(len(on))
    p = _np_params(net)
    lm = net.location_mask.numpy().astype(np.float64)
    sp = np.nonzero(net.special.numpy())[0]
    k1, k2 = _np_keep(on, lm, sp), _np_keep(on2, lm, sp)

    def bc(z, beta):
        return -_lsm(z)[rows, an] + beta * (z * z).mean(1)
    if algo == "BC":
        want = bc(_np_mnet(on, p, "i_", k1), hp["beta"]).mean()
    elif algo == "BCQ":
        pt = _np_params(net, net.target)
        q2 = _np_mnet(on2, p, "q_", k2)
        lp = _lsm(_np_mnet(on2, p, "i_", k2))
        astar = ((q2 - q2.min(1, keepdims=True)) * ((lp - lp.max(1, keepdims=True)) > hp["log_flex"])).argmax(1)
        y = rn + hp["gamma"] * (1 - tn) * _np_mnet(on2, pt, "q_", k2)[rows, astar]
        want = (_huber(_np_mnet(on, p, "q_", k1)[rows, an] - y) + bc(_np_mnet(on, p, "i_", k1), hp["beta"])).mean()
    else:
        pt = _np_params(net, net.target)

        def c(x, pp):
            h = np.maximum(np.maximum(x.astype(np.float64) @ pp["w1"] + pp["b1"], 0) @ pp["w2"] + pp["b2"], 0)
            return h @ pp["w3"] + pp["b3"]
        rs = ((r - hp["reward_mean"]) / hp["reward_den"]).numpy().astype(np.float64)
        y = rs + hp["gamma"] * (1 - tn) * c(on2, pt)[rows, c(on2, p).argmax(1)]
        q = c(on, p)
        lse = np.log(np.exp(q - q.max(1, keepdims=True)).sum(1)) + q.max(1)
        want = (_huber(q[rows, an] - y) + hp["alpha"] * (lse - q[rows, an])).mean()
    assert abs(float(ref.loss) - want) <= 1e-9 * max(1.0, abs(want)), (float(ref.loss), want)


# ---- decisions ------------------------------------------------------------------------------------------------------
def test_margins_flag_rows_at_a_switch_point():
    """A row put on the huber knee, on an argmax tie or on a relu kink is flagged; the others are clear."""
    from rl4rs_b200.policy import DistributionalQNetwork
    assert float(R.argmax_margin(torch.tensor([[1.0, 1.0, 0.0], [2.0, 0.0, 1.0]], dtype=torch.float64))[0]) == 0.0
    pol = DistributionalQNetwork(4, "cpu", seed=0, num_atoms=4, v_min=-1.0, v_max=1.0)
    g = torch.Generator().manual_seed(0)
    obs, nobs = torch.randn(3, 256, generator=g), torch.randn(3, 256, generator=g)
    nobs[1] = nobs[0]
    act = torch.zeros(3, dtype=torch.int32)
    ref = R.rainbow_grad(pol, pol.flat, pol.target, obs, act, torch.zeros(3), nobs, torch.zeros(3, dtype=torch.uint8), None,
                         1.0, 1.0)
    assert ref.clear().shape == (3,)
    with torch.no_grad():                         # zero the advantage stream: every action's Q is the same, a* is a tie
        lo, hi = pol.slices[7]
        pol.flat[lo:hi] = 0
        lo, hi = pol.slices[6]
        pol.flat[lo:hi] = 0
    ref = R.rainbow_grad(pol, pol.flat, pol.target, obs, act, torch.zeros(3), nobs, torch.zeros(3, dtype=torch.uint8), None,
                         1.0, 1.0)
    assert not bool(ref.clear().any())


# ---- the ABI's shape ranges ---------------------------------------------------------------------------------------
def _lib():
    from rl4rs_b200 import _capi
    return _capi.load_library()


def test_size_functions_at_the_range_edges():
    """The last accepted shape gets a size, the first rejected one -1."""
    lib = _lib()
    assert lib.r4_policy_num_params(2) > 0 and lib.r4_policy_num_params(512) > 0
    assert lib.r4_policy_num_params(1) == -1 and lib.r4_policy_num_params(513) == -1
    for D in (2, 64):
        assert lib.r4_gauss_num_params(D) > 0 and lib.r4_gauss_scratch_size(D) > 0
    for D in (0, 3, 33, 63, 66):
        assert lib.r4_gauss_num_params(D) == -1 and lib.r4_gauss_scratch_size(D) == -1, D
    for twin in (0, 1):
        for D in (2, 32):
            assert lib.r4_ddpg_num_params(D, twin) > 0 and lib.r4_ddpg_scratch_size(D, twin, 1) > 0
        for D in (1, 33):
            assert lib.r4_ddpg_num_params(D, twin) == -1 and lib.r4_ddpg_scratch_size(D, twin, 1) == -1
        assert lib.r4_ddpg_scratch_size(32, twin, 0) == -1
    for A, Z in ((2, 2), (512, 8), (128, 32), (2, 32), (256, 16)):
        assert lib.r4_rainbow_num_params(A, Z) > 0 and lib.r4_rainbow_scratch_size(A, Z, 1) > 0, (A, Z)
    for A, Z in ((513, 2), (1, 8), (2, 33), (2, 1), (241, 17), (512, 9)):
        assert lib.r4_rainbow_num_params(A, Z) == -1 and lib.r4_rainbow_scratch_size(A, Z, 1) == -1, (A, Z)
    for algo in (0, 1, 2):
        for K, A in ((11, 2), (4096, 284), (2998, 512), (266, 512)):
            assert lib.r4_batchrl_num_params(algo, K, A) > 0 and lib.r4_batchrl_scratch_size(algo, K, A, 1) > 0, (K, A)
        for K, A in ((2999, 512), (10, 284), (4097, 284), (266, 513), (266, 1)):
            assert lib.r4_batchrl_num_params(algo, K, A) == -1, (algo, K, A)
            assert lib.r4_batchrl_scratch_size(algo, K, A, 1) == -1 and lib.r4_batchrl_target_size(algo, K, A) == -1


def test_twin_layouts_match_the_abi_sizes():
    """The twins' flat layouts (the reference's tensor lists) have the sizes the ABI reports at every grid shape."""
    from rl4rs_b200.policy import (BatchRLNet, DeterministicActorCritic, DistributionalQNetwork, GaussianPolicy,
                                   MaskedPolicy)
    lib = _lib()
    for A in (2, 31, 512):
        assert lib.r4_policy_num_params(A) == MaskedPolicy(A, "cpu").n_params
    for D in (2, 64):
        assert lib.r4_gauss_num_params(D) == GaussianPolicy(D, "cpu").n_params
    for D in (2, 7):
        assert lib.r4_ddpg_num_params(D, 1) == DeterministicActorCritic(D, "cpu", twin=True).n_params
    for A, Z in ((2, 2), (128, 32), (2, 32)):
        assert lib.r4_rainbow_num_params(A, Z) == DistributionalQNetwork(A, "cpu", num_atoms=Z).n_params
    for algo, k in (("BC", 0), ("BCQ", 1), ("CQL", 2)):
        net = BatchRLNet(algo, 11, np.ones((4, 2)), [1], 2, "cpu")
        assert lib.r4_batchrl_num_params(k, 11, 2) == net.n_params and lib.r4_batchrl_target_size(k, 11, 2) == net.n_target
