"""CPU companion of test_gpu_padqn_shapes.py: what its reference, planted ties and gradient cases must be for the GPU
checks to mean anything, shown without a device.

  reference     padqn_ref64's float64 torch reference (qm_t, loss_and_grads_t) equals the NumPy one at small n
  planted ties  items given identical vectors (item_vectors dup, and every D = 1 item of one sign) have bitwise-equal
                float64 Q values, so "first argmax" is decided exactly on both sides
  grad cases    every gradient case of the GPU grid keeps more than 1 - MAX_DROP of its pool through the tie filter,
                keeps every planted tie row, and populates both Huber branches
  range         every grid point is inside the accepted range; r4_padqn_num_params / _scratch_size / _cache_size return
                -1 exactly one step past each edge (A 2..512, D 1..512, n 1..4194240), and the entry points refuse there
                with no launch
"""
import ctypes as C

import numpy as np
import pytest
import torch

import padqn_ref64 as ref
from test_gpu_padqn_shapes import GRAD_GRID, GRAD_NS, MAXN, NS, PAIR_GRID
from rl4rs_b200 import _capi
from rl4rs_b200.policy import ParametricQNetwork
from rl4rs_b200.trainer import PADQN_MAX_ROWS, PADQNKernelOps


def _net(A, D, onehot=False, seed=0):
    pol = ParametricQNetwork(ref.item_vectors(A, D, seed=seed, onehot=onehot, dup=not onehot), "cpu", seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        pol.flat.add_(0.05 * torch.randn(pol.n_params, generator=g))
        pol.flat[pol.slices[4][0]:pol.slices[4][1]] *= 2.0
        pol.target.copy_(pol.flat.detach() + 0.05 * torch.randn(pol.n_params, generator=g))
    return pol


@pytest.mark.parametrize("A,D", [(2, 1), (33, 7), (129, 33)])
def test_torch_reference_equals_numpy(A, D):
    pol = _net(A, D, seed=A)
    n = 9
    g = torch.Generator().manual_seed(2)
    obs, new_obs = torch.randn(n, 256, generator=g), torch.randn(n, 256, generator=g)
    mask = ref.plant_ties(ref.env_like_masks(n, A, 1), A)
    mask[5] = 0
    action = torch.randint(0, A, (n,), generator=g, dtype=torch.int32)
    reward = torch.randn(n, generator=g) * 2
    done = torch.tensor([1, 0, 0, 1, 0, 0, 0, 1, 0], dtype=torch.uint8)
    w = torch.rand(n, generator=g) + 0.5
    emb = pol.emb.double().numpy()
    P, PT = ref.params(pol.flat.detach().numpy(), D), ref.params(pol.target.numpy(), D)
    pt, ptt = ref.params_t(pol.flat, D, "cpu"), ref.params_t(pol.target, D, "cpu")
    q64 = ref.qm(P, obs.double().numpy(), mask, emb)
    assert np.abs(ref.qm_t(pt, obs, torch.as_tensor(mask), pol.emb).numpy() - q64).max() <= 1e-12 * np.abs(q64[mask != 0]).max()
    loss, td, q, grads = ref.loss_and_grads(P, PT, emb, obs.double().numpy(), action.numpy(), reward.double().numpy(),
                                            new_obs.double().numpy(), done.double().numpy(), mask, w.double().numpy(),
                                            gamma=0.9, inv_n=0.3)
    r = ref.loss_and_grads_t(pt, ptt, pol.emb, obs, action, reward, new_obs, done, torch.as_tensor(mask), w, 0.9, 0.3)
    assert abs(float(r["loss"]) - loss) <= 1e-12 * abs(loss)
    assert np.abs(r["td"].numpy() - td).max() <= 1e-12 * np.abs(td).max()
    assert np.abs(r["q"].numpy() - q).max() <= 1e-12 * np.abs(q).max()
    for k in ref.NAMES:
        assert np.abs(r["grads"][k].numpy() - grads[k]).max() <= 1e-12 * np.abs(grads[k]).max(), k
    st = r["stats"].numpy()
    assert np.allclose(st, [loss, td.sum() * 0.3, q.sum() * 0.3], rtol=1e-12, atol=0)


@pytest.mark.parametrize("A,D", [(2, 1), (2, 512), (31, 7), (284, 1), (512, 33)])
def test_planted_ties_are_exact_in_float64(A, D):
    pol = _net(A, D, seed=A + D)
    obs = torch.randn(40, 256, generator=torch.Generator().manual_seed(0))
    mask = torch.ones(40, A, dtype=torch.uint8)
    q = ref.qm_t(ref.params_t(pol.flat, D, "cpu"), obs, mask, pol.emb)
    emb = pol.emb.numpy()
    for a, b in ref.tie_pairs(A):
        assert np.array_equal(emb[a], emb[b])
        assert torch.equal(q[:, a], q[:, b]), (a, b)
    # every pair of items with equal vectors ties exactly (at D = 1: all of one sign), and no others
    same = (emb[:, None, :] == emb[None, :, :]).all(2)
    eq = (q[:, :, None] == q[:, None, :]).all(0).numpy()
    assert np.array_equal(eq, same)
    # the planted rows: top_gap counts the tie as one value, and argmax takes the first of the pair
    m = torch.as_tensor(ref.plant_ties(np.ones((40, A), np.uint8), A))
    qm = ref.qm_t(ref.params_t(pol.flat, D, "cpu"), obs, m, pol.emb)
    rows = torch.arange(3, 40, 11)
    first = torch.tensor([min(ref.tie_pairs(A)[k % len(ref.tie_pairs(A))]) for k in range(len(rows))])
    assert torch.equal(qm.argmax(1)[rows], first)
    assert bool((ref.top_gap(qm)[rows] > 1e30).all())


@pytest.mark.parametrize("A,D,onehot,gamma,weighted,inv_scale", GRAD_GRID)
def test_grad_cases_keep_their_pools_and_populate_both_huber_branches(A, D, onehot, gamma, weighted, inv_scale):
    """At n = 33 (a 256-row pool, the grid's smallest) every case: the filter drops less than MAX_DROP (asserted inside
    grad_case), keeps every planted tie row, and the selected rows hold td on both sides of the kink, clear of it."""
    pol = _net(A, D, onehot, seed=2 * A + D)
    case = ref.grad_case(pol.flat.detach(), pol.target, pol.emb, 33, gamma, weighted, seed=33, inv_n=inv_scale / 33)
    td = case["ref"]["td"].abs()
    assert int((td < 1).sum()) >= 8 and int((td > 1).sum()) >= 8
    assert float(case["ref"]["kink"].min()) > 0.05
    ties = torch.arange(3, ref.pool_size(33), 11)
    assert bool(case["clear"][ties].all())
    assert case["ref"]["a_star"].shape == (33,)
    if not onehot:
        t = case["idx"][(case["idx"] % 11 == 3)]
        assert t.numel() > 0


def test_dead_next_case_has_non_terminal_all_masked_rows():
    pol = _net(284, 32, seed=5)
    case = ref.grad_case(pol.flat.detach(), pol.target, pol.emb, 64, 0.9, True, seed=5, dead_next=True)
    dead = ~case["next_mask"][case["idx"]].bool().any(1) & (case["done"][case["idx"]] == 0)
    assert int(dead.sum()) >= 3 and bool((case["ref"]["td"][dead] > 1e38).all())
    assert np.isfinite(float(case["ref"]["loss"]))                       # finite in float64; it overflows float32


def test_grid_is_inside_the_accepted_range():
    lib = _capi.load_library()
    ns = set(NS) | set(GRAD_NS) | {65536} | {(s - 1) * 128 // 284 + k for s in (114, 132) for k in (0, 1)}
    for A, D, _ in PAIR_GRID + [g[:3] for g in GRAD_GRID]:
        assert lib.r4_padqn_num_params(A, D) > 0 and lib.r4_padqn_cache_size(A) > 0
        for n in ns:
            assert lib.r4_padqn_scratch_size(A, D, n) > 0, (A, D, n)
    assert lib.r4_padqn_scratch_size(512, 512, 8192) * 4 < 1 << 30            # the largest grid point's scratch: < 1 GB
    assert lib.r4_padqn_scratch_size(512, 32, 65536) * 4 < 1 << 30


def test_minus_one_exactly_one_step_past_each_edge():
    lib = _capi.load_library()
    assert MAXN == PADQN_MAX_ROWS == 4194240
    for D in (1, 512):
        assert lib.r4_padqn_num_params(2, D) > 0 and lib.r4_padqn_num_params(512, D) > 0
        assert lib.r4_padqn_num_params(1, D) == -1 and lib.r4_padqn_num_params(513, D) == -1
    for A in (2, 512):
        assert lib.r4_padqn_num_params(A, 0) == -1 and lib.r4_padqn_num_params(A, 513) == -1
    assert lib.r4_padqn_cache_size(2) > 0 and lib.r4_padqn_cache_size(512) > 0
    assert lib.r4_padqn_cache_size(1) == -1 and lib.r4_padqn_cache_size(513) == -1
    for A in (2, 284, 512):
        for D in (1, 32, 512):
            assert lib.r4_padqn_scratch_size(A, D, 1) > 0 and lib.r4_padqn_scratch_size(A, D, 0) == -1
            assert lib.r4_padqn_scratch_size(A, D, MAXN) > 0, (A, D)
            assert lib.r4_padqn_scratch_size(A, D, MAXN + 1) == -1, (A, D)
        assert lib.r4_padqn_scratch_size(1, 32, 1) == -1 and lib.r4_padqn_scratch_size(513, 32, 1) == -1
        assert lib.r4_padqn_scratch_size(A, 0, 1) == -1 and lib.r4_padqn_scratch_size(A, 513, 1) == -1


def test_entry_points_refuse_past_the_row_limit_without_a_launch():
    """The scratch size is asserted -1 first: r4_padqn_grad and r4_padqn_train_step are called at MAXN + 1 only then."""
    lib = _capi.load_library()
    p = C.c_void_p(16)
    for A in (2, 284, 512):
        assert lib.r4_padqn_scratch_size(A, 32, MAXN + 1) == -1
    n0 = lib.r4_learner_launch_count()
    for A in (2, 284, 512):
        n = MAXN + 1
        assert lib.r4_padqn_act(p, p, p, p, n, A, 32, 0, 0, 0, p, None, p, None) == -1
        assert lib.r4_padqn_grad(p, p, p, p, p, A, 32, p, p, p, p, p, p, p, None, n, 0.9, 0.1, p, p, None, None, None) == -1
        assert lib.r4_padqn_train_step(p, p, p, p, p, p, C.c_void_p(32), A, 32, p, p, p, p, p, p, p, p, 100, n, p, 0.4,
                                       0.6, 1e-6, 1.0, 1, 5e-4, 1e-8, 40.0, 0, p, None, None) == -1
    assert lib.r4_padqn_act(p, p, p, p, MAXN + 1, 284, 32, 0, 0, 0, p, None, p, None) == -1
    assert b"n 1..4194240" in lib.r4_last_error(None)
    assert lib.r4_learner_launch_count() == n0
    emb = torch.zeros(284, 32)
    with pytest.raises(ValueError, match="1..4194240 rows"):
        PADQNKernelOps(emb, "cpu", lib.r4_padqn_num_params(284, 32), MAXN + 1)
