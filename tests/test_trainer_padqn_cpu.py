"""CPU: PA-DQN on the discrete env -- the get_rl_model dispatch and its refusals, the parameter layout and init, the torch
twin against the float64 reference (planted masks, done rows, all-masked rows), the next-mask store, SoftQ frequencies, the
target-copy schedule, checkpoints, the C-ABI's refusals without a launch, and learning on a fake env whose reward depends
on the item vectors."""
import os
import tempfile

import numpy as np
import pytest
import torch

import padqn_ref64 as ref
from rl4rs_b200.policy import ParametricQNetwork
from rl4rs_b200.trainer import PADQNTrainer, PAReplayBuffer, get_rl_model

A, D = 40, 8


class FakeEnv(object):
    """Torch-format env protocol on CPU with the RLlib mask: random obs [B, 256], random masks (at least one item per row),
    reward = e(a) . u for a fixed direction u of the item space, done on the last step."""

    def __init__(self, B, T=4, seed=0, A=A, D=D, **flags):
        self.config = dict({"max_steps": T, "batch_size": B, "action_size": A, "support_rllib_mask": True}, **flags)
        self.B, self.T, self.A = B, T, A
        self.g = torch.Generator().manual_seed(seed)
        emb = ref.item_vectors(A, D, seed=7)
        engine = type("E", (), {"device": torch.device("cpu"), "action_emb": emb})()
        self.sim = type("S", (), {"engine": engine})()
        u = np.zeros(D)
        u[0] = 1.0
        self.item_reward = torch.as_tensor(emb @ u, dtype=torch.float32)

    def _obs(self):
        m = (torch.rand(self.B, self.A, generator=self.g) < 0.5).to(torch.uint8)
        m[:, 0] = 1
        return {"obs": torch.randn(self.B, 256, generator=self.g), "action_mask": m}

    def reset(self):
        self.t = 0
        self.last = self._obs()
        return self.last

    def step(self, a):
        assert a.dtype == torch.int32 and a.shape == (self.B,)
        assert bool(self.last["action_mask"][torch.arange(self.B), a.long()].all()), "a masked action was taken"
        self.t += 1
        r = self.item_reward[a.long()]
        self.last = self._obs()
        return self.last, r, torch.full((self.B,), int(self.t >= self.T)), {}


def test_dispatch_and_refusals():
    assert type(get_rl_model("PADQN", {}, env=FakeEnv(8), device="cpu")) is PADQNTrainer
    with pytest.raises(ValueError, match="support_rllib_mask"):
        get_rl_model("PADQN", {}, env=FakeEnv(8, support_rllib_mask=False), device="cpu")
    with pytest.raises(ValueError, match="support_conti_env"):
        get_rl_model("PADQN", {}, env=FakeEnv(8, support_conti_env=True), device="cpu")
    with pytest.raises(NotImplementedError):
        get_rl_model("PADQN_rawstate", {}, env=FakeEnv(8), device="cpu")
    with pytest.raises(NotImplementedError):
        get_rl_model("PADQN", {}, env=FakeEnv(8, rawstate_as_obs=True), device="cpu")
    for algo in ("DQN", "SLATEQ", "PADQN_conti"):
        with pytest.raises(NotImplementedError):
            get_rl_model(algo, {}, env=FakeEnv(8), device="cpu")
    with pytest.raises(AssertionError):              # the name is matched exactly: any other spelling is unknown
        get_rl_model("padqn", {}, env=FakeEnv(8), device="cpu")


def test_world_above_one_is_refused(monkeypatch):
    import rl4rs_b200.trainer as tr
    monkeypatch.setattr(tr, "_world", lambda: 2)
    with pytest.raises(NotImplementedError, match="data-parallel"):
        get_rl_model("PADQN", {}, env=FakeEnv(8), device="cpu")


def test_defaults_layout_and_init():
    tr = get_rl_model("PADQN", {"no_such_key": 1}, env=FakeEnv(200, T=9, A=284, D=32), device="cpu")
    c = tr.config
    assert (c["lr"], c["adam_epsilon"], c["grad_clip"], c["gamma"]) == (5e-4, 1e-8, 40.0, 1.0)
    assert (c["buffer_size"], c["learning_starts"], c["target_network_update_freq"]) == (100000, 1000, 200)
    assert (c["prioritized_replay_alpha"], c["prioritized_replay_beta"], c["prioritized_replay_eps"]) == (0.6, 0.4, 1e-6)
    assert c["timesteps_per_iteration"] == 1000
    assert tr.n_local == 1024 and tr.replay.prio is not None and tr.replay.action.dtype == torch.int32
    assert tr.replay.next_mask.shape == (100000, 284) and tr.replay.next_mask.dtype == torch.uint8
    assert get_rl_model("PADQN", {}, env=FakeEnv(8, T=9), device="cpu").n_local == 72
    pol = tr.policy
    assert pol.n_params == (256 + 32) * 256 + 256 + 256 * 256 + 256 + 256 + 1 == 140033 and len(pol.slices) == 6
    from rl4rs_b200 import _capi
    lib = _capi.load_library()
    assert lib.r4_padqn_num_params(284, 32) == 140033 and lib.r4_padqn_num_params(284, 284) == pol.n_params + 252 * 256
    p = {k: v.detach() for k, v in pol.params().items()}
    for k, std in (("w1", 1.0), ("w2", 1.0), ("w3", 0.01)):          # normc: column norms std
        assert torch.allclose(p[k].norm(dim=0), torch.full((p[k].shape[1],), std), rtol=1e-5)
    assert all(bool((p[k] == 0).all()) for k in ("b1", "b2", "b3"))
    assert torch.equal(pol.target, pol.flat.detach())
    assert torch.equal(pol.emb, torch.as_tensor(ref.item_vectors(284, 32, seed=7), dtype=torch.float32))


def _perturbed(seed, A=A, D=D, scale=0.05):
    pol = ParametricQNetwork(ref.item_vectors(A, D, seed=3), "cpu", seed=seed)
    g = torch.Generator().manual_seed(seed + 100)
    with torch.no_grad():
        pol.flat.add_(scale * torch.randn(pol.n_params, generator=g))
        pol.target.copy_(pol.flat.detach() + scale * torch.randn(pol.n_params, generator=g))
    return pol


@pytest.mark.parametrize("regime", ["ones", "env", "planted"])
def test_twin_qm_matches_float64(regime):
    pol = _perturbed(1)
    n = 23
    obs = torch.randn(n, 256, generator=torch.Generator().manual_seed(2))
    mask = {"ones": np.ones((n, A), np.uint8), "env": ref.env_like_masks(n, A, 1), "planted": ref.planted_masks(n, A, 1)}[regime]
    q = pol.forward(obs, torch.as_tensor(mask)).detach()
    q64 = ref.qm(ref.params(pol.flat.detach().numpy(), D), obs.double().numpy(), mask, pol.emb.double().numpy())
    assert np.array_equal(q.numpy() == ref.FLOAT_MIN, mask == 0)
    live = mask != 0
    assert np.abs(q.numpy()[live] - q64[live]).max() <= 1e-4 * np.abs(q64[live]).max()
    if regime == "planted":                       # all-masked rows: every value float32.min, the argmax is item 0
        dead = ~live.any(1)
        assert dead.sum() == 4 and bool((pol.act(obs, torch.as_tensor(mask), False)[0][torch.as_tensor(dead)] == 0).all())


def _batch(n, seed, A=A):
    g = torch.Generator().manual_seed(seed)
    obs, new_obs = torch.randn(n, 256, generator=g), torch.randn(n, 256, generator=g)
    nm = ref.planted_masks(n, A, seed)
    done = torch.zeros(n, dtype=torch.uint8)
    done[::3] = 1
    done[torch.as_tensor(~nm.any(1))] = 1           # an all-masked next state only at an episode's end
    action = torch.randint(0, A, (n,), generator=g, dtype=torch.int32)
    reward = torch.randn(n, generator=g)
    weights = torch.rand(n, generator=g) + 0.5
    return obs, action, reward, new_obs, done, torch.as_tensor(nm), weights


def test_twin_loss_and_gradient_match_float64():
    pol = _perturbed(4)
    obs, action, reward, new_obs, done, nm, weights = _batch(31, 5)
    loss, td, q = pol.loss(obs, action, reward, new_obs, done, nm, weights, gamma=0.9)
    loss.backward()
    P, PT = ref.params(pol.flat.detach().numpy(), D), ref.params(pol.target.numpy(), D)
    l64, td64, q64, g64 = ref.loss_and_grads(P, PT, pol.emb.double().numpy(), obs.double().numpy(), action.numpy(),
                                             reward.double().numpy(), new_obs.double().numpy(), done.double().numpy(),
                                             nm.numpy(), weights.double().numpy(), gamma=0.9)
    assert abs(float(loss) - l64) <= 1e-5 * max(1.0, abs(l64))
    np.testing.assert_allclose(td.numpy(), td64, atol=1e-4 * np.abs(td64).max())
    np.testing.assert_allclose(q.numpy(), q64, atol=1e-4 * np.abs(q64).max())
    assert (np.abs(td64) > 1).any() and (np.abs(td64) < 1).any()          # both Huber branches
    flat_g = pol.flat.grad.numpy()
    for (lo, hi), k in zip(pol.slices, ref.NAMES):
        g = g64[k].reshape(-1)
        assert np.abs(flat_g[lo:hi] - g).max() <= 1e-4 * np.abs(g).max(), k


def test_double_q_target_uses_online_argmax_and_target_values():
    pol = _perturbed(6)
    _, _, reward, new_obs, done, nm, _ = _batch(17, 8)
    P, PT = ref.params(pol.flat.detach().numpy(), D), ref.params(pol.target.numpy(), D)
    emb = pol.emb.double().numpy()
    a_star, y = ref.target(P, PT, new_obs.double().numpy(), nm.numpy(), reward.double().numpy(), done.double().numpy(), 1.0, emb)
    on = ref.qm(P, new_obs.double().numpy(), nm.numpy(), emb)
    tg = ref.qm(PT, new_obs.double().numpy(), nm.numpy(), emb)
    assert (tg.argmax(1) != a_star).any()           # the two nets disagree somewhere: the online argmax is what counts
    live = done.numpy() == 0
    assert np.allclose(y[live], reward.double().numpy()[live] + tg[live, a_star[live]])
    assert np.array_equal(y[~live], reward.double().numpy()[~live])
    assert np.array_equal(a_star, on.argmax(1)) and bool(nm.numpy()[np.arange(17), a_star][nm.numpy().any(1)].all())


def test_clip_adam_and_target_copy_match_float64():
    tr = get_rl_model("PADQN", {"grad_clip": 0.01}, env=FakeEnv(8), device="cpu")
    pol = tr.policy
    batch = _batch(24, 9)
    f0, t0 = pol.flat.detach().double().numpy().copy(), pol.target.double().numpy().copy()
    P, PT = ref.params(f0, D), ref.params(t0, D)
    b64 = [x.double().numpy() if x.is_floating_point() else x.numpy() for x in batch]
    _, _, _, g64 = ref.loss_and_grads(P, PT, pol.emb.double().numpy(), b64[0], b64[1], b64[2], b64[3], b64[4].astype(np.float64),
                                      b64[5], b64[6])
    tr.twin_step(*batch, copy_target=True)
    f1, t1, _, _ = ref.apply(f0, t0, ref.flat_grad(g64, D), np.zeros_like(f0), np.zeros_like(f0), 1, D, clip=0.01,
                             copy_target=True)
    # a first Adam step moves every weight by about lr: 1 % of it is the float32 bar (g near eps sets the worst element)
    assert np.abs(pol.flat.detach().double().numpy() - f1).max() < 5e-6
    assert torch.equal(pol.target, pol.flat.detach())
    g = ref.flat_grad(g64, D)
    assert sum(np.linalg.norm(g[lo:hi]) > 0.01 for lo, hi in pol.slices) >= 3   # the clip bites on most tensors


def test_next_mask_store_with_terminal_row():
    T, B, C = 3, 4, 10
    rb = PAReplayBuffer(C, A, torch.device("cpu"), True)
    g = torch.Generator().manual_seed(0)
    obs, final_obs = torch.randn(T, B, 256, generator=g), torch.randn(B, 256, generator=g)
    mask = (torch.rand(T, B, A, generator=g) < 0.5).to(torch.uint8)
    final_mask = (torch.rand(B, A, generator=g) < 0.5).to(torch.uint8)
    action = torch.randint(0, A, (T, B), generator=g, dtype=torch.int32)
    reward, done = torch.randn(T, B, generator=g), torch.zeros(T, B, dtype=torch.uint8)
    done[-1] = 1
    rb.added = 7
    rb.store(obs, final_obs, action, reward, done, mask, final_mask)
    for r in range(T * B - C, T * B):                # only the last C rows land, at (7 + r) % C
        t, b, s = r // B, r % B, (7 + r) % C
        want = final_mask[b] if t == T - 1 else mask[t + 1, b]
        assert torch.equal(rb.next_mask[s], want)
        assert torch.equal(rb.new_obs[s], final_obs[b] if t == T - 1 else obs[t + 1, b])
        assert rb.action[s] == action[t, b] and rb.done[s] == done[t, b]
    assert rb.added == 7 + T * B and len(rb.gather(torch.tensor([0, 1]))) == 6


def test_softq_frequencies_match_softmax():
    pol = _perturbed(10, scale=0.0)
    with torch.no_grad():
        pol.flat[pol.slices[4][0]:pol.slices[4][1]] *= 2000.0      # Q spread over a few units
    obs = torch.randn(1, 256, generator=torch.Generator().manual_seed(3)).repeat(20000, 1)
    mask = torch.as_tensor(ref.env_like_masks(1, A, 2, keep=0.2)).repeat(20000, 1)
    a, q = pol.act(obs, mask, True, seed=11, counter=0)
    q0 = q[0].double()
    assert float(q0[mask[0].bool()].max() - q0[mask[0].bool()].min()) > 1.0
    p = torch.softmax(q0, 0).numpy()
    cnt = np.bincount(a.numpy(), minlength=A)
    assert cnt[mask[0].numpy() == 0].sum() == 0
    live = p > 0.005
    chi2 = ((cnt[live] - 20000 * p[live]) ** 2 / (20000 * p[live])).sum()
    assert chi2 < 3 * live.sum(), chi2
    u = ref.uniforms(11, 0, 20000)
    assert np.array_equal(a.numpy(), ref.act(q.double().numpy(), u))


def test_target_copy_schedule():
    tr = get_rl_model("PADQN", {"learning_starts": 32, "timesteps_per_iteration": 32, "train_batch_size": 16,
                                "target_network_update_freq": 40}, env=FakeEnv(8), device="cpu")
    copies = []
    orig = tr.twin_step

    def spy(*a, **k):
        copies.append((tr.policy_ts, bool(a[-1])))
        return orig(*a, **k)
    tr.twin_step = spy
    for _ in range(4):
        tr.train()
    # one SGD step per rollout of 32 timesteps: a step copies once 40 timesteps were sampled since the last copy
    assert [c for _, c in copies] == [False, True, False, True]
    assert [t for t, _ in copies] == [32, 64, 96, 128]


def test_checkpoint_round_trip_and_cross_algorithm_refusal():
    cfg = {"learning_starts": 32, "timesteps_per_iteration": 32, "train_batch_size": 16}
    tr = get_rl_model("PADQN", cfg, env=FakeEnv(8, seed=1), device="cpu", seed=3)
    tr.train(); tr.train()
    with tempfile.TemporaryDirectory() as d:
        path = tr.save(d)
        tr2 = get_rl_model("PADQN", cfg, env=FakeEnv(8, seed=1), device="cpu", seed=99)
        tr2.restore(path)
        assert torch.equal(tr2.policy.flat, tr.policy.flat) and torch.equal(tr2.policy.target, tr.policy.target)
        assert (tr2.counter, tr2.policy_ts, tr2.critic_steps, tr2.last_target_update) == \
            (tr.counter, tr.policy_ts, tr.critic_steps, tr.last_target_update)
        batch = _batch(16, 12)
        s1, s2 = tr.twin_step(*batch, copy_target=False), tr2.twin_step(*batch, copy_target=False)
        assert torch.equal(s1[1], s2[1]) and torch.equal(tr.policy.flat, tr2.policy.flat)
        from test_trainer_rainbow_cpu import FakeEnv as PlainEnv
        rb = get_rl_model("RAINBOW", {}, env=PlainEnv(8), device="cpu")
        rpath = rb.save(os.path.join(d, "rb"))
        with pytest.raises(AssertionError):
            tr2.restore(rpath)
        with pytest.raises(AssertionError):
            rb.restore(path)


def test_learns_the_item_reward():
    env = FakeEnv(16, T=4, seed=5)
    tr = get_rl_model("PADQN", {"learning_starts": 64, "timesteps_per_iteration": 256, "train_batch_size": 64,
                                "target_network_update_freq": 64, "lr": 1e-3}, env=env, device="cpu", seed=0)
    torch.manual_seed(0)
    before = np.mean([tr.evaluate() for _ in range(4)])
    for _ in range(30):
        tr.train()
    after = np.mean([tr.evaluate() for _ in range(4)])
    # the best live item per step is worth ~ +1.5 in e(a)[0] units over 4 steps; the untrained net picks at random
    assert after > before + 1.0 and after > 2.0, (before, after)


def test_capi_refuses_bad_arguments_without_a_launch():
    import ctypes as C
    from rl4rs_b200 import _capi
    lib = _capi.load_library()
    p = C.c_void_p(16)
    n0 = lib.r4_learner_launch_count()
    assert lib.r4_padqn_num_params(1, 32) == -1 and lib.r4_padqn_num_params(513, 32) == -1
    assert lib.r4_padqn_num_params(2, 0) == -1 and lib.r4_padqn_num_params(512, 513) == -1
    assert lib.r4_padqn_num_params(2, 1) > 0 and lib.r4_padqn_num_params(512, 512) > 0
    assert lib.r4_padqn_scratch_size(284, 32, 0) == -1 and lib.r4_padqn_cache_size(513) == -1
    assert lib.r4_padqn_scratch_size(512, 32, (2 ** 31 - 1 - 128) // 512 + 1) == -1
    # the scratch grows with n (256 + D + A), never with n A 256
    s1, s2 = lib.r4_padqn_scratch_size(284, 32, 4096), lib.r4_padqn_scratch_size(284, 32, 8192)
    assert s2 - s1 < 4096 * 4096 and s2 < 8192 * 284 * 256 // 10
    st = None
    assert lib.r4_padqn_refresh(p, p, 284, 32, p, p, st) == -1                   # the two caches may not alias
    assert lib.r4_padqn_refresh(p, p, 1, 32, p, None, st) == -1
    assert lib.r4_padqn_act(p, p, p, None, 8, 284, 32, 0, 0, 0, p, None, p, st) == -1
    assert lib.r4_padqn_act(p, p, p, p, 0, 284, 32, 0, 0, 0, p, None, p, st) == -1
    assert lib.r4_padqn_act(p, p, p, p, 8, 284, 600, 0, 0, 0, p, None, p, st) == -1
    assert lib.r4_padqn_act(p, p, p, p, 8, 284, 32, 0, 0, 0, p, None, C.c_void_p(20), st) == -1   # an unaligned scratch
    assert lib.r4_padqn_store(p, p, p, p, p, None, None, None, 10, 284, 0, 0.6, p, p, p, p, p, p, p, 3, 4, st) == -1
    assert lib.r4_padqn_store(p, p, p, p, p, p, p, None, 10, 284, 0, 0.6, p, p, p, p, p, p, p, 3, 4, st) == -1
    assert lib.r4_padqn_grad(p, p, p, p, p, 284, 32, p, p, p, p, p, None, p, None, 8, 1.0, 0.1, p, p, None, None, st) == -1
    assert lib.r4_padqn_apply(p, p, p, p, p, p, 284, 32, p, p, 1, 5e-4, 1e-8, 40.0, 0, st) == -1
    assert lib.r4_padqn_apply(p, p, p, p, p, p, 284, 32, p, C.c_void_p(32), 0, 5e-4, 1e-8, 40.0, 0, st) == -1
    args = [p] * 6 + [C.c_void_p(32), 284, 32] + [p] * 8 + [100, 8, p, 0.4, 0.6, 1e-6, 1.0, 1, 5e-4, 1e-8, 40.0, 0, p, None, st]
    bad = list(args)
    bad[14] = None                                   # no next-mask ring
    assert lib.r4_padqn_train_step(*bad) == -1
    bad = list(args)
    bad[17] = 0                                      # an empty replay
    assert lib.r4_padqn_train_step(*bad) == -1
    assert lib.r4_learner_launch_count() == n0
