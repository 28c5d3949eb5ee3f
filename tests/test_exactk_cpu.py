"""CPU: Exact-K's torch twin against the float64 restatement (tests/exactk_ref64.py), the point-mask rule, the script's
loop against a scripted env, checkpoints, the options that are not built, and the draw hash against the device's."""
import os
import tempfile

import numpy as np
import pytest
import torch

from rl4rs_b200 import exactk as ek

import exactk_ref64 as ref

T = 284
SPECIAL = [5, 50, 200, 201]


def _gen(seed=3, T=T):
    lm = np.zeros((3, T))
    lm[0, 1:40] = lm[1, 40:148] = lm[2, 148:] = 1
    sp = np.zeros(T)
    sp[[s for s in SPECIAL if s < T]] = 1
    g = ek.Generator(lm[0], lm[1], lm[2], sp, seq_length=T, device="cpu", seed=seed)
    with torch.no_grad():                    # move LayerNorm off its init, where the second block's masks are roundoff
        for k, v in g.params().items():
            if "ln" in k:
                v += 0.1 * torch.randn(v.shape, generator=torch.Generator().manual_seed(seed))
    return g


# (seed, call, stream, element, draw24) recorded from r4_exactk.cuh's draw24
RECORDED = [(0, 1, 0, 0, 12836780), (0, 1, 1, 1000003, 14911966), (0, 1, 2, 1321467903, 3216104), (0, 1, 3, 0, 4152716),
            (7, 2, 0, 1000003, 5533210), (7, 2, 1, 1321467903, 6729115), (7, 2, 2, 0, 6159807), (7, 2, 3, 1000003, 4378821),
            (244837814094590, 123456789, 0, 1321467903, 13357794), (244837814094590, 123456789, 1, 0, 15196259),
            (244837814094590, 123456789, 2, 1000003, 16357759), (244837814094590, 123456789, 3, 1321467903, 5890175)]


def test_hash_mirror_equals_the_device_hash():
    for seed, call, stream, elem, want in RECORDED:
        assert int(ek.draw24(seed, call, stream, torch.tensor([elem]))[0]) == want


@pytest.mark.parametrize("n", [1, 7, 64])
def test_twin_matches_float64_reference(n):
    torch.manual_seed(n)
    g = _gen()
    user = torch.randn(n, 256)
    w64 = ek.unflatten(g.flat.double(), ek.generator_shapes())
    for mode in (ek.SAMPLE, ek.GREEDY):
        path, lg = g.draw(user, mode)
        with torch.no_grad():
            enc = ref.encoder(w64, user.double(), g.seed, g.call, g.rate, T)
            _, want, margin = ref.decoder(w64, enc, g.masks, mode, g.seed, g.call)
        ok = margin > (1e-4 if mode == ek.SAMPLE else 1e-3)
        assert torch.equal(path[ok], want[ok])
    reward = torch.randn(n)
    # the twin's gradient, run in float64 (the float32 twin is the CPU training path; its roundoff is not the point here)
    flat = g.flat.double().clone().requires_grad_(True)
    lg, _ = ek.twin_forward(ek.unflatten(flat, ek.generator_shapes()), user.double(), g.masks, ek.TRAIN, g.seed, g.call,
                            g.rate, target=path)
    loss = ek.policy_loss(lg, path, reward.double())
    loss.backward()
    grad = flat.grad
    want_grad, want_loss, _ = ref.generator_grad(g.flat, user, g.masks, path, reward, g.seed, g.call, g.rate)
    assert abs(float(loss.detach()) - float(want_loss)) <= 1e-4 * abs(float(want_loss))
    for (name, _), a, b in zip(ek.generator_shapes(), ek.unflatten(grad, ek.generator_shapes()).values(),
                               ek.unflatten(want_grad, ek.generator_shapes()).values()):
        assert (a - b).abs().max() <= 1e-6 * max(b.abs().max(), 1e-30), name
    d = ek.Discriminator(device="cpu")
    target = torch.randn(n)
    _, cg, cl = d._run(user, target)
    _, wg, wl = ref.critic(d.flat, user, target)
    assert (cg.double() - wg).abs().max() <= 1e-4 * wg.abs().max()
    assert abs(float(cl) - float(wl)) <= 1e-4 * float(wl)


def test_point_mask_rule_on_random_logits():
    """Random logits through the decode: position t draws from its location mask, never repeats, at most one special."""
    g = _gen()
    with torch.no_grad():
        g.flat += 0.5 * torch.randn(g.flat.shape, generator=torch.Generator().manual_seed(1))
    path, lg = g.draw(torch.randn(64, 256), ek.SAMPLE)
    for t in range(9):
        loc = g.masks[t // 3].bool()
        assert bool(loc[path[:, t]].all())
        assert bool((lg[:, t] > ek.NEG / 2).eq(ek.point_masks(g.masks, path, t)).all())
    for row in path.tolist():
        assert len(set(row)) == 9
        assert sum(i in SPECIAL for i in row) <= 1


class ScriptedEnv(object):
    """Batch env: reset hands out the next window of users; the reward of the ninth step is the scripted value for
    (window, rollout) -- so the test can see which window scored which rollout."""

    def __init__(self, B, rewards):
        self.B, self.rewards, self.resets, self.window, self.steps = B, rewards, 0, -1, 0
        self.users = torch.randn(64, B, 256, generator=torch.Generator().manual_seed(0))

    def reset(self):
        self.resets += 1
        self.window += 1
        self.steps = 0
        return self.users[self.window].numpy()

    def step(self, action):
        self.steps += 1
        r = self.rewards(self.window) if self.steps == 9 else np.zeros(self.B)
        return None, r, self.steps == 9, {}


def _config(B, **kw):
    return dict({"batch_size": B, "action_size": 40, "catalog": _Cat(), "trial_name": "t"}, **kw)


class _Cat(object):
    special_items = [3]


def test_loop_resets_scores_picks_and_normalises(monkeypatch):
    B = 6
    env = ScriptedEnv(B, lambda w: np.array([w, 1, 5, 0, 2, 9], dtype=np.float64) * (1 if w % 3 == 1 else -1))
    seen = {}
    real_critic, real_gen = ek.Discriminator.train, ek.Generator.train

    def critic_train(self, user, target):
        seen["critic"] = (user.clone(), target.clone(), self.predict(user))
        loss = real_critic(self, user, target)
        seen["closs"] = loss
        return loss

    def gen_train(self, user, target, reward):
        seen["gen"] = (user.clone(), target.clone(), reward.clone())
        return real_gen(self, user, target, reward)

    monkeypatch.setattr(ek.Discriminator, "train", critic_train)
    monkeypatch.setattr(ek.Generator, "train", gen_train)
    draws = []
    real_draw = ek.Generator.draw

    def draw(self, user, mode=ek.SAMPLE):
        p, lg = real_draw(self, user, mode)
        draws.append(p)
        return p, lg

    monkeypatch.setattr(ek.Generator, "draw", draw)
    with tempfile.TemporaryDirectory() as out:
        ek.train(_config(B, epoch=1, action_size=40), env=env, device="cpu", output_dir=out, log=None)
    assert env.resets == 3                                     # three resets per episode
    user, target, reward_ = seen["critic"]
    assert torch.equal(user, torch.as_tensor(env.users[0]))
    # rollout 1 is scored on window 0 (the obs's users), rollout 2 on window 1 -- the next batch of users; row 3 ties
    r1 = -np.array([0, 1, 5, 0, 2, 9]) * 1.0
    r2 = np.array([1, 1, 5, 0, 2, 9]) * 1.0
    best = np.where(r2 > r1, r2, r1)                           # ties keep the first rollout
    assert np.allclose(target.numpy(), best)
    assert torch.equal(seen["gen"][1], torch.where(torch.as_tensor(r2 > r1).unsqueeze(1), draws[1], draws[0]))
    # the critic's loss is the batch sum of (target - pred)^2
    assert abs(float(seen["closs"][0]) - float(((target - reward_) ** 2).sum())) < 1e-4 * float(((target - reward_) ** 2).sum())
    adv = best - reward_.double().numpy()
    assert np.allclose(seen["gen"][2].numpy(), adv / np.std(adv), rtol=1e-5)


def test_zero_advantage_std_raises(monkeypatch):
    monkeypatch.setattr(ek.Discriminator, "predict", lambda self, user: torch.zeros(user.shape[0]))
    env = ScriptedEnv(4, lambda w: np.ones(4))
    with tempfile.TemporaryDirectory() as out:
        with pytest.raises(FloatingPointError, match="episode 0"):
            ek.train(_config(4, epoch=2), env=env, device="cpu", output_dir=out, log=None)


def test_checkpoint_round_trip_and_newest_restore():
    env = ScriptedEnv(4, lambda w: np.arange(4.0) * (w + 1))
    with tempfile.TemporaryDirectory() as out:
        gen, critic, _ = ek.train(_config(4, epoch=3), env=env, device="cpu", output_dir=out, log=None)
        d = ek.model_dir(_config(4), out)
        assert d == out + "/exactk_SlateRecEnv-v0_t/"
        assert sorted(os.listdir(d)) == ["exact_k.ckpt.0", "exact_k.ckpt.2"]
        assert ek.newest_checkpoint(d).endswith("exact_k.ckpt.2")
        g2, c2 = ek.build_nets(_config(4), torch.device("cpu"), seed=9)
        assert ek.restore(ek.newest_checkpoint(d), g2, c2) == 2
        assert torch.equal(g2.flat, gen.flat) and torch.equal(c2.flat, critic.flat)
        assert torch.equal(g2.opt.m, gen.opt.m) and g2.opt.step == gen.opt.step == 3 and g2.call == gen.call
        avg = ek.evaluate(_config(4), env=env, device="cpu", output_dir=out, log=None)
        assert np.isfinite(avg)


def test_errors():
    with pytest.raises(ValueError, match="SeqSlateRecEnv-v0"):
        ek.train({"env": "SeqSlateRecEnv-v0"}, env=object())
    with pytest.raises(ValueError, match="SeqSlateRecEnv-v0"):
        ek.evaluate({"env": "SeqSlateRecEnv-v0"}, env=object())
    m = np.ones(T)
    for kw, name in (({"use_mha": False}, "use_mha"), ({"num_layers": 2}, "num_layers"), ({"num_glimpse": 2}, "num_glimpse")):
        with pytest.raises(NotImplementedError, match=name):
            ek.Generator(m, m, m, m, seq_length=T, device="cpu", **kw)
    g = _gen()
    for mode in ("BEAMSEARCH", "CUSTOM"):
        with pytest.raises(NotImplementedError, match=mode):
            g.draw(torch.randn(2, 256), mode)
    with pytest.raises(ValueError, match="stage"):
        ek.main(["test", "{}"])
