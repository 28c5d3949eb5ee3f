"""GPU: the Exact-K kernels (r4_exactk_*) against the float64 restatement tests/exactk_ref64.py, tensor by tensor, at
batch 1, 7, 256 and 2048; the sampled and greedy slates against the reference and the torch twin; the launches per
episode; and a seeded learning check on the synthetic log."""
import os
import tempfile

import numpy as np
import pytest
import torch

from rl4rs_b200 import _capi
from rl4rs_b200 import exactk as ek

import exactk_ref64 as ref

pytestmark = pytest.mark.gpu

T = 284
CHUNK = 128
# decision margins below which a row is reported and left out of the path comparisons (float32 vs float64 roundoff)
GREEDY_GAP, CDF_GAP, MASK_GAP = 1e-4, 1e-5, 1e-4


def _masks():
    from rl4rs_b200 import synth
    from rl4rs_b200.env.slate import SlateState
    lm = SlateState._location_mask(T)
    sp = np.zeros(T)
    sp[[int(x) for x in synth.make_catalog().special_items]] = 1
    return lm, sp


def _generator(seed=3):
    """A generator whose LayerNorm beta / gamma are moved off their initial values: right after init every LayerNorm
    output sums to 0 and the second block's key / query masks are decided by roundoff."""
    lm, sp = _masks()
    g = ek.Generator(lm[0], lm[1], lm[2], sp, seq_length=T, device="cuda", seed=seed)
    w = g.params()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        for k in w:
            if "ln" in k:
                w[k] += 0.1 * torch.randn(w[k].shape, device="cuda", generator=gen)
    return g


def _close(name, got, want, tol=1e-4):
    got, want = got.double(), want.double().to(got.device)
    err = (got - want).abs().max().item()
    scale = want.abs().max().item()
    assert err <= tol * max(scale, 1e-30), "%s: max err %.3g vs max |ref| %.3g" % (name, err, scale)


def _ref_decode(g, user, mode, call):
    w = ek.unflatten(g.flat.double(), ek.generator_shapes())
    paths, margins, mm = [], [], []
    for r0 in range(0, user.shape[0], CHUNK):
        u = user[r0:r0 + CHUNK].double()
        with torch.no_grad():
            enc = ref.encoder(w, u, g.seed, call, g.rate, T, r0)
            _, p, mg = ref.decoder(w, enc, g.masks, mode, g.seed, call, row0=r0)
        paths.append(p)
        margins.append(mg)
        mm.append(ref.mask_margin(w, u, g.seed, call, g.rate, T, r0))
    return torch.cat(paths), torch.cat(margins), torch.cat(mm)


@pytest.mark.parametrize("n", [1, 7, 256, 2048])
def test_generator_entry_points_match_float64(n):
    torch.manual_seed(n)
    g = _generator()
    user = torch.randn(n, 256, device="cuda")
    # SAMPLE / GREEDY: the same slate as the reference on every row away from a decision edge
    for mode, gap in ((ek.SAMPLE, CDF_GAP), (ek.GREEDY, GREEDY_GAP)):
        path, _ = g.draw(user, mode)
        want, margin, mmask = _ref_decode(g, user, mode, g.call)
        ok = (margin > gap) & (mmask > MASK_GAP)
        print("n=%d mode=%d: %d of %d rows near a decision, skipped" % (n, mode, int((~ok).sum()), n))
        assert int((~ok).sum()) <= max(1, n // 20)
        assert torch.equal(path[ok], want[ok])
    # TRAIN: logits, loss and every gradient tensor.  Rows whose key / query mask decisions lie within roundoff get
    # reward 0, so they add nothing to either gradient.  The reference takes the kernels' relu decisions (about 1.8e5
    # relu units per row: at the float32 pre-activation error, up to 3.2e-6 of the token's rms on an H100, most rows hold
    # a unit within roundoff of its kink).
    call = g.call + 1
    w64 = ek.unflatten(g.flat.double(), ek.generator_shapes())
    mm = torch.cat([ref.mask_margin(w64, user[r0:r0 + CHUNK].double(), g.seed, call, g.rate, T, r0)
                    for r0 in range(0, n, CHUNK)])
    print("n=%d: %d rows near a mask decision left out of the gradient" % (n, int((mm <= MASK_GAP).sum())))
    reward = torch.randn(n, device="cuda") * (mm > MASK_GAP)
    grad, loss = g.grad(user, path, reward)
    keep = ref.device_relu_decisions(g, n)
    got_logits = torch.empty(n, 9, T, device="cuda")
    lib = _capi.load_library()
    tgt = path.to(torch.int32).contiguous()
    _capi.check(lib, None, lib.r4_exactk_decode(_capi.ptr(g.flat), _capi.ptr(user), n, T, _capi.ptr(g.masks), ek.TRAIN, 1.0,
                                                g.seed, call, g.rate, _capi.ptr(tgt), _capi.ptr(got_logits),
                                                _capi.ptr(g._scr(n)), _capi.stream(g.device)), "r4_exactk_decode")
    want_grad = torch.zeros(g.flat.numel(), dtype=torch.float64, device="cuda")
    want_loss = 0.0
    for r0 in range(0, n, CHUNK):
        gr, l, lg = ref.generator_grad(g.flat, user[r0:r0 + CHUNK], g.masks, path[r0:r0 + CHUNK], reward[r0:r0 + CHUNK],
                                       g.seed, call, g.rate, row0=r0, n_total=n,
                                       relu_keep={k: v[r0:r0 + CHUNK] for k, v in keep.items()})
        want_grad += gr
        want_loss += float(l)
        live = lg > ref.NEG / 2
        _close("logits rows %d+" % r0, got_logits[r0:r0 + CHUNK][live], lg[live])
    _close("loss", loss, torch.tensor([want_loss]))
    rel = {}
    for (name, _), a, b in zip(ek.generator_shapes(), ek.unflatten(grad, ek.generator_shapes()).values(),
                               ek.unflatten(want_grad, ek.generator_shapes()).values()):
        rel[name] = (a.double() - b).abs().max().item() / max(b.abs().max().item(), 1e-30)
    print("n=%d gradient error / max |ref|: %s" % (n, ", ".join("%s %.2g" % kv for kv in sorted(rel.items(), key=lambda kv: -kv[1]))))
    bad = {k: v for k, v in rel.items() if v > 1e-4}
    assert not bad, bad


@pytest.mark.parametrize("n", [1, 7, 256, 2048])
def test_critic_and_adam_match_float64(n):
    torch.manual_seed(n)
    d = ek.Discriminator(device="cuda")
    user = torch.randn(n, 256, device="cuda")
    target = torch.randn(n, device="cuda")
    pred = d.predict(user)
    wp, wg, wl = ref.critic(d.flat, user, target)
    _close("pred", pred, wp)
    _, grad, loss = d._run(user, target)
    _close("critic grad", grad, wg)
    _close("critic loss", loss, wl.view(1))
    for net, flat in ((ek.CRITIC, d.flat), (ek.GENERATOR, ek.init_generator(1).cuda())):
        opt = ek._Adam(net, flat, 0.005)
        cpu = ek._Adam(net, flat.cpu().double(), 0.005)
        for _ in range(3):
            gr = torch.randn(flat.shape, device="cuda")
            opt.apply(gr)
            cpu.apply(gr.cpu().double())
        _close("adam net %d" % net, flat, cpu.flat, 1e-5)


def test_device_paths_equal_the_twin():
    """The same seed and call give the twin (torch ops on the device) and the kernels the same slates."""
    n = 64
    g = _generator(5)
    user = torch.randn(n, 256, device="cuda")
    for mode in (ek.SAMPLE, ek.GREEDY):
        path, _ = g.draw(user, mode)
        with torch.no_grad():
            _, twin = ek.twin_forward(g.params(), user, g.masks, mode, g.seed, g.call, g.rate)
        _, margin, mmask = _ref_decode(g, user, mode, g.call)
        ok = (margin > (CDF_GAP if mode == ek.SAMPLE else GREEDY_GAP)) & (mmask > MASK_GAP)
        assert torch.equal(path[ok], twin[ok])


def _env(B, n_log=None):
    from test_gpu_parity import _synthetic, make_env
    cfg, cat, log, w = _synthetic(B, False, is_eval=False, n_log=n_log or 8 * B, cache_size=8 * B)
    env = make_env(cfg, False, cat, log, w, output_format="torch")
    return dict(cfg, catalog=cat), env


LAUNCHES_PER_EPISODE = 2 * 122 + 5 + 27 + 1 + 349 + 1     # two decodes, critic predict / step / Adam, generator grad / Adam


def test_launches_per_episode():
    lib = _capi.load_library()
    cfg, env = _env(64)
    with tempfile.TemporaryDirectory() as out:
        ek.train(dict(cfg, epoch=1, trial_name="l"), env=env, output_dir=out, log=None)
        c0 = lib.r4_exactk_launch_count()
        ek.train(dict(cfg, epoch=3, trial_name="l"), env=env, output_dir=out, log=None)
        assert lib.r4_exactk_launch_count() - c0 == 3 * LAUNCHES_PER_EPISODE


def _greedy_reward(gen, env, batches=4):
    total = 0.0
    for _ in range(batches):
        obs = env.reset()
        path, _ = gen.draw(obs, ek.GREEDY)
        for step in range(9):
            _, reward, _, _ = env.step(path[:, step])
        total += float(reward.double().mean())
    return total / batches


LEARN_MARGIN = 100.0


def test_training_raises_the_greedy_reward():
    """Seeded: 150 episodes at batch 128 on the synthetic log raise the greedy slate's mean reward (dropout live, four
    batches) by at least LEARN_MARGIN over the untrained generator's.  Measured on an H100 in five runs: untrained
    231-238, trained 448-501, a gap of at least 211; the margin is under half of that."""
    B, N = 128, 150
    cfg, env = _env(B)
    torch.manual_seed(0)
    gen0, _ = ek.build_nets(dict(cfg), torch.device("cuda"))
    before = _greedy_reward(gen0, env)
    with tempfile.TemporaryDirectory() as out:
        gen, _, stats = ek.train(dict(cfg, epoch=N, trial_name="fit"), env=env, output_dir=out, log=None)
        after = _greedy_reward(gen, env)
        assert sorted(os.listdir(os.path.join(out, "exactk_SlateRecEnv-v0_fit"))) == ["exact_k.ckpt.0", "exact_k.ckpt.%d" % (N - 1)]
        avg = ek.evaluate(dict(cfg, trial_name="fit"), env=env, output_dir=out, log=None)
    print("greedy reward: untrained %.4f, after %d episodes %.4f (eval stage %.4f)" % (before, N, after, avg))
    assert all(np.isfinite(s["policy_loss"]) for s in stats)
    assert after >= before + LEARN_MARGIN, (before, after)


def test_out_of_range_targets_are_clamped():
    """A teacher path outside [0, T) is clamped into it: the same logits and gradient as the clamped path."""
    n = 7
    g = _generator(6)
    user = torch.randn(n, 256, device="cuda")
    path, _ = g.draw(user, ek.GREEDY)
    reward = torch.randn(n, device="cuda")
    bad = path.clone()
    bad[0, 0], bad[1, 4], bad[2, 8] = -5, T + 3, 10 ** 6
    fixed = bad.clamp(0, T - 1)
    call = g.call
    g.call = call
    want, wl = g.grad(user, fixed, reward)
    g.call = call
    got, gl = g.grad(user, bad, reward)
    assert torch.equal(got, want) and torch.equal(gl, wl)
