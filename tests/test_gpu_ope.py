"""GPU: the off-policy evaluation kernels (csrc/r4_ope.cuh) -- the behaviour forward against the reference's
behavior_model (tests/golden/reference/ope_behavior.npz) and a float64 NumPy forward, the per-step gather against a host
restatement, the C-ABI's rejections and launch counts, determinism -- and ope_eval end to end on the CUDA env."""
import io
import os
import sys
from contextlib import redirect_stdout

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_ope_golden as mk  # noqa: E402

# Forward tolerance: float32 dot products of up to 256 terms (worst-case relative error about 256 eps = 1.5e-5 per layer),
# five layers, then exp, where a logit error d scales a probability by exp(d).  2e-4 relative bounds that with margin.
RTOL = 2e-4


def _lib():
    from rl4rs_b200 import _capi
    return _capi.load_library()


def _weights(H, Cn, seed):
    rs = np.random.RandomState(seed)
    w = {}
    for name, _, shape in __import__("rl4rs_b200.offline_evaluation", fromlist=["dnn_plan"]).dnn_plan(H, Cn):
        scale = 0.3 if name == "emb_cat" else (1.0 / np.sqrt(shape[0]) if len(shape) == 2 else 0.1)
        w[name] = (rs.standard_normal(shape) * scale).astype(np.float32)
    return w


def _forward64(w, head, items, feat, page, K=9):
    """The behaviour net and action_probs' slices in float64 -> [B, C - 1]."""
    B = head.shape[0]
    ids = np.zeros((B, 21), np.int64)
    ids[:, :11] = head
    ids[:, 11:11 + K] = items[:, page * K:(page + 1) * K]
    d = lambda k: w[k].astype(np.float64)
    elu = lambda x: np.where(x > 0, x, np.expm1(np.minimum(x, 0)))
    cat = d("emb_cat")[ids].mean(1)
    dense = np.zeros((B, 50))
    dense[:, :5 * K] = feat[:, page * 5 * K:(page + 1) * 5 * K]
    x = elu(elu(dense @ d("dense_w1") + d("dense_b1")) @ d("dense_w2") + d("dense_b2"))
    a = elu(np.concatenate([cat, x], 1) @ d("fc_w") + d("fc_b"))
    o = elu(a @ d("obs_w") + d("obs_b"))
    z = o @ d("rew_w") + d("rew_b")
    y = np.exp(z - z.max(1, keepdims=True))
    y /= y.sum(1, keepdims=True)
    parts = [y[:, 1:40], y[:, 40:148], y[:, 148:]]
    return np.concatenate([p / p.sum(1, keepdims=True) for p in parts], 1)


def _inputs(B, P, H, seed):
    rs = np.random.RandomState(seed)
    return (rs.randint(0, H, (B, 11)).astype(np.int32), rs.randint(0, 284, (B, 9 * P)).astype(np.int32),
            rs.standard_normal((B, 45 * P)).astype(np.float32))


def _behavior(w, H, Cn, head, items, feat, page, P):
    import torch
    from rl4rs_b200._capi import ptr
    from rl4rs_b200.offline_evaluation import dnn_plan
    lib = _lib()
    flat = torch.from_numpy(np.concatenate([w[n].reshape(-1) for n, _, _ in dnn_plan(H, Cn)])).cuda()
    assert lib.r4_ope_num_params(H, Cn) == flat.numel()
    B = head.shape[0]
    t = [torch.from_numpy(x).cuda() for x in (head, items, feat)]
    out = torch.empty(B, Cn - 1, device="cuda")
    scratch = torch.empty(lib.r4_ope_behavior_scratch_size(B, Cn), device="cuda")
    n0 = lib.r4_ope_launch_count()
    rc = lib.r4_ope_behavior(B, H, Cn, 9, P, page, ptr(flat), ptr(t[0]), ptr(t[1]), ptr(t[2]), ptr(out), ptr(scratch), None)
    assert rc == 0
    torch.cuda.synchronize()
    assert lib.r4_ope_launch_count() - n0 == 7                          # per page: inputs, 5 products, softmax
    return out.cpu().numpy()


@pytest.mark.parametrize("Cn", [284, 300, 1024])
@pytest.mark.parametrize("B", [1, 7, 2048, 4097])
def test_behavior_forward_matches_float64(B, Cn):
    H, P = 3000, 4
    w = _weights(H, Cn, seed=B + Cn)
    head, items, feat = _inputs(B, P, H, seed=B)
    for page in (0, 3):
        got = _behavior(w, H, Cn, head, items, feat, page, P)
        ref = _forward64(w, head, items, feat, page)
        np.testing.assert_allclose(got, ref, rtol=RTOL, atol=1e-9)
        again = _behavior(w, H, Cn, head, items, feat, page, P)
        assert np.array_equal(got.view(np.uint32), again.view(np.uint32))          # reruns are bit-identical


def test_behavior_model_kernels_match_the_reference(tmp_path):
    from rl4rs_b200 import offline_evaluation as oe
    z = np.load(os.path.join(HERE, "golden", "reference", "ope_behavior.npz"))
    p = str(tmp_path / "w.npz")
    np.savez(p, **mk.dnn_weights())
    bm = oe.behavior_model({"action_size": 284, "page_items": 9}, p, device="cuda")
    twin = oe.behavior_model({"action_size": 284, "page_items": 9}, p, device="cuda", use_kernels=False)
    assert bm.use_kernels
    for kind, pages in (("slate", 1), ("seqslate", 4)):
        recs = list(z[kind + "/records"])
        for page in range(pages):
            for layer in range(1, 13):
                a = z["%s/%d/%d/action" % (kind, page, layer)]
                got = bm.action_probs(recs, a, layer, page=page)
                np.testing.assert_allclose(got, z["%s/%d/%d/probs" % (kind, page, layer)], rtol=RTOL, atol=1e-9)
                np.testing.assert_allclose(got, twin.action_probs(recs, a, layer, page=page), rtol=RTOL, atol=1e-9)


def _step_args(B, A, Cn, seed, logits, per_action):
    import torch
    rs = np.random.RandomState(seed)
    probs = rs.standard_normal((B, A)).astype(np.float32) * (3 if logits else 1)
    if logits:
        probs[rs.rand(B, A) < 0.3] = -4294967295.0                 # masked logits
    off = rs.randint(0, A, B).astype(np.int32)
    block = rs.uniform(0, 1, (B, Cn - 1)).astype(np.float32)
    own = rs.randint(0, A, B).astype(np.int32)
    values = rs.standard_normal((B, A) if per_action else (B,)).astype(np.float32)
    rew, offr = rs.standard_normal(B), rs.standard_normal(B)
    host = dict(probs=probs, off=off, block=block, own=own, values=values, rew=rew, offr=offr)
    return host, {k: torch.from_numpy(v).cuda() for k, v in host.items()}


def _run_step(lib, d, t, T, B, A, Cn, layer, logits, per_action, out):
    from rl4rs_b200._capi import ptr
    return lib.r4_ope_step(t, T, B, A, Cn, layer, ptr(d["probs"]), logits, ptr(d["off"]), ptr(d["block"]),
                           ptr(d["own"] if per_action else None), ptr(d["values"]), per_action, ptr(d["rew"]), ptr(d["offr"]),
                           *[ptr(x) for x in out], None)


@pytest.mark.parametrize("logits", [0, 1])
@pytest.mark.parametrize("B,A,Cn", [(1, 2, 149), (7, 284, 284), (2048, 284, 300), (4097, 1000, 1024)])
def test_step_gather_equals_the_host_restatement(B, A, Cn, logits):
    import torch
    from rl4rs_b200.offline_evaluation import block_col
    lib = _lib()
    T = 12
    out = [torch.zeros(T, B, device="cuda") for _ in range(3)] + [torch.zeros(T, B, dtype=torch.float64, device="cuda")
                                                                 for _ in range(2)]
    for t in range(T):
        per_action = t % 2
        h, d = _step_args(B, A, Cn, 100 * t + B, logits, per_action)
        layer = t // 3 + 1
        n0 = lib.r4_ope_launch_count()
        assert _run_step(lib, d, t, T, B, A, Cn, layer, logits, per_action, out) == 0
        assert lib.r4_ope_launch_count() - n0 == 1                      # one launch per step
        torch.cuda.synchronize()
        pol, beh, val, rew, offr = (x[t].cpu().numpy() for x in out)
        rows = np.arange(B)
        col = block_col(layer, torch.from_numpy(h["off"]).long()).numpy()
        assert np.array_equal(beh.view(np.uint32), h["block"][rows, col].view(np.uint32))
        want_val = h["values"][rows, h["own"]] if per_action else h["values"]
        assert np.array_equal(val.view(np.uint32), want_val.view(np.uint32))
        assert np.array_equal(rew, h["rew"]) and np.array_equal(offr, h["offr"])
        if logits:
            z = h["probs"].astype(np.float64)
            e = np.exp(z - z.max(1, keepdims=True))
            ref = e[rows, h["off"]] / e.sum(1)
            # the kernel takes expf of float32 differences z - max (half an ulp of |z - max| <= 32, then 2 ulp of expf)
            np.testing.assert_allclose(pol, ref, rtol=4e-6, atol=1e-30)
        else:
            assert np.array_equal(pol.view(np.uint32), h["probs"][rows, h["off"]].view(np.uint32))
        again = [torch.zeros_like(x) for x in out]
        assert _run_step(lib, d, t, T, B, A, Cn, layer, logits, per_action, again) == 0
        assert all(torch.equal(a[t], b[t]) for a, b in zip(again, out))


def test_entry_points_reject_one_step_past_every_edge_without_a_launch():
    import torch
    from rl4rs_b200._capi import ptr
    lib = _lib()
    B, A, Cn, T = 4, 284, 284, 9
    _, d = _step_args(B, A, Cn, 0, 0, 1)
    out = [torch.zeros(T, B, device="cuda") for _ in range(3)] + [torch.zeros(T, B, dtype=torch.float64, device="cuda")
                                                                 for _ in range(2)]
    n0 = lib.r4_ope_launch_count()
    bad_steps = [dict(t=-1), dict(t=T), dict(T=0), dict(B=0), dict(B=(1 << 21) + 1), dict(A=1), dict(A=65537, Cn=65536),
                 dict(Cn=148), dict(Cn=65537), dict(Cn=283), dict(layer=0), dict(logits=2), dict(per_action=2)]
    for bad in bad_steps:
        a = dict(t=0, T=T, B=B, A=A, Cn=Cn, layer=1, logits=0, per_action=1)
        a.update(bad)
        assert _run_step(lib, d, a["t"], a["T"], a["B"], a["A"], a["Cn"], a["layer"], a["logits"], a["per_action"], out) == -1, bad
    for k in ("probs", "off", "block", "own", "values", "rew", "offr"):
        dd = dict(d, **{k: None})
        assert _run_step(lib, dd, 0, T, B, A, Cn, 1, 0, 1, out) == -1, k
    for i in range(5):
        o = list(out)
        o[i] = None
        assert _run_step(lib, d, 0, T, B, A, Cn, 1, 0, 1, o) == -1, i
    H = 100
    flat = torch.zeros(lib.r4_ope_num_params(H, Cn), device="cuda")
    head, items, feat = (torch.from_numpy(x).cuda() for x in _inputs(B, 2, H, 0))
    res = torch.empty(B, Cn - 1, device="cuda")
    sc = torch.empty(lib.r4_ope_behavior_scratch_size(B, Cn), device="cuda")
    ok = dict(B=B, H=H, Cn=Cn, K=9, P=2, page=1)
    for bad in [dict(B=0), dict(B=(1 << 21) + 1), dict(H=0), dict(H=(1 << 24) + 1), dict(Cn=148), dict(Cn=65537), dict(K=0),
                dict(K=11), dict(P=0), dict(page=-1), dict(page=2)]:
        a = dict(ok, **bad)
        rc = lib.r4_ope_behavior(a["B"], a["H"], a["Cn"], a["K"], a["P"], a["page"], ptr(flat), ptr(head), ptr(items),
                                 ptr(feat), ptr(res), ptr(sc), None)
        assert rc == -1, bad
    args = [ptr(flat), ptr(head), ptr(items), ptr(feat), ptr(res), ptr(sc)]
    for i in range(len(args)):
        a = list(args)
        a[i] = None
        assert lib.r4_ope_behavior(B, H, Cn, 9, 2, 1, *a, None) == -1, i
    assert lib.r4_ope_num_params(0, Cn) == -1 and lib.r4_ope_num_params(H, 148) == -1
    assert lib.r4_ope_behavior_scratch_size(0, Cn) == -1 and lib.r4_ope_behavior_scratch_size(B, 65537) == -1
    assert lib.r4_ope_launch_count() == n0


# ---- end to end on the CUDA env -------------------------------------------------------------------------------
def _env(seq, B, rllib, d3rl):
    """The CUDA env over a synthetic log ingested from its text records (the behaviour model reads them)."""
    from test_gpu_parity import make_env
    from rl4rs_b200 import synth
    from rl4rs_b200.utils.datautil import FeatureUtil
    cfg = {"maxlen": 64, "batch_size": B, "action_size": 284, "class_num": 2, "dense_feature_num": 432,
           "category_feature_num": 21, "category_hash_size": 5000, "seq_num": 2, "emb_size": 128, "hidden_units": 128,
           "max_steps": 36 if seq else 9, "page_items": 9, "action_emb_size": 32, "is_eval": True, "cache_size": B,
           "support_rllib_mask": rllib, "support_d3rl_mask": d3rl}
    cat = synth.make_catalog()
    log = synth.make_log(4 * B, pages=4 if seq else 1, catalog=cat, hash_size=5000, keep_hist=True)
    log = FeatureUtil.parse_log(synth.render_records(log, cat))
    w = synth.make_weights(cfg, stress=2.0, bias_noise=0.1, bounded_scores=True)
    return cfg, cat, make_env(cfg, seq, cat, log, w, output_format="torch")


def _run(cfg, env, algo, bm, use_kernels):
    from rl4rs_b200 import offline_evaluation as oe
    host = []
    saved = oe.StepBuffers.host
    oe.StepBuffers.host = lambda self: host.append(saved(self)) or host[-1]
    try:
        with redirect_stdout(io.StringIO()):
            m = oe.ope_eval(dict(cfg, epoch=1), env, algo, sample_model=bm, use_kernels=use_kernels)
    finally:
        oe.StepBuffers.host = saved
    return m, host[0]


def _reference_metrics(pol, beh, val, rew, offr):
    """offline_evaluation.py:38-69 written out over the copied [T, B] buffers, as the script builds its arrays from the
    per-step lists, calling the estimators directly -> [1, 4, 2]."""
    from rl4rs_b200.utils import offline_policy_metrics as OPE
    rewards, q_values = list(rew), list(val)
    episode_reward = np.sum(np.array(rewards), axis=0)
    action_probs = np.array(list(pol)).swapaxes(0, 1)
    behavior_probs = np.array(list(beh)).swapaxes(0, 1)
    off_rewards = np.array(list(offr)).swapaxes(0, 1)
    off_rewards_sum = np.sum(off_rewards, axis=1)
    rewards_hat = np.array(rewards).swapaxes(0, 1)
    q_values = np.array(q_values).swapaxes(0, 1)
    action_probs_mul = np.multiply.reduce(action_probs * 100, axis=1)
    behavior_probs_mul = np.multiply.reduce(behavior_probs * 100, axis=1)
    cips = OPE.eval_CIPS(off_rewards_sum, action_probs_mul, behavior_probs_mul)
    dr = OPE.eval_doubly_robust(episode_reward, np.average(q_values, 1), off_rewards_sum, action_probs_mul,
                                behavior_probs_mul)
    wips = OPE.eval_WIPS(off_rewards, action_probs, behavior_probs)
    sdr = OPE.eval_seq_doubly_robust(rewards_hat, q_values, off_rewards, action_probs, behavior_probs)
    return np.array([(cips, dr, wips, sdr)])


@pytest.mark.parametrize("seq", [False, True])
def test_ope_eval_end_to_end_kernels_equal_the_twin(seq, tmp_path):
    from rl4rs_b200 import batchrl, offline_evaluation as oe, trainer
    B = 64
    p = str(tmp_path / "w.npz")
    np.savez(p, **dict(_weights(100000, 284, 1)))
    cases = [("BC", False, True), ("BCQ", False, True), ("CQL", False, True), ("PPO", True, False), ("RAINBOW", False, False)]
    for algo, rllib, d3rl in cases:
        cfg, cat, env = _env(seq, B, rllib, d3rl)
        cfg = dict(cfg, catalog=cat)
        if algo in batchrl.ALGOS:
            models = []
            for uk in (True, False):
                m = batchrl.get_model(cfg, algo)
                m.use_kernels = uk
                m.create_impl(env.observation_space.shape[0])
                if algo == "CQL":
                    m.reward_scaler, m.reward_mean, m.reward_std = "standard", 0.3, 1.7
                models.append(m)
            models[1].net.flat.data.copy_(models[0].net.flat.data)
        else:
            models = [trainer.get_rl_model(algo, {"use_kernels": uk}, env, seed=3) for uk in (True, False)]
            models[1].policy.flat.data.copy_(models[0].policy.flat.data)
        res = []
        for model, uk in zip(models, (True, False)):
            bm = oe.behavior_model(dict(cfg), p, device="cuda", use_kernels=uk)
            env.sim._recData.pos = 0
            res.append(_run(cfg, env, model, bm, uk))
        (m_k, h_k), (m_t, h_t) = res
        assert m_k.shape == (1, 4, 2) and np.all(np.isfinite(m_k[:, :, 0])), (algo, m_k)
        for a, b in zip(h_k, h_t):
            np.testing.assert_allclose(a, b, rtol=1e-3, atol=1e-6, err_msg=algo)
        np.testing.assert_allclose(m_k, m_t, rtol=1e-2, atol=1e-6, err_msg=algo)
        pol, beh, val, rew, offr = h_k
        if algo == "CQL":
            val = val * (1.7 + 1e-3) + 0.3
        np.testing.assert_array_equal(m_k, _reference_metrics(pol, beh, val, rew, offr))


def test_kernel_path_refuses_a_batch_other_than_the_buffers_without_a_launch(tmp_path):
    """The gather's buffers hold config['batch_size'] rows: a larger or smaller step batch raises ValueError before
    r4_ope_step could write past them; an action beyond the behaviour net's classes raises IndexError on the host,
    with no device-side fault (the context stays usable)."""
    import torch
    from rl4rs_b200 import offline_evaluation as oe
    lib = _lib()
    B, A, Cn, T = 8, 284, 284, 9
    bufs = oe.StepBuffers(T, B, "cuda", use_kernels=True)
    assert bufs.use_kernels
    n0 = lib.r4_ope_launch_count()
    for n in (B - 1, B + 1, 4 * B):
        h, d = _step_args(n, A, Cn, n, 0, 1)
        with pytest.raises(ValueError, match="batch_size"):
            bufs.gather(0, d["probs"], False, d["off"], d["block"], 1, d["own"], d["values"], d["rew"], d["offr"])
    assert lib.r4_ope_launch_count() == n0
    h, d = _step_args(B, A, Cn, 1, 0, 1)
    bufs.gather(0, d["probs"], False, d["off"], d["block"], 1, d["own"], d["values"], d["rew"], d["offr"])
    assert lib.r4_ope_launch_count() == n0 + 1
    p = str(tmp_path / "w.npz")
    np.savez(p, **mk.dnn_weights())
    bm = oe.behavior_model({"action_size": 284, "page_items": 9}, p, device="cuda")
    recs = list(np.load(os.path.join(HERE, "golden", "reference", "ope_behavior.npz"))["slate/records"])
    with pytest.raises(IndexError):
        bm.action_probs(recs, np.full(len(recs), 284), 3)
    assert np.all(np.isfinite(bm.action_probs(recs, np.full(len(recs), 283), 3)))
    torch.cuda.synchronize()
