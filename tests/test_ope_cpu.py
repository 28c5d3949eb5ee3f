"""CPU: off-policy evaluation (rl4rs_b200.offline_evaluation, utils.offline_policy_metrics) against the reference's own
code, stored under tests/golden/reference/ by tests/golden/make_ope_golden.py: the estimators, the script's flow with
recorders replaying fixed arrays, and the behaviour model's torch twin; weight loading, the trainers' full_fetch infos and
the inputs that must raise."""
import io
import os
import sys
import types
from contextlib import redirect_stdout

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "reference")
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_ope_golden as mk  # noqa: E402
from rl4rs_b200 import offline_evaluation as oe  # noqa: E402
from rl4rs_b200.utils import offline_policy_metrics as OPE  # noqa: E402


def _golden(name):
    return np.load(os.path.join(GOLDEN, name))


def test_estimators_match_the_reference_grid():
    """Every estimator on every grid point to 1e-5 relative (the reference keeps float32 ratios, so do they here); where
    the reference raises (int(n_e) of a NaN), so do they."""
    z = _golden("ope_metrics.npz")
    g = vars(OPE)
    n = 0
    for name, x in mk.metric_inputs():
        for k, f in mk.metric_calls(g, x).items():
            key = name + "/" + k
            if key + "_raises" in z.files:
                with pytest.raises(ValueError):
                    f()
                continue
            got = np.asarray(f(), np.float64)
            np.testing.assert_allclose(got, z[key], rtol=1e-5, atol=0, equal_nan=True, err_msg=key)
            n += 1
        if name + "/seqw" in z.files:
            np.testing.assert_array_equal(OPE._calc_sequential_weigths(x["pol"], x["beh"], a_min=0.1, a_max=10),
                                          z[name + "/seqw"])
        _, n_e, cv = OPE._calc_sample_weigths(x["apm"], x["bpm"], a_min=0.1, a_max=10)
        np.testing.assert_allclose([n_e, cv], z[name + "/ne_cv"], rtol=1e-6, equal_nan=True)
    assert n > 150
    assert np.isnan(z["ne1_2_1/ne_cv"][1]) and int(z["ne1_2_1/ne_cv"][0]) - 1 == 0


def _f64_restatement(x):
    """The estimators written out directly in float64."""
    from scipy import stats
    pol, beh, off, hat, q = (np.asarray(x[k], np.float64) for k in ("pol", "beh", "off", "hat", "q"))
    apm, bpm, offs, ep = (np.asarray(x[k], np.float64) for k in ("apm", "bpm", "offs", "ep"))
    B = len(apm)

    def sample(r):
        ne = B * r.mean() ** 2 / (r * r).mean()
        return ne, stats.t.ppf(1 - 0.00125, int(ne) - 1)
    r = np.clip(apm / bpm, 0.1, 10)
    ne, cv = sample(r)
    cips = (np.mean(offs * r), cv * np.std(offs * r) / np.sqrt(int(ne)))
    d = np.average(q, 1) + r * (offs - ep)
    dr = (d.mean() / offs.mean(), stats.sem(d))
    ws = np.clip(np.cumprod(np.clip(pol / beh, 0.1, 10), 1) / B, 0.1, 10)
    w = np.cumsum(ws, 1) / np.arange(1, ws.shape[1] + 1)
    wips = ((ws / w * off).sum() / max(off.sum(), 1e-8), 0)
    acc = np.zeros(B)
    for t in range(ws.shape[1] - 1, -1, -1):
        acc = q[:, t] + ws[:, t] * (off[:, t] + acc - hat[:, t])
    return {"CIPS": cips, "DR": dr, "WIPS": wips, "SeqDR": (acc.mean() / off.sum(1).mean(), 0)}


def test_estimators_match_a_float64_restatement():
    rs = np.random.RandomState(3)
    for B, T in ((7, 9), (2048, 36), (5, 1)):
        x = {"pol": rs.uniform(0.005, 0.02, (B, T)), "beh": rs.uniform(0.005, 0.02, (B, T)), "off": rs.uniform(0, 5, (B, T)),
             "hat": rs.uniform(0, 5, (B, T)), "q": rs.uniform(-1, 8, (B, T))}
        x["apm"], x["bpm"] = np.prod(x["pol"] * 100, 1), np.prod(x["beh"] * 100, 1)
        x["apm"] *= rs.choice([0.05, 1.0, 20.0], B)              # ratios on both sides of the clip
        x["offs"], x["ep"] = x["off"].sum(1), x["hat"].sum(1)
        want = _f64_restatement(x)
        got = {k: f() for k, f in mk.metric_calls(vars(OPE), x).items()}
        for k, v in want.items():
            np.testing.assert_allclose(np.asarray(got[k], np.float64), np.asarray(v, np.float64), rtol=1e-12, atol=1e-300,
                                       err_msg="%s B=%d T=%d" % (k, B, T))


def test_episode_products_are_numpys_float32_products_bit_for_bit():
    rs = np.random.RandomState(4)
    buf = rs.uniform(0.001, 0.03, (36, 2048)).astype(np.float32)           # [T, B] as the buffers hold them
    ref = np.multiply.reduce(np.array(list(buf)).swapaxes(0, 1) * 100, axis=1)
    got = oe.episode_products(buf.swapaxes(0, 1))
    assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    seq = np.ones(2048, np.float32)
    for t in range(36):
        seq = seq * (buf[t] * np.float32(100))
    assert np.array_equal(got.view(np.uint32), seq.view(np.uint32))


def test_ope_eval_flow_replays_the_reference():
    """ope_eval with the flow recorders (the env, policy and behaviour model of make_ope_golden) prints and returns what
    the reference's script computed from the same arrays, and calls the behaviour model with the same layers and pages."""
    z = _golden("ope_flow.npz")
    arr = {k: z[k] for k in ("probs", "actions", "off_action", "q", "beh", "reward", "off_reward")}
    env = mk.FlowEnv(arr)
    E, T, B = arr["probs"].shape[:3]
    sm = mk.FlowBehavior(env)
    saved = oe.policy_model
    oe.policy_model = lambda algo, config: mk.FlowPolicy(env)
    try:
        out = io.StringIO()
        with redirect_stdout(out):
            m = oe.ope_eval({"epoch": E, "batch_size": B, "max_steps": T, "page_items": 4}, env, None, sample_model=sm)
    finally:
        oe.policy_model = saved
    text = out.getvalue()
    assert "IS DR WIPS SeqDR" in text and text.count("test batch at ") == E
    assert m.shape == (E, 4, 2)
    np.testing.assert_allclose(m.mean(0), z["printed_avg"], rtol=1e-12)
    np.testing.assert_allclose(m.std(0), z["printed_std"], rtol=1e-12, atol=1e-15)
    assert np.array_equal(np.array(sm.calls), z["calls"])
    assert np.array_equal(np.array(env.taken), z["taken"])
    assert str(np.average(m, axis=0)) in text


def _npz(tmp_path, w, name="w.npz"):
    p = str(tmp_path / name)
    np.savez(p, **w)
    return p


def _bm(path, **kw):
    return oe.behavior_model({"action_size": 284, "page_items": 9}, path, device="cpu", **kw)


def test_twin_behavior_model_matches_the_reference():
    """The torch twin against behavior_model.py over the numpy dnn: 1e-5 relative (float32 products summed in another
    order, then exp and two divisions)."""
    import tempfile
    import pathlib
    z = _golden("ope_behavior.npz")
    with tempfile.TemporaryDirectory() as d:
        bm = _bm(_npz(pathlib.Path(d), mk.dnn_weights()))
    n = 0
    for kind, pages in (("slate", 1), ("seqslate", 4)):
        recs = list(z[kind + "/records"])
        for page in range(pages):
            for layer in range(1, 13):
                a = z["%s/%d/%d/action" % (kind, page, layer)]
                got = bm.action_probs(recs, a, layer, page=page)
                assert got.dtype == np.float32
                np.testing.assert_allclose(got, z["%s/%d/%d/probs" % (kind, page, layer)], rtol=1e-5, atol=1e-9)
                n += 1
            edges = np.stack([bm.action_probs(recs, np.full(len(recs), a), layer, page=page)
                              for layer in (1, 2, 3) for a in mk.EDGE_ACTIONS])
            np.testing.assert_allclose(edges, z["%s/%d/edges" % (kind, page)], rtol=1e-5, atol=1e-9)
    assert n == 12 * 5
    assert len(bm._pages) == 4                      # one forward per page of the last reset


def test_weights_load_from_npz_and_tf1_checkpoint_and_refuse_other_graphs(tmp_path):
    from rl4rs_b200.utils import tf_checkpoint
    w = mk.dnn_weights()
    a = _bm(_npz(tmp_path, w))
    prefix = str(tmp_path / "ckpt")
    tf_checkpoint.save_dnn_checkpoint(prefix, w, dict(oe.DNN_CFG, category_hash_size=mk.H, class_num=mk.C))
    b = _bm(prefix)
    assert (a.H, a.C) == (b.H, b.C) == (mk.H, mk.C)
    assert np.array_equal(a.flat.numpy(), b.flat.numpy())
    # another graph: a widedeep checkpoint, an .npz with a missing or a reshaped table
    wd = {"emb_cat": w["emb_cat"], "dense_w1": np.zeros((432, 128), np.float32), "rew_w": np.zeros((3072, 2), np.float32)}
    tf_checkpoint.save_widedeep_checkpoint(str(tmp_path / "wd"), wd)
    with pytest.raises(KeyError):
        _bm(str(tmp_path / "wd"))
    with pytest.raises(KeyError, match="fc_w"):
        _bm(_npz(tmp_path, {k: v for k, v in w.items() if k != "fc_w"}, "m.npz"))
    with pytest.raises(ValueError, match="dense_w1"):
        _bm(_npz(tmp_path, dict(w, dense_w1=np.zeros((432, 128), np.float32)), "s.npz"))
    with pytest.raises(ValueError, match="fewer than action_size"):
        oe.behavior_model({"action_size": 300}, _npz(tmp_path, w, "c.npz"), device="cpu")
    try:
        import h5py  # noqa: F401
    except ImportError:
        with pytest.raises(ImportError, match="npz"):
            _bm(str(tmp_path / "logged_policy.h5"))


def test_row_index_records_and_continuous_policies_raise(tmp_path):
    bm = _bm(_npz(tmp_path, mk.dnn_weights()))
    with pytest.raises(ValueError, match="record strings"):
        bm.action_probs(np.arange(4), np.zeros(4, int), 1)
    with pytest.raises(NotImplementedError, match="continuous"):
        oe.ope_eval({"epoch": 1, "batch_size": 2, "max_steps": 9, "support_conti_env": True}, None,
                    types.SimpleNamespace(continuous=True, reward_scaler=None))
    from rl4rs_b200 import batchrl
    with pytest.raises(NotImplementedError, match="ope"):
        batchrl.ope_eval()


def _fake_env(B=5, A=284, **cfg):
    return types.SimpleNamespace(config=dict({"max_steps": 9, "batch_size": B, "action_size": A}, **cfg))


def test_full_fetch_infos_are_rllibs_keys():
    import torch
    from rl4rs_b200 import trainer
    rs = np.random.RandomState(0)
    B, A = 5, 284
    obs = {"obs": rs.standard_normal((B, 256)).astype(np.float32), "action_mask": (rs.rand(B, A) < 0.5).astype(np.float32)}
    torch.manual_seed(0)
    ppo = trainer.get_rl_model("PPO", {}, _fake_env(support_rllib_mask=True), device="cpu")
    a, state, infos = ppo.compute_actions(obs, explore=False, full_fetch=True)
    assert state == [] and set(infos) == {"action_dist_inputs", "vf_preds", "action_logp", "action_prob"}
    assert infos["action_dist_inputs"].shape == (B, A) and infos["vf_preds"].shape == (B,)
    assert np.array_equal(a, ppo.compute_actions(obs, explore=False))
    assert np.array_equal(a, infos["action_dist_inputs"].argmax(1))
    rows = {i: {k: v[i] for k, v in obs.items()} for i in range(B)}
    d, _, infos2 = ppo.compute_actions(rows, explore=False, full_fetch=True)
    assert list(d.values()) == a.tolist() and np.array_equal(infos2["vf_preds"], infos["vf_preds"])
    rb = trainer.get_rl_model("RAINBOW", {}, _fake_env(), device="cpu")
    a, state, infos = rb.compute_actions(obs["obs"], explore=False, full_fetch=True)
    assert set(infos) == {"q_values", "action_dist_inputs"} and infos["q_values"].shape == (B, A)
    assert np.array_equal(a, infos["q_values"].argmax(1))
    # policy_model's RLlib branch: predict_q / action_probs through full_fetch
    from rl4rs_b200 import batchrl
    pm = batchrl.policy_model(ppo, {})
    act = pm.predict_with_mask(obs)
    assert np.array_equal(pm.predict_q(obs, act), infos2["vf_preds"])
    np.testing.assert_allclose(pm.action_probs(obs).sum(1), 1.0, rtol=1e-5)


def test_gather_refuses_inputs_whose_batch_is_not_batch_size():
    """The [T, B] buffers are sized from config['batch_size']; a step of another batch (or a mis-shaped input) must raise
    before any write, on every path (the kernel writes element t B + b for each of its rows)."""
    import torch
    B, A, T = 4, 284, 9
    bufs = oe.StepBuffers(T, B, "cpu", use_kernels=True)          # on the CPU the check runs ahead of the torch gather
    ok = dict(probs=torch.rand(B, A), logits=False, off=torch.zeros(B, dtype=torch.int32), beh=torch.rand(B, 283), layer=1,
              own=torch.zeros(B, dtype=torch.int32), values=torch.rand(B, A), reward=torch.rand(B, dtype=torch.float64),
              off_reward=torch.rand(B, dtype=torch.float64))
    bufs.gather(0, **ok)
    bad = [dict(probs=torch.rand(B + 1, A)), dict(probs=torch.rand(B - 1, A)), dict(off=torch.zeros(B + 1, dtype=torch.int32)),
           dict(beh=torch.rand(B + 1, 283)), dict(own=torch.zeros(B - 1, dtype=torch.int32)), dict(values=torch.rand(B, A + 1)),
           dict(values=torch.rand(B)), dict(reward=torch.rand(B + 1, dtype=torch.float64)),
           dict(off_reward=torch.rand(B - 1, dtype=torch.float64))]
    for b in bad:
        with pytest.raises(ValueError):
            bufs.gather(1, **dict(ok, **b))
    with pytest.raises(ValueError):
        bufs.gather(T, **ok)
    # through ope_eval: the flow env's batch is 6, the config says 7
    z = _golden("ope_flow.npz")
    arr = {k: z[k] for k in ("probs", "actions", "off_action", "q", "beh", "reward", "off_reward")}
    env = mk.FlowEnv(arr)
    E, T, B = arr["probs"].shape[:3]
    saved = oe.policy_model
    oe.policy_model = lambda algo, config: mk.FlowPolicy(env)
    try:
        with redirect_stdout(io.StringIO()), pytest.raises(ValueError, match="batch_size"):
            oe.ope_eval({"epoch": E, "batch_size": B + 1, "max_steps": T, "page_items": 4}, env, None,
                        sample_model=mk.FlowBehavior(env))
    finally:
        oe.policy_model = saved


def test_action_probs_refuses_an_action_beyond_the_classes(tmp_path):
    """Layer 3 reads y[:, 148:] at clip(a - 148, 0, 233): with C = 284 an action of 284 or more lands past the slice, where
    the reference raises IndexError; so does the model, checked on the host before it indexes the block."""
    bm = _bm(_npz(tmp_path, mk.dnn_weights()))
    recs = list(_golden("ope_behavior.npz")["slate/records"])
    a = np.full(len(recs), 283)
    bm.action_probs(recs, a, 3)
    bm.action_probs(recs, a + 1000, 1)                         # layers 1 and 2 clip into their slices
    with pytest.raises(IndexError):
        bm.action_probs(recs, a + 1, 3)
    with pytest.raises(ValueError):
        bm.action_probs(recs, a[:-1], 1)


def test_ope_fetch_equals_the_three_calls_of_the_reference_surface():
    """policy_model._ope_fetch, the one act ope_eval makes per step, gives what predict_with_mask, action_probs and
    predict_q give: batch-RL models (CQL with its reward scaler undone by the value fix) and a PPO trainer."""
    import torch
    from scipy.special import softmax
    from rl4rs_b200 import batchrl, trainer
    from test_batchrl_cpu import _cfg, synthetic_dataset
    obs = synthetic_dataset(266, 4, 9, seed=5)["observations"]
    rows = np.arange(len(obs))
    for algo in ("BC", "BCQ", "CQL"):
        m = batchrl.get_model(_cfg(), algo)
        m.create_impl(266)
        if algo == "CQL":
            m.reward_scaler, m.reward_mean, m.reward_std = "standard", 0.3, 1.7
        pm = batchrl.policy_model(m, _cfg())
        env_a, probs, logits, own, values, fix = pm._ope_fetch(obs)
        act = pm.predict_with_mask(obs)
        assert not logits and np.array_equal(env_a, act) and np.array_equal(own.long().numpy(), act)
        assert np.array_equal(probs.numpy(), pm.action_probs(obs))
        q = values.numpy()[rows, act]
        q = fix(q) if fix is not None else q
        assert (fix is not None) == (algo == "CQL")
        assert np.array_equal(q, pm.predict_q(obs, act))
    rs = np.random.RandomState(1)
    B, A = 5, 284
    o = {"obs": rs.standard_normal((B, 256)).astype(np.float32), "action_mask": (rs.rand(B, A) < 0.5).astype(np.float32)}
    torch.manual_seed(0)
    ppo = trainer.get_rl_model("PPO", {}, _fake_env(B, support_rllib_mask=True), device="cpu")
    pm = batchrl.policy_model(ppo, {})
    env_a, dist, logits, own, values, fix = pm._ope_fetch(o)
    act = pm.predict_with_mask(o)
    assert logits and own is None and fix is None and np.array_equal(env_a, act)
    np.testing.assert_array_equal(softmax(dist.numpy(), axis=1), pm.action_probs(o))
    assert np.array_equal(values.numpy(), pm.predict_q(o, act))
    # the gather's in-kernel softmax restated in torch against the reference's scipy softmax of the same logits
    bufs = oe.StepBuffers(1, B, "cpu", use_kernels=False)
    off = rs.randint(0, A, B)
    bufs.gather(0, dist, True, off, torch.rand(B, 283), 1, None, values, torch.zeros(B), torch.zeros(B))
    np.testing.assert_allclose(bufs.pol[0].numpy(), pm.action_probs(o)[rows[:B], off], rtol=4e-6)
