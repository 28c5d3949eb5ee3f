"""GPU: the CUDA env at the configurations r4_create admits beyond the one every other env test runs (action_size 284,
Slate 9, SeqSlate 27 / 36):

  stored scenarios   every random_scenario_NN and shape_scenario_NN (tests/test_oracle_vs_reference_random.py: records
                     made by the reference's own env) replayed through the CUDA library by the product's env classes
  sequence sims      dien / lstm / widedeep through the env at SeqSlate 81 (more than 64 previous items, Q9 over all nine
                     pages) and 9 (one page: the page cache is never rebuilt), Slate 3 and 11 (padded / truncated rows)
  kNN edges          the continuous env at action_size 149, 288 and 512 (first, tenth and sixteenth mask word), one-hot
                     at 512, r4_nearest_neighbor at 512
  hash edges         r4_dien_forward of each simulator at category_hash_size 149 and 2^24 + 8 (ids whose row offset
                     id * 128 no longer fits in an int32)
  past the log       an env longer than its log rows: offline_action / offline_reward raise where the reference does

Bars: integers, masks, features, violation, done and offline_* bit-exact; observations and rewards within
golden_util.assert_close_rel (1e-4 against max(|ref|, rms(row))) of the f32 oracle or record."""
import numpy as np
import pytest

from golden_util import assert_close_rel

pytestmark = pytest.mark.gpu

# the range r4_create admits (rl4rs_b200/csrc/r4_capi.cu): tests/test_capi_exports.py checks both sides of each edge
A_MIN, A_MAX = 149, 512               # action_size: layer 2 non-empty .. 16 mask words
SLATE_T_MIN, SLATE_T_MAX = 3, 11      # Slate max_steps: the four location_mask layers
SEQ_T_STEP = 9                        # SeqSlate max_steps: any multiple of page_items


def _cfg(B, A, seq, T, H=5000, **flags):
    cfg = {"maxlen": 64, "batch_size": B, "action_size": A, "class_num": 2, "dense_feature_num": 432,
           "category_feature_num": 21, "category_hash_size": H, "seq_num": 2, "emb_size": 128, "hidden_units": 128,
           "max_steps": T, "page_items": 9, "action_emb_size": 32, "is_eval": True, "cache_size": B}
    cfg.update(flags)
    return cfg


def _inputs(cfg, seq, n_log=None, pages=None, seed=None):
    """Catalog of action_size items, a log of ceil(T / 9) pages (or `pages`)."""
    from rl4rs_b200 import synth
    A, T = cfg["action_size"], cfg["max_steps"]
    cat = synth.make_catalog() if A == 284 else synth.make_catalog(n_items=A - 1)
    log = synth.make_log(n_log or 2 * cfg["batch_size"], pages=pages or -(-T // 9), catalog=cat,
                         hash_size=cfg["category_hash_size"], corrupt_frac=0.1, seed=seed or synth.LOG_SEED)
    return cat, log


# ---- the stored scenarios through the CUDA library -----------------------------------------------------------------------
def _stored(kind):
    from test_oracle_vs_reference_random import SHAPE_SCENARIOS
    return [(kind, i) for i in range(32 if kind == "random" else len(SHAPE_SCENARIOS))]


def _f64_rewards(cfg, seq, cat, log, w, episodes, np_seed, rec):
    """The record's rewards recomputed by the oracle env with the float64 dnn network, over the recorded actions."""
    from oracle.dnn_np import DnnOracle
    from oracle.env_np import OracleEnv
    if np_seed is not None:
        np.random.seed(np_seed)
    env = OracleEnv(dict(cfg), log, cat, DnnOracle(w, np.float64), seq=seq)
    out, k = [], 0
    for ep in range(episodes):
        env.reset()
        for t in range(cfg["max_steps"]):
            out.append(np.asarray(env.step(rec["action_in"][k])[1], dtype=np.float64))
            k += 1
    return np.stack(out)


@pytest.mark.parametrize("fmt", ["list", "numpy"])
@pytest.mark.parametrize("kind,idx", _stored("random") + _stored("shape"))
def test_stored_scenario_through_the_cuda_library(kind, idx, fmt):
    """The reference's record of one scenario, replayed through the product's env classes over the real Engine.
    The random scenarios run the dnn network at stress-2 weights, where the reward logits reach |z| ~ 50: a reward's
    relative error is then the absolute error of the logits, and the CUDA rewards miss the f32 record by up to 1.2e-4 and
    the float64 network by up to 1.75e-4 of the reward, element by element (the record misses float64 by 0.19 of the bar).
    There the rewards are held to the float64 network (the oracle env over the same rows and actions) with the bar the
    observations use, 1e-4 of max(|ref|, rms of the step's rewards).  The shape scenarios run stress-1 weights and are
    held to the record element by element.  Everything else is held to the record."""
    from rl4rs_b200.utils.datautil import FeatureUtil
    from test_host_layer_cpu import make_env, replay_through_host_layer
    from test_oracle_vs_reference_random import scenario
    cfg, seq, cat, records, w, episodes, np_seed, rec = scenario(kind, idx)
    log = FeatureUtil.parse_log(records, 64)
    if kind == "random":
        rec = dict(rec, reward=_f64_rewards(cfg, seq, cat, log, w, episodes, np_seed, rec))
    if np_seed is not None:
        np.random.seed(np_seed)
    env = make_env(dict(cfg), seq, cat, log, w, output_format=fmt)
    replay_through_host_layer(env, cfg, rec, episodes, "%s scenario %d (cuda, %s)" % (kind, idx, fmt), fmt,
                              floor_rewards=kind == "random")
    env.sim.engine.close()


# ---- the simulators that read sequences, at the lengths the dnn grid cannot exercise -------------------------------------
def _seq_sim(sim, cfg):
    from rl4rs_b200 import synth
    if sim == "dien":
        from oracle.dien_np import DienOracle
        return synth.make_weights(cfg, stress=2.0, bias_noise=0.1, bounded_scores=True), DienOracle
    if sim == "lstm":
        from oracle.lstm_np import LstmOracle
        return synth.make_lstm_weights(cfg, stress=1.5, bias_noise=0.1, gru_stress=2.5, gru_bias_noise=1.5), LstmOracle
    from oracle.widedeep_np import WideDeepOracle
    return synth.make_widedeep_weights(cfg, stress=1.0, bias_noise=0.1), WideDeepOracle


def _obs_close(sim, got, ref, what):
    if sim == "widedeep":             # the Flatten() half of widedeep's observation is a pure gather
        np.testing.assert_array_equal(got[:, 384:], ref[:, 384:], err_msg=what)
        got, ref = got[:, :384], ref[:, :384]
    assert_close_rel(got, ref, what=what)


@pytest.mark.parametrize("length", ["seqslate81", "seqslate9", "slate3", "slate11"])
@pytest.mark.parametrize("sim", ["dien", "lstm", "widedeep"])
def test_sequence_simulator_env_at_every_length(sim, length):
    """B = 33, rllib mask, info fetch, 80 % logged actions.  At SeqSlate 81 the second sequence of pages 8 and 9 holds the
    LAST 64 of 72 previous items (k_seq_ids / k_seq_rows); at SeqSlate 9 the page cache is never rebuilt.  A Slate of 11
    always violates (steps 9 and 10 may only hold item 0), so its reward pass is held to the oracle by click_p alone."""
    from test_gpu_parity import make_env
    from oracle.env_np import OracleEnv
    seq = length.startswith("seq")
    T = int(length[len("seqslate" if seq else "slate"):])
    B = 33
    cfg = _cfg(B, 284, seq, T, algo=sim, support_rllib_mask=True, simulator_info_fetch=True)
    cat, log = _inputs(cfg, seq)
    w, Oracle = _seq_sim(sim, cfg)
    env = make_env(dict(cfg), seq, cat, log, w, output_format="numpy")
    ref = OracleEnv(dict(cfg), log, cat, Oracle(w, np.float32), seq=seq)
    rs = np.random.RandomState(T)
    o, r = env.reset(), ref.reset()
    _obs_close(sim, o["obs"], r["obs"], "%s %s reset obs" % (sim, length))
    paid = 0
    for t in range(T):
        a = np.where(rs.rand(B) < 0.8, ref.offline_action, rs.randint(0, 284, B))
        o, rew, done, info = env.step(a)
        r, rrew, rdone, rinfo = ref.step(a)
        np.testing.assert_array_equal(env.samples.prev_actions, ref.samples.prev_actions, err_msg="prev_actions %d" % t)
        np.testing.assert_array_equal(o["action_mask"], r["action_mask"], err_msg="mask %d" % t)
        np.testing.assert_array_equal(done, rdone)
        np.testing.assert_array_equal(env.samples.get_violation(), ref.samples.get_violation(), err_msg="violation %d" % t)
        _obs_close(sim, o["obs"], r["obs"], "%s %s obs step %d" % (sim, length, t))
        assert_close_rel(rew, rrew, what="%s %s reward step %d" % (sim, length, t))
        pays = (t + 1) % 9 == 0 if seq else t == T - 1
        if pays:
            cp = np.stack([i["click_p"] for i in info]) if isinstance(info, list) else info["click_p"]
            assert_close_rel(cp, np.stack([i["click_p"] for i in rinfo]), what="%s %s click_p" % (sim, length))
        paid += int((np.asarray(rrew) != 0).any())
    seqs, dense, catf = ref.samples.features()
    if seq and T > 72:
        assert (seqs[:, 1] != 0).sum(1).max() == 64          # the cut to the last 64 previous items was exercised
    _obs_close(sim, o["obs"], Oracle(w, np.float64).obs_layer((seqs, dense, catf, None)), "%s %s obs vs f64" % (sim, length))
    assert paid >= 1 or length == "slate11"
    env.sim.engine.close()


# ---- masked kNN at the mask-word edges ----------------------------------------------------------------------------------
@pytest.mark.parametrize("A", [A_MIN, 288, A_MAX])
def test_knn_at_the_mask_word_edges(A):
    """The continuous env (dnn simulator) with f64 and f32 actions, all-zero rows (every score ties: the first allowed
    index wins) and logged embeddings.  At A = 149 layer 2 holds item 148 alone: once it is taken (or special-masked),
    every later layer-2 row is all-masked and resolves to item 0 (argmax over a row of -2^31, slate.py:186-191)."""
    from rl4rs_b200 import synth
    from oracle.dnn_np import DnnOracle
    from oracle.env_np import OracleEnv
    from test_gpu_parity import make_env
    B = 40
    cfg = _cfg(B, A, False, 9, algo="dnn", support_rllib_mask=True, support_conti_env=True)
    cat, log = _inputs(cfg, False)
    w = synth.make_dnn_weights(cfg, stress=1.0, bias_noise=0.1)
    env = make_env(dict(cfg), False, cat, log, w, output_format="numpy")
    ref = OracleEnv(dict(cfg), log, cat, DnnOracle(w, np.float32))
    rs = np.random.RandomState(A)
    o, r = env.reset(), ref.reset()
    np.testing.assert_array_equal(o["action_mask"], r["action_mask"])
    for t in range(9):
        a = rs.uniform(-1, 1, (B, 32))
        a[:4] = 0.0
        a[4:12] = ref.offline_action[4:12]
        a = a.astype(np.float32) if t % 2 else a
        o, rew, _, _ = env.step(a)
        r, rrew, _, _ = ref.step(a)
        np.testing.assert_array_equal(env.samples.prev_actions, ref.samples.prev_actions, err_msg="kNN A=%d step %d" % (A, t))
        np.testing.assert_array_equal(o["action_mask"], r["action_mask"], err_msg="mask A=%d step %d" % (A, t))
        assert_close_rel(o["obs"], r["obs"], what="kNN A%d obs step %d" % (A, t))
    assert_close_rel(rew, rrew, what="kNN A%d reward" % A)
    if A == A_MIN:
        assert (env.samples.prev_actions[:, 7:9] == 0).all()
    env.sim.engine.close()


def test_onehot_and_nearest_neighbor_at_512():
    """One-hot actions at A = 512 (a 512-wide embedding) through the masked kNN, and the unmasked r4_nearest_neighbor
    over the 512 32-wide action embeddings (zero rows included)."""
    from rl4rs_b200 import synth
    from oracle.dnn_np import DnnOracle
    from oracle.env_np import OracleEnv
    from test_gpu_parity import make_env
    B = 24
    cfg = _cfg(B, A_MAX, False, 9, algo="dnn", support_conti_env=True, support_onehot_action=True)
    cat, log = _inputs(cfg, False)
    w = synth.make_dnn_weights(cfg, stress=1.0, bias_noise=0.1)
    env = make_env(dict(cfg), False, cat, log, w, output_format="numpy")
    ref = OracleEnv(dict(cfg), log, cat, DnnOracle(w, np.float32))
    rs = np.random.RandomState(5)
    env.reset(); ref.reset()
    for t in range(9):
        a = rs.uniform(0, 1, (B, A_MAX))
        a[0] = 0.0
        env.step(a); ref.step(a)
        np.testing.assert_array_equal(env.samples.prev_actions, ref.samples.prev_actions, err_msg="one-hot step %d" % t)
    env.sim.engine.close()
    cfg = _cfg(B, A_MAX, False, 9, algo="dnn", support_conti_env=True)
    env = make_env(dict(cfg), False, cat, log, w, output_format="numpy")
    q = rs.uniform(-1, 1, (77, 32))
    q[0] = 0.0
    q[1] = env.samples.action_emb[A_MAX - 1]
    got = env.sim.engine.nearest_neighbor(q).cpu().numpy()
    np.testing.assert_array_equal(got, env.samples.get_nearest_neighbor(q, env.samples.action_emb))
    assert got[0] == 0
    env.sim.engine.close()


# ---- category / sequence ids at the hash edges, through r4_dien_forward --------------------------------------------------
HASH_BIG = (1 << 24) + 8


def _edge_rows(H, R, rs):
    """Feature rows whose ids sit at the edges of [0, H): at H = 2^24 + 8 the ids 2^24 - 1, 2^24, 2^24 + 7, whose
    row offsets id * 128 pass 2^31."""
    edges = np.array([0, 148] if H < (1 << 24) else [0, (1 << 24) - 1, 1 << 24, H - 1], np.int64)
    catf = np.where(rs.rand(R, 21) < 0.5, rs.choice(edges, (R, 21)), rs.randint(0, H, (R, 21)))
    seq = np.zeros((R, 2, 64), np.int64)
    n = rs.randint(0, 65, (R, 2))
    n[0] = 64
    ids = np.where(rs.rand(R, 2, 64) < 0.5, rs.choice(edges[1:], (R, 2, 64)), rs.randint(1, H, (R, 2, 64)))
    keep = np.arange(64)[None, None, :] >= (64 - n)[:, :, None]
    seq[keep] = ids[keep]
    dense = rs.normal(0, 2, (R, 432)).astype(np.float32)
    return seq, dense, catf


def _host_peak_gb():
    import resource
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2.0 ** 20


@pytest.mark.parametrize("H", [A_MIN, HASH_BIG])
@pytest.mark.parametrize("sim", ["dien", "dnn", "widedeep", "lstm"])
def test_simulator_forward_at_the_hash_edges(sim, H):
    """The embedding tables are built on the device, zero except the rows the batch reads, and handed to r4_load_weight
    as device pointers; the oracle runs over the tables compacted to those rows (ids renumbered in order, 0 stays 0).
    One env at a time: at H = 2^24 + 8 each table is 8.6 GB on the device and, staged by r4_load_weight, on the host."""
    import torch
    from rl4rs_b200 import synth
    from rl4rs_b200.engine import Engine
    from oracle.dnn_np import DnnOracle
    rs = np.random.RandomState(H % 1000)
    R = 96
    seq, dense, catf = _edge_rows(H, R, rs)
    ids = np.unique(np.concatenate([catf.ravel(), seq.ravel(), [0]]))
    assert ids[0] == 0
    A = 284 if H >= 284 else A_MIN
    cfg = _cfg(8, A, False, 9, H=H, algo=sim)
    small = dict(cfg, category_hash_size=len(ids))
    if sim == "dnn":
        w, Oracle = synth.make_dnn_weights(small, stress=2.0, bias_noise=0.1), DnnOracle
    else:
        w, Oracle = _seq_sim(sim, small)
    cat, log = _inputs(cfg, False, n_log=8)
    torch.cuda.synchronize()
    free0, total = torch.cuda.mem_get_info()
    dev_w = dict(w)
    idx = torch.from_numpy(ids).cuda()
    for name in ("emb_cat", "emb_seq"):
        if name in w:
            big = torch.zeros((H, 128), dtype=torch.float32, device="cuda")
            big[idx] = torch.from_numpy(np.asarray(w[name], np.float32)).cuda()
            dev_w[name] = big
    eng = Engine(dict(cfg), False, cat, dev_w, log)
    torch.cuda.synchronize()
    peak_dev = (free0 - torch.cuda.mem_get_info()[0]) / 2.0 ** 30
    del dev_w, big
    torch.cuda.empty_cache()
    obs, probs = eng.dien_forward(seq, dense, catf)
    obs, probs = obs.cpu().numpy(), probs.cpu().numpy()
    eng.close()
    print("\n[hash edges] %s H=%d: device memory in use after the weights were loaded %.1f GB (of %.0f), host peak RSS %.1f GB"
          % (sim, H, peak_dev, total / 2.0 ** 30, _host_peak_gb()))
    remap = lambda x: np.searchsorted(ids, x).astype(np.int32)
    o_ref, p_ref = Oracle(w, np.float32).forward(remap(seq), dense, remap(catf))
    _obs_close(sim, obs, o_ref, "hash edge %s H=%s obs" % (sim, "2^24+8" if H == HASH_BIG else H))
    assert_close_rel(probs, p_ref, what="hash edge %s H=%s probs" % (sim, "2^24+8" if H == HASH_BIG else H))


# ---- an env longer than its log -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("seq,T,pages", [(False, 11, 1), (True, 45, 4)])
def test_offline_policy_past_the_logged_slots_raises(seq, T, pages):
    """Slate 11 over 9-slot rows, SeqSlate 45 over 36-slot rows.  The reference raises where the log has no slot:
    offline_action at a step >= the logged slots (IndexError, slate.py:156) and the SeqSlate offline_reward at a page end
    past the log ((B, 9) x (B, 0), seqslate.py:77-85).  The CUDA env raises at exactly those calls (R4_ERR_STATE) and
    matches the oracle at every call before them, including offline_reward after the last Slate step (every logged slot)."""
    from rl4rs_b200 import synth, _capi
    from oracle.dnn_np import DnnOracle
    from oracle.env_np import OracleEnv
    from test_gpu_parity import make_env
    B = 6
    cfg = _cfg(B, 284, seq, T, algo="dnn", support_rllib_mask=True)
    cat, log = _inputs(cfg, seq, pages=pages)
    S = 9 * pages
    w = synth.make_dnn_weights(cfg, stress=1.0, bias_noise=0.1)
    env = make_env(dict(cfg), seq, cat, log, w, output_format="numpy")
    ref = OracleEnv(dict(cfg), log, cat, DnnOracle(w, np.float32), seq=seq)
    o, r = env.reset(), ref.reset()
    for t in range(T):
        if t < S:
            a = ref.offline_action
            np.testing.assert_array_equal(np.asarray(env.offline_action), a)
        else:
            with pytest.raises(IndexError):
                ref.offline_action
            with pytest.raises(_capi.R4Error, match="past the"):
                env.offline_action
            a = np.zeros(B, np.int64)
        o, rew, _, _ = env.step(a)
        r, rrew, _, _ = ref.step(a)
        np.testing.assert_array_equal(o["action_mask"], r["action_mask"])
        assert_close_rel(rew, rrew, what="past-the-log reward step %d" % t)
        if seq and (t + 1) % 9 == 0 and t + 1 > S:
            with pytest.raises(ValueError):
                ref.offline_reward
            with pytest.raises(_capi.R4Error, match="past the"):
                env.offline_reward
        else:
            assert_close_rel(np.asarray(env.offline_reward), ref.offline_reward, rtol=1e-12, what="past-the-log offline_reward")
    assert np.asarray(env.offline_action).tolist() == [0] * B          # cur_steps == max_steps: item 0, as the reference
    env.sim.engine.close()
