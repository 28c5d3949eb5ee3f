"""GPU: the `dnn` simulator (config['algo'] = 'dnn'; rl4rs/env/slate.py:239-242 -> rl4rs/nets/dnn.py:8-45) through the
same env API against the CPU oracle (oracle/dnn_np.py): the gather kernel k_cat_pool (bulk-TMA staged embedding rows),
the dense tower and the two 256-wide FC layers on wgmma, reward / violation / masks unchanged."""
import numpy as np
import pytest

from golden_util import assert_close_rel
from test_gpu_parity import make_env
from test_gpu_parity_regimes import _cfg, _sublog

pytestmark = pytest.mark.gpu


def _dnn_setup(B, seq, hash_size=100000, stress=1.0, bias_noise=0.0, n_log=None, **flags):
    from rl4rs_b200 import synth
    cfg = dict(_cfg(B, seq, **flags), algo="dnn", category_hash_size=hash_size)
    cat = synth.make_catalog()
    log = synth.make_log(n_log or 4 * B, pages=4 if seq else 1, catalog=cat, hash_size=hash_size, corrupt_frac=0.1)
    return cfg, cat, log, synth.make_dnn_weights(cfg, stress=stress, bias_noise=bias_noise)


@pytest.mark.parametrize("regime", ["default", "stress"])
def test_dnn_forward_alone_matches_oracle(regime):
    from oracle.dnn_np import DnnOracle
    # stress 2: at 3 the reward logits reach |z| ~ 340 and even the f32 oracle misses the f64 one on probs (ill-conditioned)
    kw = {} if regime == "default" else {"stress": 2.0, "bias_noise": 0.1}
    cfg, cat, log, w = _dnn_setup(8, False, **kw)
    env = make_env(cfg, False, cat, log, w, output_format="numpy")
    rs = np.random.RandomState(4)
    R = 1000                                                  # ragged against the 4-row CTAs and 128-row GEMM tiles
    seq = np.zeros((R, 2, 64), np.int32)
    dense = rs.normal(0, 2, (R, 432)).astype(np.float32)
    catf = rs.randint(0, 100000, (R, 21)).astype(np.int32)
    obs, probs = env.sim.engine.dien_forward(seq, dense, catf)
    o_ref, p_ref = DnnOracle(w, np.float32).forward(seq, dense, catf)
    assert_close_rel(obs.cpu().numpy(), o_ref, what="dnn obs [%s]" % regime)
    assert_close_rel(probs.cpu().numpy(), p_ref, what="dnn probs [%s]" % regime)
    o64, _ = DnnOracle(w, np.float64).forward(seq, dense, catf)
    assert_close_rel(obs.cpu().numpy(), o64, what="dnn obs vs f64 [%s]" % regime)


@pytest.mark.parametrize("seq", [False, True])
def test_dnn_env_matches_oracle(seq):
    from oracle.dnn_np import DnnOracle
    from oracle.env_np import OracleEnv
    B = 48
    # default-scale kernels + bias noise: with the x2 "stress" kernels the reward logits reach |z| ~ 50 and the click
    # probabilities inherit a relative error of ~|z| x the f32 rounding of the observation (1.7e-4 on the summed reward --
    # the f32 and f64 oracles differ by as much); the numerics of the stressed net are covered by the forward-alone test
    cfg, cat, log, w = _dnn_setup(B, seq, stress=1.0, bias_noise=0.1, support_rllib_mask=True, simulator_info_fetch=True)
    env = make_env(cfg, seq, cat, log, w, output_format="numpy")
    ref = OracleEnv(cfg, log, cat, DnnOracle(w, np.float32), seq=seq)
    rs = np.random.RandomState(5)
    for ep in range(2):
        o, r = env.reset(), ref.reset()
        assert_close_rel(o["obs"], r["obs"], what="dnn env reset obs")
        np.testing.assert_array_equal(o["action_mask"], r["action_mask"])
        paid = 0
        for t in range(cfg["max_steps"]):
            a = np.where(rs.rand(B) < 0.8, ref.offline_action, rs.randint(0, 284, B))
            o, rew, done, info = env.step(a)
            r, rrew, rdone, _ = ref.step(a)
            np.testing.assert_array_equal(o["action_mask"], r["action_mask"], err_msg="mask %d" % t)
            np.testing.assert_array_equal(done, rdone)
            np.testing.assert_array_equal(env.samples.get_violation(), ref.samples.get_violation())
            assert_close_rel(o["obs"], r["obs"], what="dnn env obs step %d" % t)
            assert_close_rel(rew, rrew, what="dnn env reward step %d" % t)
            paid += int((np.asarray(rrew) != 0).any())
        assert paid >= 1          # (SeqSlate: one early violation zeroes every later page, so only the first pages pay)


def test_dnn_big_batch_oracle_sample():
    """B = 16 384 rows (default weights): 128 rows replayed through the oracle, rows compared by index."""
    from oracle.dnn_np import DnnOracle
    from oracle.env_np import OracleEnv
    B = 16384
    cfg, cat, log, w = _dnn_setup(B, False, n_log=B, support_rllib_mask=True)
    env = make_env(cfg, False, cat, log, w, output_format="numpy")
    rs = np.random.RandomState(6)
    idx = np.sort(rs.choice(B, 128, replace=False))
    ref = OracleEnv(dict(cfg, batch_size=128, cache_size=128), _sublog(log, idx), cat, DnnOracle(w, np.float32))
    o, r = env.reset(reset_file=True), ref.reset(reset_file=True)
    assert_close_rel(o["obs"][idx], r["obs"], what="dnn B=16384 sample reset obs")
    for t in range(9):
        a = np.asarray(env.offline_action)
        o, rew, done, _ = env.step(a)
        r, rrew, rdone, _ = ref.step(a[idx])
        np.testing.assert_array_equal(o["action_mask"][idx], r["action_mask"])
        assert_close_rel(o["obs"][idx], r["obs"], what="dnn B=16384 sample obs step %d" % t)
        assert_close_rel(np.asarray(rew)[idx], rrew, what="dnn B=16384 sample reward step %d" % t)


# ---- widedeep (config['algo'] = 'widedeep'; rl4rs/nets/widedeep.py:8-45): 'simulator_obs' is the 3072-wide concat --------
def _wd_setup(B, seq, stress=1.0, bias_noise=0.0, **flags):
    from rl4rs_b200 import synth
    cfg = dict(_cfg(B, seq, **flags), algo="widedeep")
    cat = synth.make_catalog()
    log = synth.make_log(4 * B, pages=4 if seq else 1, catalog=cat, hash_size=100000, corrupt_frac=0.1)
    return cfg, cat, log, synth.make_widedeep_weights(cfg, stress=stress, bias_noise=bias_noise)


def test_widedeep_forward_alone_matches_oracle():
    from oracle.widedeep_np import WideDeepOracle
    from test_gpu_parity_regimes import _random_feature_rows
    cfg, cat, log, w = _wd_setup(8, False, stress=2.0, bias_noise=0.1)
    env = make_env(cfg, False, cat, log, w, output_format="numpy")
    seq, dense, catf = _random_feature_rows(700, 8, 100000)
    obs, probs = env.sim.engine.dien_forward(seq, dense, catf)
    o_ref, p_ref = WideDeepOracle(w, np.float32).forward(seq, dense, catf)
    assert obs.shape == (700, 3072)
    np.testing.assert_array_equal(obs.cpu().numpy()[:, 384:], o_ref[:, 384:])          # the Flatten() half is a pure gather
    assert_close_rel(obs.cpu().numpy()[:, :384], o_ref[:, :384], what="widedeep obs (dense halves)")
    assert_close_rel(probs.cpu().numpy(), p_ref, what="widedeep probs")


@pytest.mark.parametrize("seq", [False, True])
def test_widedeep_env_matches_oracle(seq):
    from oracle.widedeep_np import WideDeepOracle
    from oracle.env_np import OracleEnv
    B = 40
    cfg, cat, log, w = _wd_setup(B, seq, stress=1.0, bias_noise=0.1, support_rllib_mask=True)
    env = make_env(cfg, seq, cat, log, w, output_format="numpy")
    assert env.observation_space["obs"].shape == (3072,)
    ref = OracleEnv(cfg, log, cat, WideDeepOracle(w, np.float32), seq=seq)
    rs = np.random.RandomState(7)
    o, r = env.reset(), ref.reset()
    assert_close_rel(o["obs"][:, :384], r["obs"][:, :384], what="widedeep env reset obs")
    paid = 0
    for t in range(cfg["max_steps"]):
        a = np.where(rs.rand(B) < 0.85, ref.offline_action, rs.randint(0, 284, B))
        o, rew, done, info = env.step(a)
        r, rrew, rdone, _ = ref.step(a)
        np.testing.assert_array_equal(o["action_mask"], r["action_mask"], err_msg="mask %d" % t)
        np.testing.assert_array_equal(o["obs"][:, 384:], r["obs"][:, 384:], err_msg="flatten half %d" % t)
        assert_close_rel(o["obs"][:, :384], r["obs"][:, :384], what="widedeep env obs step %d" % t)
        assert_close_rel(rew, rrew, what="widedeep env reward step %d" % t)
        paid += int((np.asarray(rrew) != 0).any())
    assert paid >= 1


# ---- lstm (config['algo'] = 'lstm'; rl4rs/nets/lstm.py:8-45): Keras GRUs over both sequences and over the category embeddings ----
def _lstm_setup(B, seq, stress=1.0, bias_noise=0.0, gru=(2.5, 1.5), **flags):
    from rl4rs_b200 import synth
    cfg = dict(_cfg(B, seq, **flags), algo="lstm")
    cat = synth.make_catalog()
    log = synth.make_log(4 * B, pages=4 if seq else 1, catalog=cat, hash_size=100000, corrupt_frac=0.1)
    # gru = (kernel scale, bias sigma): ~25 % of the hard-sigmoid gates clip (synth.make_lstm_weights)
    return cfg, cat, log, synth.make_lstm_weights(cfg, stress=stress, bias_noise=bias_noise, gru_stress=gru[0], gru_bias_noise=gru[1])


@pytest.mark.parametrize("n_rows,gru", [(300, (2.5, 1.5)), (700, (1.0, None))])
def test_lstm_forward_alone_matches_oracle(n_rows, gru):
    from oracle.lstm_np import LstmOracle
    from test_gpu_parity_regimes import _random_feature_rows
    cfg, cat, log, w = _lstm_setup(8, False, stress=1.5, bias_noise=0.1, gru=gru)
    env = make_env(cfg, False, cat, log, w, output_format="numpy")
    seq, dense, catf = _random_feature_rows(n_rows, 8, 100000)
    obs, probs = env.sim.engine.dien_forward(seq, dense, catf)
    o_ref, p_ref = LstmOracle(w, np.float32).forward(seq, dense, catf)
    o64, p64 = LstmOracle(w, np.float64).forward(seq, dense, catf)
    assert obs.shape == (n_rows, 256)
    assert_close_rel(obs.cpu().numpy(), o_ref, what="lstm obs")
    assert_close_rel(obs.cpu().numpy(), o64, what="lstm obs vs f64")
    assert_close_rel(probs.cpu().numpy(), p_ref, what="lstm probs")


@pytest.mark.parametrize("seq", [False, True])
def test_lstm_env_matches_oracle(seq):
    from oracle.lstm_np import LstmOracle
    from oracle.env_np import OracleEnv
    B = 40
    cfg, cat, log, w = _lstm_setup(B, seq, stress=1.5, bias_noise=0.1, support_rllib_mask=True)
    env = make_env(cfg, seq, cat, log, w, output_format="numpy")
    assert env.observation_space["obs"].shape == (256,)
    ref = OracleEnv(cfg, log, cat, LstmOracle(w, np.float32), seq=seq)
    rs = np.random.RandomState(11)
    o, r = env.reset(), ref.reset()
    assert_close_rel(o["obs"], r["obs"], what="lstm env reset obs")
    paid = 0
    for t in range(cfg["max_steps"]):
        a = np.where(rs.rand(B) < 0.85, ref.offline_action, rs.randint(0, 284, B))
        o, rew, done, info = env.step(a)
        r, rrew, rdone, _ = ref.step(a)
        np.testing.assert_array_equal(o["action_mask"], r["action_mask"], err_msg="mask %d" % t)
        assert_close_rel(o["obs"], r["obs"], what="lstm env obs step %d" % t)
        assert_close_rel(rew, rrew, what="lstm env reward step %d" % t)
        np.testing.assert_array_equal(done, rdone)
        paid += int((np.asarray(rrew) != 0).any())
    assert paid >= 1
