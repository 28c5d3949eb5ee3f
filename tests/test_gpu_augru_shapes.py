"""GPU: launch shapes of the wgmma recurrences (r4_recur.cuh) that no other test isolates.  A CTA holds 64 rows, split
by columns between two consumer warpgroups: row counts just below / above one and two tiles, a ragged multi-wave launch,
and the 21-step category GRU of the `lstm` simulator on a partial second tile."""
import numpy as np
import pytest

from golden_util import assert_close_rel
from test_gpu_parity import make_env
from test_gpu_parity_regimes import _default_regime, _random_feature_rows

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dien():
    cfg, cat, log, w = _default_regime(8, False)
    return make_env(cfg, False, cat, log, w, output_format="numpy"), w


@pytest.mark.parametrize("R", [1, 63, 65, 129, 4160])
def test_dien_forward_row_counts(dien, R):
    from oracle.dien_np import DienOracle
    env, w = dien
    seq, dense, catf = _random_feature_rows(R, 30 + R % 17, 100000)
    obs, probs = env.sim.engine.dien_forward(seq, dense, catf)
    obs, probs = obs.cpu().numpy(), probs.cpu().numpy()
    assert np.isfinite(obs).all()
    idx = np.arange(R) if R <= 129 else np.unique(np.concatenate([np.arange(0, R, 37), [R - 64, R - 1]]))
    o_ref, p_ref = DienOracle(w, np.float32).forward(seq[idx], dense[idx], catf[idx])
    assert_close_rel(obs[idx], o_ref, what="dien obs R=%d" % R)
    assert_close_rel(probs[idx], p_ref, what="dien probs R=%d" % R)


def test_dien_forward_repeats_bit_identical(dien):
    env, _ = dien
    seq, dense, catf = _random_feature_rows(4160, 5, 100000)
    outs = [env.sim.engine.dien_forward(seq, dense, catf)[0].cpu().numpy() for _ in range(3)]
    for o in outs[1:]:
        np.testing.assert_array_equal(o.view(np.uint32), outs[0].view(np.uint32))


def test_lstm_category_gru_65_rows():
    from oracle.lstm_np import LstmOracle
    from test_gpu_dnn import _lstm_setup
    cfg, cat, log, w = _lstm_setup(8, False, stress=1.5, bias_noise=0.1)
    env = make_env(cfg, False, cat, log, w, output_format="numpy")
    seq, dense, catf = _random_feature_rows(65, 11, 100000)
    obs, probs = env.sim.engine.dien_forward(seq, dense, catf)
    o_ref, p_ref = LstmOracle(w, np.float32).forward(seq, dense, catf)
    assert_close_rel(obs.cpu().numpy(), o_ref, what="lstm obs R=65")
    assert_close_rel(probs.cpu().numpy(), p_ref, what="lstm probs R=65")
