"""GPU: r4_finalize_weights checks a simulator's whole W-table before it frees or uploads anything, and its error names the
missing or mis-shaped tensor, for every kind of entry: a plain device buffer, a k_gemm_tc weight image, a GRU that is
re-laid for the recurrence kernel, and dien's per-sequence attention / AUGRU weights."""
import pytest

from test_gpu_parity_regimes import _cfg

pytestmark = pytest.mark.gpu

HASH = 1000          # small embedding tables: the check only compares element counts

# simulator -> (W-table maker in rl4rs_b200.synth, {kind of entry: one required tensor of that kind})
TABLES = {
    "dien": ("make_weights", {"plain": "obs_b", "image": "obs_w", "gru": "gru1_wc", "per_seq": "att1_k"}),
    "dnn": ("make_dnn_weights", {"plain": "fc_b", "image": "fc_w"}),
    "widedeep": ("make_widedeep_weights", {"plain": "emb_seq", "image": "dense_w1"}),
    "lstm": ("make_lstm_weights", {"plain": "rew_w", "image": "obs_w", "gru": "sgru1_rk"}),
}
MIS_SHAPED = {"dien": "augru0_wg", "dnn": "obs_w", "widedeep": "rew_w", "lstm": "cgru_b"}

_WEIGHTS = {}


def _weights(algo):
    from rl4rs_b200 import synth
    if algo not in _WEIGHTS:
        cfg = dict(_cfg(8, False), algo=algo, category_hash_size=HASH)
        _WEIGHTS[algo] = getattr(synth, TABLES[algo][0])(cfg)
    return dict(_WEIGHTS[algo])


def _engine(algo, weights):
    from rl4rs_b200 import synth
    from rl4rs_b200.engine import Engine
    cfg = dict(_cfg(8, False), algo=algo, category_hash_size=HASH)
    cat = synth.make_catalog()
    return Engine(cfg, False, cat, weights, synth.make_log(16, catalog=cat, hash_size=HASH))


def _assert_rejected(algo, weights, name):
    from rl4rs_b200 import _capi
    with pytest.raises(_capi.R4Error) as exc:
        _engine(algo, weights)
    assert str(exc.value).endswith("r4_finalize_weights(%s): missing or mis-shaped %s" % (algo, name)), str(exc.value)


@pytest.mark.parametrize("algo,kind", [(a, k) for a, (_, kinds) in TABLES.items() for k in kinds])
def test_missing_weight_is_named(algo, kind):
    name = TABLES[algo][1][kind]
    w = _weights(algo)
    del w[name]
    _assert_rejected(algo, w, name)


@pytest.mark.parametrize("algo", sorted(MIS_SHAPED))
def test_mis_shaped_weight_is_named(algo):
    name = MIS_SHAPED[algo]
    w = _weights(algo)
    w[name] = w[name][:-1]                   # one row (or one bias element) short
    _assert_rejected(algo, w, name)
