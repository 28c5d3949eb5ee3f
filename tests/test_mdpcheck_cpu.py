"""CPU: the MDP checker (rl4rs_b200/mdpchecker) against the reference's own code -- preprocess.py's rl4rs branch,
mdp_checker.py's data preparation and decoder.py's searches, each run under stand-ins for the packages it imports and
stored under tests/golden/reference/ -- and the torch twin's pieces against NumPy float64 restatements."""
import os
import random
import sys
import tempfile
import types

import numpy as np
import pytest
import torch

from rl4rs_b200 import synth
from rl4rs_b200.mdpchecker import decoder as dc
from rl4rs_b200.mdpchecker import mdp_checker, preprocess
from rl4rs_b200.mdpchecker import transformer as tf

from golden_util import reference_result


def _ref_path(*p):
    from oracle import ref_harness
    return os.path.join(ref_harness.REFERENCE_ROOT, *p)


def _records(d):
    cat = synth.make_catalog()
    log = synth.make_log(60, pages=4, catalog=cat, hash_size=5000, keep_hist=True)
    with open(os.path.join(d, "rl4rs_dataset_a.csv"), "w") as f:
        f.write("\n".join(synth.render_records(log, cat)) + "\n")


def test_preprocess_rl4rs_matches_reference():
    with tempfile.TemporaryDirectory() as d:
        _records(d)
        preprocess.preprocess("rl4rs", d, print_fn=lambda *a: None)
        ours = open(os.path.join(d, "rl4rs.csv")).read()

        def compute():
            with tempfile.TemporaryDirectory() as d2:
                _records(d2)
                saved = sys.argv, dict(sys.modules)
                sys.modules["pandas"] = types.ModuleType("pandas")
                ps = types.ModuleType("pandasql")
                ps.sqldf = lambda q, g: None
                sys.modules["pandasql"] = ps
                sys.argv = ["preprocess.py", "rl4rs", d2]
                try:
                    src = open(_ref_path("script", "mdpchecker", "preprocess.py")).read()
                    exec(compile(src, "preprocess.py", "exec"), {"__name__": "__main__", "print": lambda *a: None})
                finally:
                    sys.argv = saved[0]
                    sys.modules.clear()
                    sys.modules.update(saved[1])
                return {"text": open(os.path.join(d2, "rl4rs.csv")).read()}
        assert ours == reference_result("mdpcheck_preprocess_rl4rs", compute)["text"]
    with pytest.raises(NotImplementedError, match="movielens"):
        preprocess.preprocess("movielens", "/nonexistent")


def _sessions(d, name, seed):
    rs = np.random.RandomState(seed)
    lines = ["sessionid items"]
    for s in range(80):
        k = rs.randint(3, 60)
        lines.append("%d %s" % (s, ",".join(str(x) for x in rs.randint(1, 40, k))))
    with open(os.path.join(d, name + ".csv"), "w") as f:
        f.write("\n".join(lines) + "\n")


@pytest.mark.parametrize("name", ["rl4rs", "cikm2016", "recsys15", "movielens"])
def test_data_preparation_matches_reference(name):
    with tempfile.TemporaryDirectory() as d:
        _sessions(d, name, seed=len(name))
        enc, dec, out, sdict, tdict, tl = mdp_checker.prepare(name + ".csv", d, print_fn=lambda *a: None)
        random.seed(1)
        sample = random.sample(enc[-30:], 16)

        def compute():
            with tempfile.TemporaryDirectory() as d2:
                _sessions(d2, name, seed=len(name))
                src = open(_ref_path("script", "mdpchecker", "mdp_checker.py")).read()
                src = src[:src.index("# Build & fit model")]
                kt = types.ModuleType("keras_transformer")
                kt.get_model = kt.decode = None
                dec_mod = types.ModuleType("rl4rs.mdpchecker.decoder")
                dec_mod.beam_search = dec_mod.token_probs = None
                saved = sys.argv, dict(sys.modules)
                sys.modules.update({"keras_transformer": kt, "rl4rs": types.ModuleType("rl4rs"),
                                    "rl4rs.mdpchecker": types.ModuleType("rl4rs.mdpchecker"),
                                    "rl4rs.mdpchecker.decoder": dec_mod})
                sys.argv = ["mdp_checker.py", name, d2]
                g = {"__name__": "__main__", "print": lambda *a: None}
                try:
                    exec(compile(src, "mdp_checker.py", "exec"), g)
                finally:
                    sys.argv = saved[0]
                    sys.modules.clear()
                    sys.modules.update(saved[1])
                random.seed(1)
                return {"enc": np.array(g["encode_input"]), "dec": np.array(g["decode_input"]),
                        "out": np.array(g["decode_output"]), "sample": np.array(random.sample(g["encode_input"][-30:], 16)),
                        "dict": sorted(g["source_token_dict"].items()), "tl": g["target_len"]}
        r = reference_result("mdpcheck_prepare_" + name, compute)
        assert np.array_equal(np.array(enc), r["enc"]) and np.array_equal(np.array(dec), r["dec"])
        assert np.array_equal(np.array(out), r["out"]) and np.array_equal(np.array(sample), r["sample"])
        assert [list(x) for x in sorted(sdict.items())] == r["dict"] and sdict is tdict and tl == r["tl"]


# ---- twin pieces against NumPy float64 ---------------------------------------------------------------------------
def test_trig_position_embedding():
    T, E = 9, 64
    p = np.arange(T)[:, None]
    k = np.arange(E)[None, :] // 2 * 2
    ang = p / np.power(10000.0, k / E)
    want = np.where(np.arange(E) % 2 == 0, np.sin(ang), np.cos(ang))
    assert np.abs(tf.trig(T, E, torch.float64, "cpu").numpy() - want).max() < 1e-5


def _np_forward(w, cfg, enc, dec):
    def ln(z, g, b):
        mu = z.mean(-1, keepdims=True)
        return (z - mu) / np.sqrt(((z - mu) ** 2).mean(-1, keepdims=True) + 1e-14) * g + b

    def mha(name, xq, xkv, km, causal):
        p = lambda k: w["%s/%s_%s:0" % (name, name, k)]
        q, k, v = xq @ p("Wq") + p("bq"), xkv @ p("Wk") + p("bk"), xkv @ p("Wv") + p("bv")
        n, Tq, E = q.shape
        Tk, dh = k.shape[1], E // cfg.H
        out = np.zeros_like(q)
        for h in range(cfg.H):
            sl = slice(h * dh, (h + 1) * dh)
            s = q[:, :, sl] @ k[:, :, sl].transpose(0, 2, 1) / np.sqrt(dh)
            if causal:
                s = s - 10000.0 * (np.arange(Tk)[None, :] > np.arange(Tq)[:, None])
            s = s - 10000.0 * (1 - km[:, None, :])
            e = np.exp(s - s.max(-1, keepdims=True))
            out[:, :, sl] = (e / e.sum(-1, keepdims=True)) @ v[:, :, sl]
        return out @ p("Wo") + p("bo")

    def ffn(name, x):
        p = lambda k: w["%s/%s_%s:0" % (name, name, k)]
        return np.maximum(x @ p("W1") + p("b1"), 0) @ p("W2") + p("b2")

    def norm(name, z):
        return ln(z, w[name + "-Norm/gamma:0"], w[name + "-Norm/beta:0"])

    pe = lambda T: tf.trig(T, cfg.E, torch.float64, "cpu").numpy()
    x = w["Encoder-Token-Embedding/embeddings:0"][enc] + pe(enc.shape[1])
    a, f = "Encoder-1-MultiHeadSelfAttention", "Encoder-1-FeedForward"
    x = norm(a, x + mha(a, x, x, (enc != 0).astype(float), False))
    e = norm(f, x + ffn(f, x))
    emb = w["Decoder-Token-Embedding/embeddings:0"]
    x = emb[dec] + pe(dec.shape[1])
    a, q, f = "Decoder-1-MultiHeadSelfAttention", "Decoder-1-MultiHeadQueryAttention", "Decoder-1-FeedForward"
    x = norm(a, x + mha(a, x, x, (dec != 0).astype(float), True))
    x = norm(q, x + mha(q, x, e, (enc != 0).astype(float), False))
    x = norm(f, x + ffn(f, x))
    z = x @ emb.T + w["Output/bias:0"]
    z = np.exp(z - z.max(-1, keepdims=True))
    return z / z.sum(-1, keepdims=True)


def test_twin_forward_and_loss_against_numpy():
    m = tf.get_model([30, 33], 64, 1, 1, 4, 64, use_same_embed=False, device="cpu", seed=4)
    rs = np.random.RandomState(0)
    enc, dec, y = rs.randint(1, 30, (5, 7)), rs.randint(1, 33, (5, 4)), rs.randint(0, 33, (5, 4))
    enc[:, 5:] = 0
    dec[2, 2:] = 0
    w64 = {k: v.astype(np.float64) for k, v in m.weights().items()}
    want = _np_forward(w64, m.cfg, enc, dec)
    got = torch.softmax(tf.forward(tf.unflatten(m.flat.double(), m.cfg), m.cfg, torch.as_tensor(enc), torch.as_tensor(dec)),
                        -1).numpy()
    assert np.abs(got - want).max() < 1e-12
    q = np.clip(want, 1e-7, 1 - 1e-7)
    ce = np.log(q.sum(-1)) - np.log(np.take_along_axis(q, y[..., None], -1)[..., 0])
    mask = dec != 0
    lw = (ce * mask).sum() / mask.sum()
    lg = tf.loss_fn(tf.forward(tf.unflatten(m.flat.double(), m.cfg), m.cfg, torch.as_tensor(enc), torch.as_tensor(dec)),
                    torch.as_tensor(dec), torch.as_tensor(y))
    assert abs(float(lg) - lw) < 1e-12


# ---- searches against the reference's decoder.py ------------------------------------------------------------------
class _Stub(object):
    """A Keras-like model whose predict is the twin's (float32), for the reference's decoder.py."""
    def __init__(self, m):
        self.m = m

    def predict(self, x):
        return self.m.predict(x)


def _ref_decoder():
    bn = types.ModuleType("bottleneck")
    bn.argpartition = lambda a, k, axis=-1: np.argpartition(a, k, axis=axis)
    bn.partition = lambda a, k, axis=-1: np.partition(a, k, axis=axis)
    sys.modules["bottleneck"] = bn
    if not hasattr(np, "int"):
        np.int = int
    g = {"__name__": "ref_decoder", "print": lambda *a: None}
    exec(compile(open(_ref_path("rl4rs", "mdpchecker", "decoder.py")).read(), "decoder.py", "exec"), g)
    return g


def _search_model():
    m = tf.get_model([30, 33], 32, 1, 1, 1, 64, use_same_embed=False, device="cpu", seed=9)
    rs = np.random.RandomState(1)
    enc = rs.randint(3, 30, (12, 6))
    enc[:, 0] = 1
    return m, enc


@pytest.mark.parametrize("beam,cand", [(1, 0), (4, 0), (5, 6)])
def test_beam_search_matches_reference(beam, cand):
    m, enc = _search_model()
    path, score = dc.beam_search(m, enc, beam, 5, use_candidates=cand > 0, candidates_size=cand)

    def compute():
        g = _ref_decoder()
        p, s = g["beam_search"](_Stub(m), list(enc), beam, 5, use_candidates=cand > 0, candidates_size=cand)
        return {"path": np.asarray(p, np.int64), "score": np.asarray(s, np.float64)}
    r = reference_result("mdpcheck_beam_%d_%d" % (beam, cand), compute)
    same = (path == r["path"]).all(axis=(1, 2))
    # a row whose paths differ must be a near-tie: the same scores in another order, or tokens of equal probability
    tie = ~same & np.isclose(np.sort(score, 1), np.sort(r["score"], 1), rtol=1e-5).all(axis=1)
    assert (same | tie).all(), np.where(~(same | tie))[0]
    assert np.allclose(score[same], r["score"][same], rtol=1e-6)
    print("beam %d cand %d: %d near-tie rows of %d" % (beam, cand, int(tie.sum()), len(same)))
    assert path.shape == (12, beam, 6) and score.shape == (12, beam)


def test_decode_step_and_token_probs_shapes():
    m, enc = _search_model()
    dec = np.ones((12, 1), np.int64)
    st = dc.decode_step(m, enc, dec, beam_size=3)
    assert st.shape == (12, 3, 2) and st.dtype == np.float64
    assert (np.diff(st[..., 0], axis=1) <= 0).all()
    tp = dc.token_probs(m, enc, dec)
    assert tp.shape == (12, 33) and np.allclose(tp.sum(-1), 1, atol=1e-5)
    assert np.allclose(st[:, :, 0], np.sort(tp, axis=1)[:, ::-1][:, :3])


# ---- the Keras surface and learning ---------------------------------------------------------------------------------
def test_model_surface_and_weights_roundtrip(tmp_path):
    with pytest.raises(NotImplementedError, match="sgd"):
        tf.get_model(10, 32, 1, 1, 1, 32, device="cpu").compile("sgd", "sparse_categorical_crossentropy")
    with pytest.raises(NotImplementedError, match="mse"):
        tf.get_model(10, 32, 1, 1, 1, 32, device="cpu").compile("adam", "mse")
    for opt in ({"attention_activation": "relu"}, {"feed_forward_activation": "gelu"}, {"use_adapter": True},
                {"embed_weights": np.zeros((10, 32))}, {"trainable": False}):
        with pytest.raises(NotImplementedError, match=list(opt)[0]):
            tf.get_model(10, 32, 1, 1, 1, 32, device="cpu", **opt)
    m = tf.get_model([20, 22], 32, 1, 2, 2, 32, dropout_rate=0.1, use_same_embed=False, device="cpu")
    m.compile("adam", "sparse_categorical_crossentropy")
    rs = np.random.RandomState(0)
    enc, dec, y = rs.randint(1, 20, (40, 5)), rs.randint(1, 22, (40, 3)), rs.randint(0, 22, (40, 3, 1))
    m.fit([enc, dec], y, epochs=1, batch_size=16, verbose=0)
    m.save_weights(str(tmp_path / "w.npz"))
    with pytest.raises(ValueError, match="h5"):
        m.save_weights(str(tmp_path / "w.h5"))
    m2 = tf.get_model([20, 22], 32, 1, 2, 2, 32, dropout_rate=0.1, use_same_embed=False, device="cpu", seed=5)
    m2.load_weights(str(tmp_path / "w.npz"))
    assert np.array_equal(m.predict([enc, dec]), m2.predict([enc, dec]))
    assert "Decoder-2-MultiHeadQueryAttention/Decoder-2-MultiHeadQueryAttention_Wq:0" in np.load(tmp_path / "w.npz").files


def test_twin_learns_a_planted_continuation():
    rs = np.random.RandomState(0)
    n, V = 400, 20
    enc = rs.randint(3, V, (n, 4))
    enc[:, 0] = 1
    nxt = (enc[:, 3] * 3) % (V - 3) + 3
    dec = np.stack([np.ones(n, int), nxt], 1)
    y = np.stack([nxt, np.full(n, 2)], 1)
    torch.manual_seed(0)
    np.random.seed(0)
    m = tf.get_model(V, 32, 1, 1, 1, 64, device="cpu")
    m.compile("adam", "sparse_categorical_crossentropy")
    h = m.fit([enc, dec], y, epochs=60, batch_size=50, verbose=0)
    assert h.history["loss"][-1] < 0.3 * h.history["loss"][0]
    path, _ = dc.beam_search(m, enc[:50], 1, 1)
    assert (path[:, 0, 1] == nxt[:50]).mean() >= 0.9
