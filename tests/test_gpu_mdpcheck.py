"""GPU: the MDP checker's transformer kernels (r4_s2s_*) against the float64 autograd reference tests/mdpcheck_ref64.py,
tensor by tensor; training against the torch twin, reruns and the epoch call; predict and the beam searches against the
twin; the C-ABI's argument checks and launch counts; and main() end to end on a planted dataset."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from rl4rs_b200 import _capi
from rl4rs_b200.mdpchecker import decoder as dc
from rl4rs_b200.mdpchecker import transformer as tf

import mdpcheck_ref64 as ref

pytestmark = pytest.mark.gpu


def _data(n, Ts, Tt, V, seed, pad=True):
    rs = np.random.RandomState(seed)
    enc = rs.randint(3, V, (n, Ts))
    enc[:, 0] = 1
    dec = rs.randint(3, V, (n, Tt))
    dec[:, 0] = 1
    y = rs.randint(0, V, (n, Tt))
    if pad:
        for r in range(n):
            enc[r, rs.randint(1, Ts + 1):] = 0
            dec[r, rs.randint(1, Tt + 1):] = 0
    return enc, dec, y


def _model(V, E, H, F, Le, Ld, same, seed=0, rate=0.0):
    m = tf.get_model([V, V + 3] if not same else V, E, Le, Ld, H, F, dropout_rate=rate, use_same_embed=same, seed=seed,
                     device="cuda")
    with torch.no_grad():   # move LayerNorm and biases off their initial values
        g = torch.Generator(device="cuda").manual_seed(seed)
        for k, t in tf.unflatten(m.flat, m.cfg).items():
            if t.dim() == 1:
                t.add_(0.1 * torch.randn(t.shape, generator=g, device="cuda"))
    return m


GRID = [  # n, V, Ts, Tt, H, Le, Ld, same, rate
    (1, 4, 2, 2, 1, 1, 1, True, 0.0),
    (7, 286, 18, 7, 4, 2, 2, False, 0.1),
    (256, 5003, 18, 7, 1, 1, 1, False, 0.0),
    (257, 286, 64, 2, 4, 1, 2, True, 0.05),
    (256, 286, 2, 7, 1, 2, 1, False, 0.0),
]


def _kernel_grad(m, enc, dec, y, call):
    """(loss, gradient, the kernels' relu decisions per FeedForward) of one r4_s2s_grad call."""
    lib = _capi.load_library()
    c = m.cfg.c()
    n, Ts = enc.shape
    Tt = dec.shape[1]
    scr = torch.empty(lib.r4_s2s_scratch_size(C.byref(c), _capi.S2S_TRAIN, n, Ts, Tt, 1, 0) // 4 + 1, device="cuda")
    g = torch.empty_like(m.flat)
    loss = torch.empty(1, device="cuda")
    e32, d32, y32 = (torch.as_tensor(a.astype(np.int32), device="cuda") for a in (enc, dec, y))
    _capi.check(lib, None, lib.r4_s2s_grad(C.byref(c), _capi.ptr(m.flat), _capi.ptr(e32), _capi.ptr(d32), _capi.ptr(y32),
                                           n, Ts, Tt, m.seed, call, m.dropout_rate, _capi.ptr(g), _capi.ptr(loss),
                                           _capi.ptr(scr), _capi.stream(m.flat.device)), "r4_s2s_grad")
    offs = (C.c_int64 * (m.cfg.Le + m.cfg.Ld))()
    assert lib.r4_s2s_relu_offsets(C.byref(c), n, Ts, Tt, offs) == m.cfg.Le + m.cfg.Ld
    keep = []
    for k, o in enumerate(offs):
        T = Ts if k < m.cfg.Le else Tt
        h = scr[o // 4:o // 4 + n * T * m.cfg.F].view(n, T, m.cfg.F)
        keep.append((h > 0).double().cpu())
    return float(loss.item()), g, keep


@pytest.mark.parametrize("n,V,Ts,Tt,H,Le,Ld,same,rate", GRID)
def test_gradient_against_float64(n, V, Ts, Tt, H, Le, Ld, same, rate):
    m = _model(V, 64, H, 64, Le, Ld, same, seed=n, rate=rate)
    enc, dec, y = _data(n, Ts, Tt, m.cfg.Vt, seed=n)
    loss, g, keep = _kernel_grad(m, enc, dec, y, call=3)
    rloss, rg, probs = ref.grad64(m.flat, m.cfg, enc, dec, y, seed=m.seed, call=3, rate=rate, relu_keep=keep)
    edge = ref.clip_edge_rows(probs, dec)
    assert abs(loss - rloss) <= 1e-5 * max(1.0, abs(rloss)), (loss, rloss)
    gv, rv = tf.unflatten(g.cpu().double(), m.cfg), tf.unflatten(rg, m.cfg)
    worst, bad = 0.0, []
    top = float(rg.abs().max())
    for k in gv:
        if k.endswith("_bk:0"):
            # a key bias shifts every score of a softmax row alike: its gradient is zero in exact arithmetic, so both
            # sides are roundoff, held to an absolute bound instead
            assert float(gv[k].abs().max()) < 1e-5 * top and float(rv[k].abs().max()) < 1e-5 * top, k
            continue
        scale = float(rv[k].abs().max())
        if scale == 0.0:        # e.g. a row with one unmasked key: that softmax is constant
            assert float(gv[k].abs().max()) < 1e-6 * top, k
            continue
        err = float((gv[k] - rv[k]).abs().max()) / scale
        worst = max(worst, err)
        if err >= 1e-4:
            bad.append((k, err))
    assert not bad, (bad, "loss positions at a clip edge: %d" % edge)
    print("n=%d V=%d Ts=%d Tt=%d H=%d: loss %.6f worst rel err %.2e, %d loss positions at a clip edge"
          % (n, V, Ts, Tt, H, loss, worst, edge))


def test_training_matches_twin_rerun_and_epoch():
    enc, dec, y = _data(300, 10, 6, 286, seed=5)
    runs = []
    for dev in ("cuda", "cuda", "cpu"):
        m = tf.get_model(286, 64, 1, 1, 2, 64, dropout_rate=0.05, use_same_embed=False, seed=2, device=dev)
        m.compile("adam", "sparse_categorical_crossentropy")
        np.random.seed(7)
        h = m.fit([enc, dec], y, epochs=2, batch_size=32, verbose=0)     # 10 steps per epoch, 20 chained steps
        runs.append((m.flat.cpu().clone(), h.history["loss"]))
    assert torch.equal(runs[0][0], runs[1][0]) and runs[0][1] == runs[1][1]
    scale = float(runs[2][0].abs().max())
    assert float((runs[0][0] - runs[2][0]).abs().max()) < 2e-3 * scale
    assert np.allclose(runs[0][1], runs[2][1], rtol=1e-3)
    # the epoch call equals its steps
    m1 = tf.get_model(286, 64, 1, 1, 2, 64, dropout_rate=0.05, use_same_embed=False, seed=2, device="cuda")
    m1.compile("adam", "sparse_categorical_crossentropy")
    np.random.seed(7)
    idx = np.arange(300)
    np.random.shuffle(idx)
    for k in range(10):
        b = idx[k * 32:(k + 1) * 32]
        _, g = m1.grad(enc[b], dec[b], y[b], call=k)
        m1.apply(g)
    m2 = tf.get_model(286, 64, 1, 1, 2, 64, dropout_rate=0.05, use_same_embed=False, seed=2, device="cuda")
    m2.compile("adam", "sparse_categorical_crossentropy")
    np.random.seed(7)
    m2.fit([enc, dec], y, epochs=1, batch_size=32, verbose=0)
    assert torch.equal(m1.flat, m2.flat)


def _near_tie_rows(path, score, rpath, rscore):
    """Rows whose paths differ; each must be a near-tie (the same scores, in another order or with other tokens of equal
    probability)."""
    same = (path == rpath).all(axis=(1, 2))
    tie = ~same & np.isclose(np.sort(score, 1), np.sort(rscore, 1), rtol=1e-4).all(axis=1)
    assert (same | tie).all(), np.where(~(same | tie))[0][:5]
    assert np.allclose(score[same], rscore[same], rtol=1e-5)
    return int(tie.sum())


def test_predict_and_searches_against_reference_and_twin():
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mdpcheck", "search.npz"))
    cfg = dict(token_num=[120, 120], embed_dim=32, encoder_num=1, decoder_num=1, head_num=2, hidden_dim=64)
    m = tf.get_model(use_same_embed=False, device="cuda", **cfg)
    cpu = tf.get_model(use_same_embed=False, device="cpu", **cfg)
    m.flat.copy_(torch.as_tensor(z["flat"]))
    cpu.flat = torch.as_tensor(z["flat"]).clone()
    enc, dec = z["enc"].astype(np.int64), z["dec"].astype(np.int64)
    # predict at batch 2048 against the twin and float64
    full = np.concatenate([np.ones((2048, 1), int), np.tile(dec[:, 1:], (8, 1))], 1)
    p = m.predict([enc, full])
    assert np.abs(p - cpu.predict([enc, full])).max() < 1e-5
    assert np.abs(p[:256] - ref.probs64(m.flat, m.cfg, enc[:256], full[:256])).max() < 1e-5
    # the reference's decode_step and token_probs
    st = dc.decode_step(m, enc[:256], dec, beam_size=10)
    assert st.shape == (256, 10, 2) and st.dtype == np.float64
    rst = z["step"]
    same = (st[..., 1] == rst[..., 1]).all(axis=1)
    assert np.allclose(np.sort(st[..., 0], 1), np.sort(rst[..., 0], 1), rtol=1e-5)
    tp = dc.token_probs(m, enc[:256], dec)
    assert tp.shape == (256, 120) and tp.dtype == np.float32 and np.abs(tp - z["probs"]).max() < 1e-5
    print("decode_step: %d of 256 rows order near-ties differently" % int((~same).sum()))
    for beam, cand, grows in ((1, 0, 2048), (20, 20, 2048), (100, 0, 128)):
        path, score = dc.beam_search(m, enc, beam, 5, use_candidates=cand > 0, candidates_size=cand)
        assert path.shape == (2048, beam, 6) and score.shape == (2048, beam) and score.dtype == np.float64
        key = "%d_%d" % (beam, cand)
        gt = _near_tie_rows(path[:grows], score[:grows], z["path_" + key].astype(np.int64),
                            z["score_" + key].astype(np.float64))
        tpath, tscore = dc.beam_search(cpu, enc, beam, 5, use_candidates=cand > 0, candidates_size=cand)
        tt = _near_tie_rows(path, score, tpath, tscore)
        print("beam %d cand %d: near-tie rows %d of %d against the reference, %d of 2048 against the twin"
              % (beam, cand, gt, grows, tt))
    pp = dc.path_probs(m, enc, path)
    assert np.allclose(np.prod(pp.astype(np.float64), -1), score, rtol=1e-4)


def test_capi_rejects_and_counts():
    lib = _capi.load_library()
    c = _capi.S2SConfig(286, 286, 48, 1, 128, 1, 1, 0)           # embed_dim not a multiple of 32
    assert lib.r4_s2s_num_params(C.byref(c)) == -1
    n0 = lib.r4_s2s_launch_count()
    rc = lib.r4_s2s_grad(C.byref(c), None, None, None, None, 4, 5, 5, 0, 0, 0.0, None, None, None, None)
    assert rc == -1 and lib.r4_s2s_launch_count() == n0
    m = _model(286, 64, 1, 64, 1, 1, False)
    counts = []
    for n in (8, 64):
        enc, dec, y = _data(n, 10, 7, 289, seed=n)
        k0 = lib.r4_s2s_launch_count()
        m.grad(enc, dec, y)
        k1 = lib.r4_s2s_launch_count()
        dc.beam_search(m, enc, 4, 5)
        counts.append((k1 - k0, lib.r4_s2s_launch_count() - k1))
    assert counts[0] == counts[1], counts
    print("launches per train step %d, per 5-step search %d" % counts[0])


def _planted(path, n=30000, V=200, seed=0):
    rs = np.random.RandomState(seed)
    lines = ["sessionid items"]
    for s in range(n):
        hist = rs.randint(1, V, 16)
        nxt = [(int(hist[-1]) * 7 + k * 13) % V + 1 for k in range(5)]
        lines.append("%d %s" % (s, ",".join(str(x) for x in list(hist) + nxt)))
    with open(os.path.join(path, "rl4rs.csv"), "w") as f:
        f.write("\n".join(lines) + "\n")


def test_main_end_to_end(tmp_path):
    from rl4rs_b200.mdpchecker import mdp_checker
    _planted(str(tmp_path))
    out = []
    res = mdp_checker.main("rl4rs", str(tmp_path), epochs=4, holdout=2000, eval_rows=512, beam_size=20,
                           weights_path=str(tmp_path / "w.npz"), print_fn=lambda *a: out.append(" ".join(map(str, a))))
    enc = np.asarray(res["encode_input"])
    inv = {v: k for k, v in mdp_checker.prepare("rl4rs.csv", str(tmp_path), lambda *a: None)[4].items()}
    greedy = res["output_greedy"][:, 0, 1:6]
    hits = 0
    for r in range(len(enc)):
        last = int(inv[int(enc[r, 16])])
        want = [str((last * 7 + k * 13) % 200 + 1) for k in range(5)]
        hits += [inv[int(t)] for t in greedy[r]] == want
    print("greedy reproduces the planted continuation on %d of %d rows" % (hits, len(enc)))
    assert hits >= 0.95 * len(enc)
    assert "experiment II results" in out and "experiment I results" in out
    assert np.asarray(res["experiment_i"]).shape == (5, 2)
