"""GPU: the MDP checker's kernels (r4_s2s_*) at the edges of what their C-ABI accepts, beyond test_gpu_mdpcheck.py.

  gradient grid   one point per edge (the test id names it), each held to the float64 reference of mdpcheck_ref64.py run
                  on the GPU in torch, which takes the kernels' relu decisions: the loss within 1e-5, each tensor within
                  1e-4 of its largest reference element (1e-3 at the 65 535-row point, POINT_BAR), key biases against
                  1e-5 of the largest element of the gradient
  training        20 chained fit steps at the script's model size against the torch twin; reruns bit-identical, the
                  epoch call equal to its steps
  clipped loss    planted weights (mdpcheck_ref64.plant_clip) put targets below 1e-7 and top tokens above 1 - 1e-7, every
                  probability at least 100 times from its edge, at the same bars
  exact selection planted ties (bit-identical logit columns, a zero-probability group) straddling the k-th and beam-th
                  positions; decode_step and every search step equal to the NumPy replay of the selection rule fed by
                  predict's probabilities -- indices exact, values and scores bit for bit, no near-tie allowance
  rejections      one step past each edge every entry point returns R4_ERR_ARG and launches nothing

Every gradient and clip comparison is recorded as an `mdpcheck ...` row of the margin report.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import mdpcheck_ref64 as ref
from golden_util import record_margin
from rl4rs_b200 import _capi
from rl4rs_b200.mdpchecker import decoder as dc
from rl4rs_b200.mdpchecker import transformer as tf

pytestmark = pytest.mark.gpu

LOSS_BAR, GRAD_BAR, BK_BAR = 1e-5, 1e-4, 1e-5
# The 65 535-row point sums each embedding-gradient element over up to 131 070 positions, and each weight-gradient tile
# over 65 535 or 131 070 rows, sequentially in float32, and those sums cancel.  On the H100 its worst tensor missed
# float64 by 6.8e-4, and torch's float32 autograd of the same model by 1.7e-4 (DESIGN.md): the 1e-4 bar is below float32
# roundoff there, so that point is held to 1e-3, and the float32 autograd's error is printed beside the kernels'.
POINT_BAR = {"n_heads_65535": 1e-3}

GRID = [  # edge, n, Vs, Vt, Ts, Tt, E, H, F, Le, Ld, same, dropout
    ("every_minimum", 1, 4, 4, 1, 1, 32, 1, 32, 1, 1, True, 0.0),
    ("script_model_size", 65, 286, 286, 18, 7, 256, 1, 128, 1, 1, False, 0.1),
    ("one_column_heads_maxV_len64", 3, 33, 65536, 64, 64, 32, 32, 32, 1, 1, False, 0.0),
    ("odd_heads_maxF_len33_32", 9, 300, 301, 33, 32, 96, 3, 1024, 2, 2, False, 0.5),
    ("maxE_6_blocks_each", 2, 286, 286, 17, 9, 512, 8, 64, 6, 6, True, 0.1),
    ("n_heads_65535", 65535, 4, 4, 1, 2, 32, 1, 32, 1, 1, False, 0.0),
    ("large_src_small_tgt", 64, 65536, 4, 64, 8, 128, 4, 256, 1, 1, False, 0.0),
    ("tgt_len1_dropout09", 257, 5003, 5003, 64, 1, 64, 2, 64, 1, 1, True, 0.9),
]


def _data(n, Ts, Tt, Vs, Vt, seed):
    rs = np.random.RandomState(seed)
    enc = rs.randint(3, Vs, (n, Ts))
    enc[:, 0] = 1
    dec = rs.randint(3, Vt, (n, Tt))
    dec[:, 0] = 1
    y = rs.randint(0, Vt, (n, Tt))
    for r in range(n):
        enc[r, rs.randint(1, Ts + 1):] = 0
        dec[r, rs.randint(1, Tt + 1):] = 0
    return enc, dec, y


def _model(Vs, Vt, E, H, F, Le, Ld, same, seed, rate):
    m = tf.get_model([Vs, Vt], E, Le, Ld, H, F, dropout_rate=rate, use_same_embed=same, seed=seed, device="cuda")
    with torch.no_grad():   # move LayerNorm and biases off their initial values
        g = torch.Generator(device="cuda").manual_seed(seed)
        for k, t in tf.unflatten(m.flat, m.cfg).items():
            if t.dim() == 1:
                t.add_(0.1 * torch.randn(t.shape, generator=g, device="cuda"))
    return m


def _kernel_grad(m, enc, dec, y, call):
    """(loss, flat gradient, the kernels' relu decisions per FeedForward, on the device) of one r4_s2s_grad call."""
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
        keep.append((scr[o // 4:o // 4 + n * T * m.cfg.F].view(n, T, m.cfg.F) > 0).double())
    return float(loss.item()), g.double().cpu(), keep


def _hold(tag, m, enc, dec, y, call, bar=GRAD_BAR):
    """The kernels' loss and gradient against float64 at the bars; returns the reference probabilities."""
    loss, g, keep = _kernel_grad(m, enc, dec, y, call)
    rloss, rg, probs = ref.grad64(m.flat, m.cfg, enc, dec, y, seed=m.seed, call=call, rate=m.dropout_rate,
                                  relu_keep=keep, device="cuda")
    worst, bad, bk = ref.grad_errors(g, rg, m.cfg)
    if bar != GRAD_BAR:
        # the yardstick of a looser bar: the same autograd in float32 on the same inputs, against the same reference
        _, g32, _ = ref.grad64(m.flat, m.cfg, enc, dec, y, seed=m.seed, call=call, rate=m.dropout_rate, relu_keep=keep,
                               device="cuda", dtype=torch.float32)
        w32, bad32, _ = ref.grad_errors(g32, rg, m.cfg)
        print("%s: float32 autograd misses float64 by %.2e (%s); the kernels by %.2e (%s)"
              % (tag, w32, [(k, "%.1e" % e) for k, e in bad32], worst, [(k, "%.1e" % e) for k, e in bad]))
        bad = [(k, e) for k, e in bad if e >= bar]
    lerr = abs(loss - rloss) / max(1.0, abs(rloss))
    record_margin("mdpcheck %s loss" % tag, np.array([lerr]), np.array([LOSS_BAR]), np.array([rloss]))
    record_margin("mdpcheck %s grad" % tag, np.array([worst]), np.array([bar]), np.array([1.0]))
    record_margin("mdpcheck %s key bias" % tag, np.array([bk]), np.array([BK_BAR]), np.array([1.0]))
    edge = ref.clip_edge_rows(probs, dec)
    print("%s: loss %.6f (err/bar %.2f), worst tensor err/bar %.3f, key bias/bar %.3f, %d loss positions at a clip edge"
          % (tag, loss, lerr / LOSS_BAR, worst / bar, bk / BK_BAR, edge))
    assert lerr <= LOSS_BAR, (loss, rloss)
    assert not bad, (bad, "loss positions at a clip edge: %d" % edge)
    assert bk < BK_BAR
    return probs


@pytest.mark.parametrize("edge,n,Vs,Vt,Ts,Tt,E,H,F,Le,Ld,same,rate", GRID, ids=[p[0] for p in GRID])
def test_gradient_at_the_edges(edge, n, Vs, Vt, Ts, Tt, E, H, F, Le, Ld, same, rate):
    m = _model(Vs, Vt, E, H, F, Le, Ld, same, seed=n % 1000 + E, rate=rate)
    enc, dec, y = _data(n, Ts, Tt, m.cfg.Vs, m.cfg.Vt, seed=n % 1000 + F)
    _hold(edge, m, enc, dec, y, call=5, bar=POINT_BAR.get(edge, GRAD_BAR))


def test_training_at_the_script_size():
    enc, dec, y = _data(320, 18, 7, 286, 286, seed=9)
    runs = []
    for dev in ("cuda", "cuda", "cpu"):
        m = tf.get_model(286, 256, 1, 1, 1, 128, dropout_rate=0.1, use_same_embed=False, seed=4, device=dev)
        m.compile("adam", "sparse_categorical_crossentropy")
        np.random.seed(7)
        h = m.fit([enc, dec], y, epochs=2, batch_size=32, verbose=0)     # 10 steps per epoch, 20 chained steps
        runs.append((m.flat.cpu().clone(), h.history["loss"]))
    assert torch.equal(runs[0][0], runs[1][0]) and runs[0][1] == runs[1][1]
    scale = float(runs[2][0].abs().max())
    err = float((runs[0][0] - runs[2][0]).abs().max())
    record_margin("mdpcheck training script size", np.array([err]), np.array([2e-3 * scale]), np.array([scale]))
    assert err < 2e-3 * scale
    assert np.allclose(runs[0][1], runs[2][1], rtol=1e-3)
    m1 = tf.get_model(286, 256, 1, 1, 1, 128, dropout_rate=0.1, use_same_embed=False, seed=4, device="cuda")
    m1.compile("adam", "sparse_categorical_crossentropy")
    np.random.seed(7)
    idx = np.arange(320)
    np.random.shuffle(idx)
    for k in range(10):
        b = idx[k * 32:(k + 1) * 32]
        _, g = m1.grad(enc[b], dec[b], y[b], call=k)
        m1.apply(g)
    m2 = tf.get_model(286, 256, 1, 1, 1, 128, dropout_rate=0.1, use_same_embed=False, seed=4, device="cuda")
    m2.compile("adam", "sparse_categorical_crossentropy")
    np.random.seed(7)
    m2.fit([enc, dec], y, epochs=1, batch_size=32, verbose=0)
    assert torch.equal(m1.flat, m2.flat)
    print("training at E 256: flat err %.2e of %.3f, losses %s vs twin %s" % (err, scale, runs[0][1], runs[2][1]))


def test_clipped_loss_planted():
    m, enc, dec, y = ref.clip_case(device="cuda")
    probs = _hold("clipped loss", m, enc, dec, y, call=0)
    margin = ref.clip_margin(probs, dec)
    clipped_t, clipped_top = ref.clip_counts(probs, dec, y)
    pos = int((dec != 0).sum())
    # the kernels' own float32 probabilities make the same clip decisions
    p32 = m.predict([enc, dec]).astype(np.float64)
    assert ref.clip_counts(p32, dec, y) == (clipped_t, clipped_top)
    print("clipped loss: %d loss positions, %d with a clipped target, %d with a top token clipped high, margin %.0fx"
          % (pos, clipped_t, clipped_top, margin))
    assert margin >= 100.0 and clipped_t >= 0.3 * pos and clipped_top >= 0.15 * pos


# ---- exact selection -------------------------------------------------------------------------------------------------
def _tie_model(Vt, groups, zero, E=32, H=1, Vs=64, seed=4):
    m = ref.tie_model(Vs, Vt, E, H, 32, seed, groups, zero, device="cuda")
    p = m.predict([np.ones((1, 1), int), np.ones((1, 1), int)])[0, 0]
    for _, toks in groups:                     # the ties are there, bit for bit
        assert (p[toks] == p[toks[0]]).all()
    assert (p[zero] == 0).all()
    return m


def _enc(n, Ts, Vs, seed):
    rs = np.random.RandomState(seed)
    enc = rs.randint(3, Vs, (n, Ts))
    enc[:, 0] = 1
    return enc


TIE_V65536 = dict(groups=[(6.0, list(range(100, 200))), (3.0, list(range(1000, 10000)))], zero=list(range(20000, 30000)))
TIE_V8193 = dict(groups=[(4.0, list(range(10, 40))), (2.0, list(range(100, 8191)))], zero=[8191, 8192])
TIE_V300 = dict(groups=[(4.0, list(range(10, 20))), (2.0, list(range(30, 290)))], zero=list(range(290, 300)))
TIE_V8000 = dict(groups=[(4.0, list(range(10, 20))), (2.0, list(range(100, 6100)))], zero=list(range(7000, 8000)))

STEPS = [  # id, Vt, ties, k, candidates per row (0: none)
    ("k8192_V65536", 65536, TIE_V65536, 8192, 0),
    ("k8192_V65536_cand8192", 65536, TIE_V65536, 8192, 8192),
    ("k8192_V8193", 8193, TIE_V8193, 8192, 0),
    ("k12_V300_cand40", 300, TIE_V300, 12, 40),
]


@pytest.mark.parametrize("what,Vt,ties,k,C", STEPS, ids=[s[0] for s in STEPS])
def test_decode_step_equals_replay(what, Vt, ties, k, C):
    m = _tie_model(Vt, **ties)
    n, Tt = 6, 4
    rs = np.random.RandomState(k)
    enc = _enc(n, 9, 64, seed=k)
    dec = np.concatenate([np.ones((n, 1), int), rs.choice(ties["groups"][1][1], (n, Tt - 1))], 1)
    dec[0, 2] = ties["groups"][0][1][3]
    cand = None
    if C:
        cand = np.stack([rs.permutation(Vt)[:C] for _ in range(n)])
        cand[:, :2] = ties["zero"][:2]             # candidates of probability 0
    st = dc.decode_step(m, enc, dec, candidates=cand, beam_size=k)
    p = m.predict([enc, dec])
    keys = p[:, -1].astype(np.float64)
    if cand is not None:
        mask = np.zeros_like(keys)
        np.put_along_axis(mask, cand, 1.0, 1)
        keys = keys * mask
    val, idx = ref.top_rule(keys, k)
    assert np.array_equal(st[..., 1].astype(np.int64), idx)
    assert np.array_equal(st[..., 0], val)           # bit for bit: predict's f32 probabilities as doubles
    # the k-th position cuts a tie in every row: the radix select's equal-key path decided which tokens go in
    srt = -np.sort(-keys, 1)
    assert (srt[:, k - 1] == srt[:, k]).all()
    assert np.abs(p - ref.probs64(m.flat, m.cfg, enc, dec, device="cuda")).max() < 1e-5


SEARCHES = [  # id, n, Vt, ties, beam, candidates, target length
    ("beam256_n255", 255, 300, TIE_V300, 256, 0, 3),
    ("beam255_n257", 257, 300, TIE_V300, 255, 0, 3),
    ("target_len63", 3, 300, TIE_V300, 4, 0, 63),
    ("cand8192_V65536", 4, 65536, TIE_V65536, 8, 8192, 3),
    ("cand6000", 4, 8000, TIE_V8000, 20, 6000, 3),
    ("cand5_lt_beam16", 8, 300, TIE_V300, 16, 5, 4),
]


@pytest.mark.parametrize("what,n,Vt,ties,beam,ncand,T", SEARCHES, ids=[s[0] for s in SEARCHES])
def test_search_steps_equal_replay(what, n, Vt, ties, beam, ncand, T):
    m = _tie_model(Vt, **ties)
    enc = _enc(n, 7, 64, seed=beam)
    p1 = m.predict([enc, np.ones((n, 1), int)])[:, -1]
    rp, rsc, mask = ref.replay_first(p1, beam, ncand)
    encr = np.repeat(enc, beam, axis=0)
    ties_seen = 0
    for t in range(1, T + 1):
        path, score = dc.beam_search(m, enc, beam, t, use_candidates=ncand > 0, candidates_size=ncand)
        assert np.array_equal(path, rp), (what, t)
        assert np.array_equal(score, rsc), (what, t)          # bit for bit
        ties_seen += int((score[:, 1:] == score[:, :-1]).sum())
        if t < T:
            # the replay of step t + 1, fed by predict on this search's own paths
            q = m.predict_tensor(encr, path.reshape(n * beam, t + 1))[:, -1].cpu().numpy()
            rp, rsc = ref.replay_step(q, path, score, mask)
    print("%s: %d steps equal to the replay, %d tied adjacent scores" % (what, T, ties_seen))
    assert ties_seen > 0
    if what == "target_len63":
        # Experiment I's scores: r4_s2s_score at L = 64, bit-equal to predict along the same paths
        pp = dc.path_probs(m, enc, path)
        full = m.predict([encr, path[:, :, :T].reshape(n * beam, T)])
        want = np.take_along_axis(full, path[:, :, 1:].reshape(n * beam, T, 1), 2).reshape(n, beam, T)
        assert pp.shape == (n, beam, 63) and np.array_equal(pp, want)


def test_chunked_search_equals_another_split():
    m = _tie_model(300, **TIE_V300)
    n, beam = 300, 255
    enc = _enc(n, 7, 64, seed=3)
    rows, _ = m._chunk(_capi.S2S_SEARCH, n, 7, 2, beam, 0)
    assert rows == 257 and n % rows != 0                # 65 535 // 255: chunks of 257 and 43 rows
    path, score = dc.beam_search(m, enc, beam, 2)
    parts = [dc.beam_search(m, enc[a:b], beam, 2) for a, b in ((0, 150), (150, 300))]
    assert np.array_equal(path, np.concatenate([x[0] for x in parts]))
    assert np.array_equal(score, np.concatenate([x[1] for x in parts]))


def test_rejections_launch_nothing():
    lib = _capi.load_library()
    buf = torch.zeros(16, device="cuda")
    torch.cuda.synchronize()
    n0 = lib.r4_s2s_launch_count()
    got = ref.abi_rejections(lib, _capi.ptr(buf))
    assert [x for x in got if x[1] != -1] == []
    assert lib.r4_s2s_launch_count() == n0
    torch.cuda.synchronize()
    print("%d rejections, no launch" % len(got))
