"""A float64 autograd reference for the MDP checker's transformer: the restatement in rl4rs_b200/mdpchecker/transformer.py
(forward, loss_fn) run in float64, on the CPU or in chunks on the GPU (device=), with the same dropout draws, so the
kernels' gradients are held to it tensor by tensor.  relu_keep hands it the kernels' relu decisions (a pre-activation
within roundoff of 0 could otherwise be decided differently in float32 and float64).

Also here, shared by the CPU and GPU shape modules: the planted models of the clipped-loss and exact-selection tests, and
the search replay -- the documented selection rule of decoder.py written out in NumPy float64."""
import numpy as np
import torch

from rl4rs_b200.mdpchecker import transformer as tf

CLIP = 1e-7
HI = float(np.float32(1) - np.float32(CLIP))       # the upper clip edge, as the kernels and the twin hold it


def grad64(flat, cfg, enc, dec, target, seed=0, call=0, rate=0.0, relu_keep=None, device="cpu", loss_fn=None,
           dtype=torch.float64):
    """(loss, flat gradient, probabilities [n, Tt, Vt]) in float64 at the float32 weights flat.  loss_fn replaces
    transformer.loss_fn (the CPU tests swap in faulty variants of it); dtype float32 runs the same autograd in float32,
    a yardstick for the roundoff of a float32 computation."""
    dev = torch.device(device)
    p = flat.detach().to(dev).to(dtype).requires_grad_(True)
    enc, dec, target = (torch.as_tensor(np.asarray(a), dtype=torch.int64, device=dev) for a in (enc, dec, target))
    keep = None if relu_keep is None else [torch.as_tensor(k, dtype=dtype, device=dev) for k in relu_keep]
    logits = tf.forward(tf.unflatten(p, cfg), cfg, enc, dec, seed, call, rate, relu_keep=keep)
    loss = (loss_fn or tf.loss_fn)(logits, dec, target)
    loss.backward()
    return (float(loss.detach()), p.grad.detach().cpu().double(),
            torch.softmax(logits.detach().double(), -1).cpu().numpy())


def clip_edge_rows(probs, dec, rel=1e-3):
    """Loss positions (decoder input != 0) holding a probability within rel of a clip edge (1e-7 or 1 - 1e-7), where
    float32 and float64 may pass or stop the gradient differently."""
    near = (np.abs(probs - CLIP) < rel * CLIP) | (np.abs(probs - (1 - CLIP)) < rel * CLIP)
    return int((near.any(-1) & (np.asarray(dec) != 0)).sum())


def clip_margin(probs, dec):
    """The least factor by which any probability of a loss position stays away from its clip edge: p against 1e-7, and
    1 - p against 1e-7 (inf when there is no loss position)."""
    p = probs[np.asarray(dec) != 0]
    if p.size == 0:
        return np.inf
    lo = np.maximum(p / CLIP, CLIP / np.maximum(p, 1e-300))
    q = np.maximum(1.0 - p, 1e-300)
    hi = np.maximum(q / CLIP, CLIP / q)
    return float(min(lo.min(), hi.min()))


def clip_counts(probs, dec, target):
    """(loss positions whose target probability is clipped, loss positions whose top probability is clipped high)."""
    m = np.asarray(dec) != 0
    pt = np.take_along_axis(probs, np.asarray(target)[..., None], -1)[..., 0]
    clipped_t = (pt < CLIP) | (pt > HI)
    top = probs.max(-1) > HI
    return int((clipped_t & m).sum()), int((top & m).sum())


def loss_noclip(logits, dec, target):
    """A faulty loss: the cross-entropy without keras' clip."""
    ce = -torch.log_softmax(logits, -1).gather(-1, target.unsqueeze(-1)).squeeze(-1)
    m = (dec != 0).to(ce.dtype)
    return (ce * m).sum() / m.sum()


def loss_passthrough(logits, dec, target):
    """A faulty loss: the clipped values of keras' loss, but the gradient passed through the clipped entries."""
    p = torch.softmax(logits, -1)
    q = p + (p.clamp(CLIP, HI) - p).detach()
    ce = torch.log(q.sum(-1)) - torch.log(q.gather(-1, target.unsqueeze(-1)).squeeze(-1))
    m = (dec != 0).to(ce.dtype)
    return (ce * m).sum() / m.sum()


def probs64(flat, cfg, enc, dec, device="cpu", rows=None):
    """Softmax probabilities [n, Tt, Vt] in float64, `rows` source rows at a time (all at once when None)."""
    dev = torch.device(device)
    n = len(enc)
    rows = rows or n
    out = []
    with torch.no_grad():
        w = tf.unflatten(flat.detach().to(dev).double(), cfg)
        for r0 in range(0, n, rows):
            e, d = (torch.as_tensor(np.asarray(a[r0:r0 + rows]), dtype=torch.int64, device=dev) for a in (enc, dec))
            out.append(torch.softmax(tf.forward(w, cfg, e, d), -1).cpu().numpy())
    return np.concatenate(out)


# ---- planted models ---------------------------------------------------------------------------------------------------
def plant_clip(model, rs):
    """Weights that put probabilities far from both clip edges (transformer.Model, use_same_embed False, Vt >= 16).
    Token 2: output bias -40, so p ~ 1e-19 in every row.  Token 3: bias set so p ~ 1e-10 to 1e-9, at least 100 times
    below 1e-7 yet close enough that a gradient let through the clip would be visible.  Token 4 (the trigger): a large
    decoder embedding along a unit direction u and a bias of -u's typical score: where a row's decoder input is token 4
    its top probability is 1 - O(1e-40), elsewhere token 4's is O(1e-40).  The other embeddings are scaled down so every
    ordinary probability stays near 1 / V; the sub-layers' output projections are scaled down so the trigger's direction
    survives to the last LayerNorm.  Returns (A_deep, A_near, trigger) token ids."""
    cfg = model.cfg
    w = tf.unflatten(model.flat, cfg)
    with torch.no_grad():
        emb = w["Decoder-Token-Embedding/embeddings:0"]
        emb.mul_(0.3)
        for k, t in w.items():
            if k.endswith(("_Wo:0", "_W2:0")):
                t.mul_(0.1)
        u = torch.as_tensor(rs.randn(cfg.E), dtype=emb.dtype)
        u = u - u.mean()
        u = u / u.norm()
        emb[4] = (60.0 * u).to(emb.device)
        b = w["Output/bias:0"]
        b[2] = -40.0
        b[3] = -17.5
        b[4] = -60.0 * 0.5 * float(np.sqrt(cfg.E))
    return 2, 3, 4


def plant_ties(model, groups, zero=()):
    """Bit-identical logit columns: each group (token ids) gets one decoder-embedding row and one output bias, (bias,
    tokens) per group; tokens of `zero` get bias -1000, so their f32 probabilities are exactly 0.  use_same_embed False."""
    cfg = model.cfg
    w = tf.unflatten(model.flat, cfg)
    with torch.no_grad():
        emb, b = w["Decoder-Token-Embedding/embeddings:0"], w["Output/bias:0"]
        for bias, toks in groups:
            toks = torch.as_tensor(np.asarray(toks), dtype=torch.int64, device=emb.device)
            emb[toks] = emb[toks[0]].clone()
            b[toks] = float(bias)
        if len(zero):
            b[torch.as_tensor(np.asarray(zero), dtype=torch.int64, device=b.device)] = -1000.0


def clip_case(device="cpu"):
    """(model, enc, dec, target) of the clipped-loss test: 64 rows, 128 tokens, lengths 8, the weights of
    mdpcheck_ref64.plant_clip; targets 20 % the deep-clipped token, 20 % the near-clipped one; decoder inputs 30 % the
    trigger (whose rows have a top probability clipped high)."""
    V, n, Ts, Tt = 128, 64, 8, 8
    m = tf.get_model([V, V], 64, 1, 1, 2, 64, use_same_embed=False, seed=3, device=device)
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for k, t in tf.unflatten(m.flat, m.cfg).items():
            if t.dim() == 1:
                t.add_((0.1 * torch.randn(t.shape, generator=g)).to(t.device))
    rs = np.random.RandomState(11)
    deep, near, trig = plant_clip(m, rs)
    enc = rs.randint(3, V, (n, Ts))
    enc[:, 0] = 1
    dec = rs.randint(5, V, (n, Tt))
    dec[:, 0] = 1
    dec[rs.rand(n, Tt) < 0.3] = trig
    y = rs.randint(5, V, (n, Tt))
    u = rs.rand(n, Tt)
    y[u < 0.2] = deep
    y[(u >= 0.2) & (u < 0.4)] = near
    for r in range(n):
        dec[r, rs.randint(2, Tt + 1):] = 0
    return m, enc, dec, y


def tie_model(Vs, Vt, E, H, F, seed, groups, zero, device="cpu"):
    m = tf.get_model([Vs, Vt], E, 1, 1, H, F, use_same_embed=False, seed=seed, device=device)
    plant_ties(m, groups, zero)
    return m


# ---- the search replay ------------------------------------------------------------------------------------------------
def top_rule(keys, k):
    """(values, indices) of the k largest of each row of keys (f64): value descending, ties to the lower index."""
    order = np.argsort(-keys, axis=1, kind="stable")[:, :k]
    return np.take_along_axis(keys, order, 1), order


def replay_first(p, beam, n_cand=0):
    """Step 1 from the START probabilities p [n, V] (f32): (paths [n, beam, 2], scores [n, beam], candidate mask or
    None).  The candidates are the top n_cand of the same probabilities."""
    keys = p.astype(np.float64)
    val, idx = top_rule(keys, beam)
    n = len(p)
    path = np.ones((n, beam, 2), np.int64)
    path[:, :, 1] = idx
    mask = None
    if n_cand:
        mask = np.zeros_like(keys)
        np.put_along_axis(mask, top_rule(keys, n_cand)[1], 1.0, 1)
    return path, val, mask


def replay_step(p, path, score, mask=None):
    """One step from the next-token probabilities p [n * beam, V] (f32) after each path [n, beam, L]: a token's key is
    its probability as a double times the candidate mask; each prefix keeps its top beam; the new beams are the top beam
    of score[b, i] * val[b, i, j] in double, ties to the lower flat index i beam + j.  Returns (paths [n, beam, L + 1],
    scores)."""
    n, beam, L = path.shape
    keys = p.astype(np.float64)
    if mask is not None:
        keys = keys * np.repeat(mask, beam, axis=0)
    val, tok = top_rule(keys, beam)
    prod = (score[:, :, None] * val.reshape(n, beam, beam)).reshape(n, beam * beam)
    sv, f = top_rule(prod, beam)
    i, j = f // beam, f % beam
    rows = np.arange(n)[:, None]
    out = np.concatenate([path[rows, i], tok.reshape(n, beam, beam)[rows, i, j][..., None]], axis=2)
    return out, sv


# ---- gradient comparison -----------------------------------------------------------------------------------------------
def grad_errors(g, rg, cfg):
    """Per tensor of the flat gradients g (under test) and rg (the reference), both float64 on the CPU: (worst |g - rg| /
    max |rg| over the tensors, [(name, err)] of the tensors at or above 1e-4, worst key-bias magnitude / max |rg|).  Key
    biases shift every score of a softmax row alike, so their gradient is zero in exact arithmetic and both sides are
    roundoff: they are returned apart, for an absolute bound (1e-5 of the largest reference element).  A tensor whose
    reference is exactly zero is held to 1e-6 of the largest reference element."""
    gv, rv = tf.unflatten(g, cfg), tf.unflatten(rg, cfg)
    top = float(rg.abs().max())
    worst, bad, bk = 0.0, [], 0.0
    for k in gv:
        if k.endswith("_bk:0"):
            bk = max(bk, float(gv[k].abs().max()) / top, float(rv[k].abs().max()) / top)
            continue
        scale = float(rv[k].abs().max())
        if scale == 0.0:
            err = float(gv[k].abs().max()) / top * 1e2          # held to 1e-6 of top: reported on the 1e-4 scale
        else:
            err = float((gv[k] - rv[k]).abs().max()) / scale
        worst = max(worst, err)
        if err >= 1e-4:
            bad.append((k, err))
    return worst, bad, bk


# ---- the C-ABI's edges -------------------------------------------------------------------------------------------------
def abi_rejections(lib, P):
    """[(label, rc)] of r4_s2s_* entry points called one step past each edge their arguments accept.  P: a non-NULL
    address passed for every buffer; each call is refused on the host before anything is read or launched, so P is never
    dereferenced.  Only the entry points an edge applies to are called.  Every rc must be R4_ERR_ARG (-1)."""
    import ctypes as C
    from rl4rs_b200 import _capi

    def cfg(t):
        return C.byref(_capi.S2SConfig(*t))

    def calls(c, names, n=4, Ts=5, Tt=5, rate=0.0, beam=4, tl=5, ncand=0, k=4, sbeam=4, stl=5):
        """the entry points `names` at config c and these shapes (each called only when named)"""
        fn = {"num_params": lambda: lib.r4_s2s_num_params(c),
              "scratch train": lambda: lib.r4_s2s_scratch_size(c, _capi.S2S_TRAIN, n, Ts, Tt, 1, 0),
              "scratch search": lambda: lib.r4_s2s_scratch_size(c, _capi.S2S_SEARCH, n, Ts, tl, beam, ncand),
              "scratch step": lambda: lib.r4_s2s_scratch_size(c, _capi.S2S_STEP, n, Ts, Tt, 1, k),
              "relu_offsets": lambda: lib.r4_s2s_relu_offsets(c, n, Ts, Tt, P),
              "grad": lambda: lib.r4_s2s_grad(c, P, P, P, P, n, Ts, Tt, 0, 0, rate, P, P, P, None),
              "apply": lambda: lib.r4_s2s_apply(c, P, P, P, P, 1, 1e-3, 0.9, 0.999, 1e-7, None),
              "epoch": lambda: lib.r4_s2s_epoch(c, P, P, P, P, P, P, P, n, Ts, Tt, P, n, n, 0, 0, 0, rate, 1e-3, 0.9,
                                                0.999, 1e-7, P, P, None),
              "predict": lambda: lib.r4_s2s_predict(c, P, P, P, n, Ts, Tt, P, P, None),
              "decode_step": lambda: lib.r4_s2s_decode_step(c, P, P, n, Ts, P, Tt, None, 0, k, P, P, P, None),
              "beam_search": lambda: lib.r4_s2s_beam_search(c, P, P, n, Ts, beam, tl, ncand, P, P, P, None),
              "score": lambda: lib.r4_s2s_score(c, P, P, n, Ts, P, sbeam, stl, P, P, None)}
        return [(f, fn[f]()) for f in names]

    ALL = ("num_params", "scratch train", "scratch search", "scratch step", "relu_offsets", "grad", "apply", "epoch",
           "predict", "decode_step", "beam_search", "score")
    TRAIN = ("scratch train", "relu_offsets", "grad", "epoch", "predict", "decode_step")
    SEARCH = ("scratch search", "beam_search")
    bad_cfg = {"E 544": (286, 286, 544, 1, 64, 1, 1, 0), "E 48": (286, 286, 48, 1, 64, 1, 1, 0),
               "F 1056": (286, 286, 64, 1, 1056, 1, 1, 0), "H 3 of E 64": (286, 286, 64, 3, 64, 1, 1, 0),
               "7 encoder blocks": (286, 286, 64, 1, 64, 7, 1, 0), "7 decoder blocks": (286, 286, 64, 1, 64, 1, 7, 0),
               "Vs 3": (3, 286, 64, 1, 64, 1, 1, 0), "Vt 3": (286, 3, 64, 1, 64, 1, 1, 0),
               "Vs 65537": (65537, 286, 64, 1, 64, 1, 1, 0), "Vt 65537": (286, 65537, 64, 1, 64, 1, 1, 0),
               "one shared table of two sizes": (286, 300, 64, 1, 64, 1, 1, 1)}
    out = []
    for what, t in bad_cfg.items():
        out += [("%s: %s" % (what, f), rc) for f, rc in calls(cfg(t), ALL)]
    c = cfg((286, 286, 64, 2, 64, 1, 1, 0))
    for T in (0, 65):
        out += [("src_len %d: %s" % (T, f), rc) for f, rc in calls(c, TRAIN + SEARCH + ("score",), Ts=T)]
        out += [("tgt_len %d: %s" % (T, f), rc) for f, rc in calls(c, TRAIN, Tt=T)]
        out += [("score target_len %d: %s" % (T, f), rc) for f, rc in calls(c, ("score",), stl=T)]
    for tl in (0, 64):
        out += [("search target_len %d: %s" % (tl, f), rc) for f, rc in calls(c, SEARCH, tl=tl)]
    out += [("n H 65536: %s" % f, rc) for f, rc in calls(c, TRAIN, n=32768)]                # H = 2
    c1 = cfg((200, 200, 64, 1, 64, 1, 1, 0))
    big = cfg((65536, 65536, 32, 1, 32, 1, 1, 1))
    out += [("beam 257: %s" % f, rc) for f, rc in calls(c1, SEARCH, beam=257)]
    out += [("beam 257: %s" % f, rc) for f, rc in calls(c1, ("score",), sbeam=257)]
    out += [("beam = V: %s" % f, rc) for f, rc in calls(c1, ("beam_search",), beam=200)]
    out += [("n beam H 65536: %s" % f, rc) for f, rc in calls(c1, SEARCH, n=256, beam=256)]
    out += [("n beam H 65536: %s" % f, rc) for f, rc in calls(c1, ("score",), n=256, sbeam=256)]
    out += [("candidates 8193: %s" % f, rc) for f, rc in calls(big, SEARCH, ncand=8193)]
    out += [("candidates = V: %s" % f, rc) for f, rc in calls(c1, ("beam_search",), ncand=200)]
    out += [("k = V: %s" % f, rc) for f, rc in calls(c1, ("decode_step",), k=200)]
    out += [("k 0: %s" % f, rc) for f, rc in calls(c1, ("decode_step", "scratch step"), k=0)]
    out += [("k 8193: %s" % f, rc) for f, rc in calls(big, ("decode_step", "scratch step"), k=8193)]
    out += [("candidates 8193: decode_step", lib.r4_s2s_decode_step(c1, P, P, 4, 5, P, 5, P, 8193, 4, P, P, P, None))]
    out += [("dropout 1.0: %s" % f, rc) for f, rc in calls(c, ("grad", "epoch"), rate=1.0)]
    return out
