"""A float64 restatement of Exact-K's generator and critic (nets/exact_k/model.py, layers.py, modules.py), written the way
the TF1 graph computes them: heads split along the last axis and stacked along the batch (tf.split / tf.concat), masks by
tf.where with the -2^32 + 1 padding, LayerNorm through the moments, the pointer-network decoder as call_cell / attention /
glimpse / intra_attention, and the policy loss through sparse softmax cross-entropy.  The tests hold the device kernels and
the torch twin to it.

Rows are independent except through the weight gradients, so the reference runs on any set of rows of a batch of n_total
(the draws are keyed by global row, the loss is divided by n_total) and its gradients add up.  `row0` is the first global
row of a contiguous slice, or an int64 tensor of the global rows themselves (a planted, non-contiguous set).

Also here: the mask regimes the shape tests run (masks_for), the all-masked step's rule, the chunking that keeps one
reference chunk at a few GB at any T, the reading of the kernels' relu decisions from the scratch, the TF1 Adam update
and the C-ABI rejections."""
import ctypes as C

import numpy as np
import torch

from rl4rs_b200 import exactk as ek

NEG = -2.0 ** 32 + 1


def _rows(row0, N, dev):
    if torch.is_tensor(row0):
        return row0.to(dev, torch.int64)
    return torch.arange(row0, row0 + N, dtype=torch.int64, device=dev)


def _keep(seed, call, stream, row0, m, per_row, shape, rate, dev):
    if rate <= 0:
        return torch.ones(shape, dtype=torch.float64, device=dev)
    e = (_rows(row0, m, dev).unsqueeze(1) * per_row + torch.arange(per_row, dtype=torch.int64, device=dev)).reshape(-1)
    u = ek.draw24(seed, call, stream, e).to(torch.float32) * (1.0 / 16777216.0)
    return ((u >= rate).to(torch.float64) / float(1.0 - np.float32(rate))).view(shape)


def _dense(x, w, b, act=None, keep=None):
    """x w + b; act "relu": relu, or, given keep (bool, the float32 run's relu decisions), y * keep."""
    y = torch.tensordot(x, w, dims=([x.dim() - 1], [0])) + b
    if act != "relu":
        return y
    return torch.relu(y) if keep is None else y * keep


def _normalize(x, beta, gamma):
    mean = x.mean(-1, keepdim=True)
    variance = x.var(-1, unbiased=False, keepdim=True)
    return gamma * ((x - mean) / ((variance + 1e-8) ** 0.5)) + beta


def _mha(x, w, p, seed, call, stream, row0, rate, keep=None):
    N, T, _ = x.shape
    Q, K, V = _dense(x, w[p + "qkv_w"], w[p + "qkv_b"], "relu", keep).split(128, -1)
    Q_, K_, V_ = (torch.cat(torch.split(t, 32, dim=2), 0) for t in (Q, K, V))      # (h*N, T, 32)
    out = Q_ @ K_.transpose(1, 2) / (32 ** 0.5)
    key_masks = torch.sign(torch.abs(x.sum(-1))).repeat(4, 1).unsqueeze(1).expand(-1, T, -1)
    out = torch.where(key_masks == 0, torch.full_like(out, NEG), out)
    out = torch.softmax(out, -1)
    query_masks = torch.sign(torch.abs(x.sum(-1))).repeat(4, 1).unsqueeze(-1)
    out = out * query_masks
    # dropout keyed by the kernel's (row, head, i, j) order; the reference graph's order is (head, row) -> permute
    keep = _keep(seed, call, stream, row0, N, 4 * T * T, (N, 4, T, T), rate, x.device).transpose(0, 1).reshape(4 * N, T, T)
    out = out * keep
    out = out @ V_
    out = torch.cat(torch.split(out, N, dim=0), 2)
    return _normalize(out + x, w[p + "ln1_b"], w[p + "ln1_g"])


def encoder(w, user, seed, call, rate, T, row0=0, relu_keep=None):
    """relu_keep (optional): {"u", "b0_qkv", "b0_f1", "b1_qkv", "b1_f1"} -> bool, the relu decisions to take instead
    of the float64 ones (a float32 run's, so that a pre-activation within roundoff of 0 takes the same branch)."""
    k = relu_keep or {}
    N = user.shape[0]
    enc_user = _dense(user, w["u_w"], w["u_b"], "relu", k.get("u"))
    enc_item = w["emb"][torch.arange(T, device=user.device)] * (64 ** 0.5)
    enc = torch.cat([torch.stack(T * [enc_user], 1), enc_item.unsqueeze(0).expand(N, T, 64)], 2)
    enc = enc * _keep(seed, call, ek.ST_INPUT, row0, N, T * 128, (N, T, 128), rate, user.device)
    for i in range(2):
        p = "b%d_" % i
        enc = _mha(enc, w, p, seed, call, ek.ST_ATT0 + i, row0, rate, k.get(p + "qkv"))
        ff = _dense(_dense(enc, w[p + "f1_w"], w[p + "f1_b"], "relu", k.get(p + "f1")), w[p + "f2_w"], w[p + "f2_b"])
        enc = _normalize(ff + enc, w[p + "ln2_b"], w[p + "ln2_g"])
    return enc


def dead_pick(mode, seed, call, rows, t, T, temperature):
    """The choice at an all-masked step (every logit -2^32 + 1): GREEDY takes candidate 0 (the first of the equal
    maxima); SAMPLE is the uniform inverse CDF, the first j with j + 1 >= u T, with u T formed in float32 as the kernel
    forms it (exact: the running sum of T ones is exact in float32), so no margin applies."""
    if mode == ek.GREEDY:
        return torch.zeros(rows.shape[0], dtype=torch.int64, device=rows.device)
    bits = ek.draw24(seed, call, ek.ST_SAMPLE, rows * 9 + t)
    u = (bits.float() + 0.5) * np.float32(1.0 / 16777216.0) * np.float32(T)
    return (torch.ceil(u.double()).long() - 1).clamp(0, T - 1)


def decoder(w, enc, masks, mode, seed, call, target=None, temperature=1.0, row0=0, dead_out=None):
    """ptn_rnn_decoder: -> (logits [N, 9, T], path [N, 9], margins [N] float64: the smallest decision margin of each row
    (GREEDY: top-2 logit gap; SAMPLE: distance of the draw to a CDF edge, relative to the total)).  A step whose point
    mask is empty is its own kind of decision: it takes dead_pick's rule and adds no margin; dead_out (a list), if given,
    receives the [N, 9] bool of those steps."""
    N, T, _ = enc.shape
    refs = {a: torch.tensordot(enc, w[a + "_w_ref"], dims=([2], [0])) for a in ("g", "p")}

    def attention(a, query, dec_ref, with_softmax):
        scores = (w[a + "_v"] * torch.tanh(refs[a] + (query @ w[a + "_w_q"]).unsqueeze(1) +
                                           (dec_ref @ w[a + "_w_dec"]).unsqueeze(1) + w[a + "_bias"])).sum(-1)
        return torch.softmax(scores, -1) if with_softmax else scores

    def intra_attention(bef, query):
        if len(bef) == 0:
            return torch.zeros(N, 128, dtype=enc.dtype, device=enc.device)
        if len(bef) == 1:
            return bef[0]
        bef = torch.stack(bef, 1)
        scores = (w["v_dec"] * torch.tanh(torch.tensordot(bef, w["w_bef"], dims=([2], [0])) +
                                          (query @ w["w_b"]).unsqueeze(1) + w["bias_dec"])).sum(-1)
        return (torch.softmax(scores, 1).unsqueeze(2) * bef).sum(1)

    state = (w["c0"].expand(N, 128), w["h0"].expand(N, 128))
    output_ref, logits_all, idxs = [], [], []
    margins = torch.full((N,), float("inf"), dtype=torch.float64, device=enc.device)
    rows = torch.arange(N, device=enc.device)
    grows = _rows(row0, N, enc.device)
    dead = torch.zeros(N, 9, dtype=torch.bool, device=enc.device)
    inp = w["x0"].expand(N, 128)
    path = torch.zeros(N, 9, dtype=torch.int64, device=enc.device)
    for i in range(9):
        c, h = state
        lstm = torch.cat([inp, h], 1) @ w["lstm_w"] + w["lstm_b"]
        gi, gj, gf, go = torch.split(lstm, 128, 1)
        c = torch.sigmoid(gf + 1.0) * c + torch.sigmoid(gi) * torch.tanh(gj)
        h = torch.sigmoid(go) * torch.tanh(c)
        state = (c, h)
        intra = intra_attention(output_ref, h)
        output_ref.append(h)
        glimpse = (attention("g", h, intra, True).unsqueeze(2) * enc).sum(1)
        logits = attention("p", glimpse, intra, False)
        pm = ek.point_masks(masks, path, i)
        logits = torch.where(pm, logits, torch.full_like(logits, NEG))
        logits_all.append(logits)
        lg = logits.detach()
        dead[:, i] = ~pm.any(1)
        inf = torch.full_like(margins, float("inf"))
        if mode == ek.TRAIN:
            idx = target[:, i].long()
        elif mode == ek.GREEDY:
            top = lg.topk(2, 1)
            idx = top.indices[:, 0]
            margins = torch.minimum(margins, torch.where(dead[:, i], inf, top.values[:, 0] - top.values[:, 1]))
        else:
            x = lg / temperature
            e = torch.exp(x - x.max(1, keepdim=True).values)
            cdf = torch.cumsum(e, 1) / e.sum(1, keepdim=True)
            bits = ek.draw24(seed, call, ek.ST_SAMPLE, grows * 9 + i)
            u = ((bits.double() + 0.5) / 16777216.0).unsqueeze(1)
            idx = (cdf < u).sum(1)
            last = T - 1 - torch.flip(e > 0, [1]).int().argmax(1)
            idx = torch.where(idx < T, idx.clamp(max=T - 1), last)
            margins = torch.minimum(margins, torch.where(dead[:, i], inf, (cdf - u).abs().min(1).values))
        if mode != ek.TRAIN:
            idx = torch.where(dead[:, i], dead_pick(mode, seed, call, grows, i, T, temperature), idx)
        path[:, i] = idx
        idxs.append(idx)
        inp = enc[rows, idx]
    if dead_out is not None:
        dead_out.append(dead)
    return torch.stack(logits_all, 1), path, margins


def mask_margin(w, user, seed, call, rate, T, row0=0):
    """The smallest |sum_c X| / max|X| over the tokens entering both blocks, per row (the key / query mask decision)."""
    with torch.no_grad():
        N = user.shape[0]
        enc_user = _dense(user, w["u_w"], w["u_b"], "relu")
        enc = torch.cat([torch.stack(T * [enc_user], 1), (w["emb"][:T] * 8.0).unsqueeze(0).expand(N, T, 64)], 2)
        enc = enc * _keep(seed, call, ek.ST_INPUT, row0, N, T * 128, (N, T, 128), rate, user.device)
        out = torch.full((N,), float("inf"), dtype=torch.float64, device=user.device)
        for i in range(2):
            out = torch.minimum(out, (enc.sum(-1).abs() / enc.abs().amax(-1).clamp_min(1e-30)).min(1).values)
            p = "b%d_" % i
            enc = _mha(enc, w, p, seed, call, ek.ST_ATT0 + i, row0, rate)
            ff = _dense(_dense(enc, w[p + "f1_w"], w[p + "f1_b"], "relu"), w[p + "f2_w"], w[p + "f2_b"])
            enc = _normalize(ff + enc, w[p + "ln2_b"], w[p + "ln2_g"])
        return out


def generator_grad(flat, user, masks, target, reward, seed, call, rate, row0=0, n_total=None, relu_keep=None):
    """float64 autograd of the policy loss sum_b(sum_t CE(logits[b, t], target[b, t]) reward[b]) / n_total over the rows
    of user -> (grad [num_params], loss, logits).  relu_keep: as encoder's."""
    n_total = n_total or user.shape[0]
    flat = flat.detach().double().clone().requires_grad_(True)
    w = ek.unflatten(flat, ek.generator_shapes())
    T = masks.shape[1]
    enc = encoder(w, user.double(), seed, call, rate, T, row0, relu_keep)
    logits, _, _ = decoder(w, enc, masks, ek.TRAIN, seed, call, target=target, row0=row0)
    r_loss = -torch.log_softmax(logits, -1).gather(2, target.long().unsqueeze(2)).squeeze(2)
    loss = (r_loss.sum(1) * reward.double()).sum() / n_total
    loss.backward()
    return flat.grad.detach(), loss.detach(), logits.detach()


def critic(flat, user, target=None):
    """-> (pred, grad of sum (target - pred)^2 or None, loss or None) in float64."""
    flat = flat.detach().double().clone().requires_grad_(target is not None)
    w = ek.unflatten(flat, ek.critic_shapes())
    d = user.double()
    for i in (1, 2, 3):
        d = torch.relu(d @ w["w%d" % i] + w["b%d" % i])
    pred = (d @ w["w4"] + w["b4"])[:, 0]
    if target is None:
        return pred.detach(), None, None
    loss = torch.square(torch.abs(target.double() - pred)).sum()
    loss.backward()
    return pred.detach(), flat.grad.detach(), loss.detach()


# ---- what the shape tests run ------------------------------------------------------------------------------------------
MASK_REGIMES = ("ones", "slate", "sparse")


def masks_for(T, regime, device="cpu"):
    """u8 [4, T]: the location masks of positions 0-2, 3-5, 6-8 and the special items.
      ones    every candidate at every position, no special item
      slate   SlateState._location_mask(T) with the synthetic catalog's special items below T (below T = 41 positions
              3-8 have no candidate, below 149 positions 6-8 have none: all-masked steps of the env's own masks)
      sparse  positions 0-5 take every candidate; positions 6-8 take three special items (the last three candidates) and
              one other (candidate 0).  A slate holds one special item at most, so positions 6-8 can fill two of their
              three places: every row meets an all-masked step by position 8, earlier when it chose a special item first."""
    m = np.zeros((4, T))
    if regime == "ones":
        m[:3] = 1
    elif regime == "slate":
        from rl4rs_b200 import synth
        from rl4rs_b200.env.slate import SlateState
        m[:3] = SlateState._location_mask(T)[:3]
        m[3, [int(x) for x in synth.make_catalog().special_items if int(x) < T]] = 1
    elif regime == "sparse":
        m[:2] = 1
        m[3, T - 3:] = 1
        m[2, T - 3:] = 1
        m[2, 0] = 1
    else:
        raise ValueError(regime)
    return torch.tensor(m != 0, dtype=torch.uint8, device=device)


# one [m, 4, T, T] float64 plane per chunk at most this many bytes (autograd holds about a dozen of them per block)
PLANE_BYTES = 1 << 27


def chunk_rows(T):
    return int(max(1, min(128, PLANE_BYTES // (32 * T * T))))


def chunks(rows, T):
    """Split a sorted int64 row tensor into reference chunks of chunk_rows(T) rows."""
    c = chunk_rows(T)
    return [rows[i:i + c] for i in range(0, rows.numel(), c)]


def ref_decode(flat, user, masks, mode, seed, call, rate, temperature=1.0, rows=None):
    """The reference's SAMPLE / GREEDY decode of the global rows `rows` (default: all of user's), chunked:
    -> (path [m, 9], margins [m], mask margins [m], dead [m, 9] bool)."""
    T = masks.shape[1]
    w = unflat64(flat)
    rows = torch.arange(user.shape[0], device=user.device) if rows is None else rows.to(user.device)
    out = [[], [], [], []]
    for r in chunks(rows, T):
        u = user[r].double()
        dead = []
        with torch.no_grad():
            enc = encoder(w, u, seed, call, rate, T, r)
            _, p, mg = decoder(w, enc, masks, mode, seed, call, temperature=temperature, row0=r, dead_out=dead)
        for k, v in enumerate((p, mg, mask_margin(w, u, seed, call, rate, T, r), dead[0])):
            out[k].append(v)
    return tuple(torch.cat(v) for v in out)


def unflat64(flat):
    return ek.unflatten(flat.detach().double(), ek.generator_shapes())


def device_relu_decisions(g, n):
    """The relu decisions of the kernels' last forward over n rows of generator g, read from the activation planes at
    the head of the scratch (the order include/rl4rs_b200.h documents for r4_exactk_grad), at g.T candidates:
    {"u", "b0_qkv", "b0_f1", "b1_qkv", "b1_f1"} -> bool."""
    T = g.T
    f = g._scr(n).view(torch.float32)
    nT, S4, o, out = n * T, n * 4 * T * T, 0, {}

    def take(k, shape=None):
        nonlocal o
        plane = f[o:o + k]
        o += (k + 63) // 64 * 64
        return None if shape is None else plane.view(shape) > 0

    out["u"] = take(n * 64, (n, 64))
    take(nT * 128)
    for l in range(2):
        take(nT)
        out["b%d_qkv" % l] = take(nT * 384, (n, T, 384))
        for k in (S4, S4, nT * 128, nT * 128, nT * 128, nT):
            take(k)
        out["b%d_f1" % l] = take(nT * 256, (n, T, 256))
        for k in (nT * 128, nT * 128, nT):
            take(k)
    return out


def grad_rows(flat, user, masks, target, reward, seed, call, rate, rows, n_total, relu_keep=None):
    """generator_grad summed over the chunks of the global rows `rows` (user, target, reward, relu_keep indexed by
    global row) -> (grad, loss, [(rows, logits)])."""
    T = masks.shape[1]
    grad, loss, logits = 0, 0.0, []
    for r in chunks(rows, T):
        keep = None if relu_keep is None else {k: v[r] for k, v in relu_keep.items()}
        gr, l, lg = generator_grad(flat, user[r], masks, target[r], reward[r], seed, call, rate, row0=r, n_total=n_total,
                                   relu_keep=keep)
        grad = grad + gr
        loss += float(l)
        logits.append((r, lg))
    return grad, loss, logits


def tensor_errors(got, want, shapes=None):
    """{tensor name: (max err, max |ref|)} over the flat layout of the generator (or shapes)."""
    shapes = shapes or ek.generator_shapes()
    a, b = ek.unflatten(got.double(), shapes), ek.unflatten(want.double().to(got.device), shapes)
    return {k: ((a[k] - b[k]).abs().max().item(), b[k].abs().max().item()) for k in a}


def adam64(flat, grad, m, v, step, lr, beta1=0.9, beta2=0.98, eps=1e-8):
    """TF1 AdamOptimizer (ResourceApplyAdam) in float64: -> (params, m, v) after step `step` (1-based)."""
    flat, grad, m, v = (x.double() for x in (flat, grad, m, v))
    alpha = lr * (1 - beta2 ** step) ** 0.5 / (1 - beta1 ** step)
    m = m + (grad - m) * (1 - beta1)
    v = v + (grad * grad - v) * (1 - beta2)
    return flat - alpha * m / (v.sqrt() + eps), m, v


def abi_rejections(lib, P):
    """[(label, rc)] of the r4_exactk_* entry points called one step past each edge their arguments accept, and of
    r4_exactk_scratch_size at each shape edge.  P: a non-NULL address passed for every buffer; each call is refused on
    the host before anything is read or launched, so P is never dereferenced.  Every rc must be R4_ERR_ARG (-1), and
    every scratch size -1."""
    nan = float("nan")
    cap_T500 = ek.MAX_NTT // (500 * 500) + 1            # the first n past n T^2 <= 4096 * 284^2 at T = 500
    base = dict(params=P, user=P, n=7, T=32, masks=P, mode=ek.SAMPLE, temperature=1.0, dropout=0.1, path=P, logits=P,
                target=P, reward=P, grad=P, loss=P, scratch=P)

    def decode(a):
        return lib.r4_exactk_decode(a["params"], a["user"], a["n"], a["T"], a["masks"], a["mode"], a["temperature"], 3, 1,
                                    a["dropout"], a["path"], a["logits"], a["scratch"], None)

    def grad(a):
        return lib.r4_exactk_grad(a["params"], a["user"], a["n"], a["T"], a["masks"], a["target"], a["reward"], 3, 1,
                                  a["dropout"], a["grad"], a["loss"], a["scratch"], None)

    shape_edges = [dict(n=0), dict(n=4097), dict(T=8), dict(T=501), dict(n=cap_T500, T=500), dict(n=4096, T=285)]
    out = []
    for e in shape_edges + [dict(dropout=-1e-7), dict(dropout=1.0), dict(dropout=nan)]:
        for name, fn in (("decode", decode), ("grad", grad)):
            out.append(("%s %s" % (name, e), fn(dict(base, **e))))
    for e in (dict(temperature=0.0), dict(temperature=-1.0), dict(temperature=nan), dict(mode=-1), dict(mode=3)):
        out.append(("decode %s" % e, decode(dict(base, **e))))
    for k in ("params", "user", "masks", "path", "scratch"):
        out.append(("decode %s NULL" % k, decode(dict(base, **{k: None}))))
    for k in ("params", "user", "masks", "target", "reward", "grad", "scratch"):
        out.append(("grad %s NULL" % k, grad(dict(base, **{k: None}))))
    for e in shape_edges:
        a = dict(base, **e)
        out.append(("scratch_size generator %s" % e, lib.r4_exactk_scratch_size(ek.GENERATOR, a["n"], a["T"])))
    for n in (0, 4097):
        out.append(("scratch_size critic n=%d" % n, lib.r4_exactk_scratch_size(ek.CRITIC, n, 0)))
        out.append(("critic n=%d" % n, lib.r4_exactk_critic(P, P, n, P, P, P, P, P, None)))
    out.append(("scratch_size net 2", lib.r4_exactk_scratch_size(2, 7, 32)))
    crit = dict(params=P, user=P, target=P, pred=P, grad=P, loss=P, scratch=P)
    for k in ("params", "user", "scratch"):
        a = dict(crit, **{k: None})
        out.append(("critic %s NULL" % k, lib.r4_exactk_critic(a["params"], a["user"], 7, a["target"], a["pred"], a["grad"],
                                                                a["loss"], a["scratch"], None)))
    out.append(("critic target without grad", lib.r4_exactk_critic(P, P, 7, P, P, None, P, P, None)))
    adam = dict(net=ek.CRITIC, params=P, grad=P, m=P, v=P, step=1)
    for e in (dict(net=2), dict(net=-1), dict(step=0), dict(params=None), dict(grad=None), dict(m=None), dict(v=None)):
        a = dict(adam, **e)
        out.append(("adam %s" % e, lib.r4_exactk_adam(a["net"], a["params"], a["grad"], a["m"], a["v"], a["step"], 1e-3, 0.9,
                                                      0.98, 1e-8, None)))
    return out
