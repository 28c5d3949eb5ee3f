"""A float64 restatement of Exact-K's generator and critic (nets/exact_k/model.py, layers.py, modules.py), written the way
the TF1 graph computes them: heads split along the last axis and stacked along the batch (tf.split / tf.concat), masks by
tf.where with the -2^32 + 1 padding, LayerNorm through the moments, the pointer-network decoder as call_cell / attention /
glimpse / intra_attention, and the policy loss through sparse softmax cross-entropy.  The tests hold the device kernels and
the torch twin to it.

Rows are independent except through the weight gradients, so the reference runs on any slice of rows [row0, row0 + m) of
a batch of n_total (the draws are keyed by global row, the loss is divided by n_total) and its gradients add up."""
import numpy as np
import torch

from rl4rs_b200 import exactk as ek

NEG = -2.0 ** 32 + 1


def _keep(seed, call, stream, row0, m, per_row, shape, rate, dev):
    if rate <= 0:
        return torch.ones(shape, dtype=torch.float64, device=dev)
    e = torch.arange(row0 * per_row, (row0 + m) * per_row, dtype=torch.int64, device=dev)
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


def decoder(w, enc, masks, mode, seed, call, target=None, temperature=1.0, row0=0):
    """ptn_rnn_decoder: -> (logits [N, 9, T], path [N, 9], margins [N] float64: the smallest decision margin of each row
    (GREEDY: top-2 logit gap; SAMPLE: distance of the draw to a CDF edge, relative to the total))."""
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
        logits = torch.where(ek.point_masks(masks, path, i), logits, torch.full_like(logits, NEG))
        logits_all.append(logits)
        lg = logits.detach()
        if mode == ek.TRAIN:
            idx = target[:, i].long()
        elif mode == ek.GREEDY:
            top = lg.topk(2, 1)
            idx = top.indices[:, 0]
            margins = torch.minimum(margins, top.values[:, 0] - top.values[:, 1])
        else:
            x = lg / temperature
            e = torch.exp(x - x.max(1, keepdim=True).values)
            cdf = torch.cumsum(e, 1) / e.sum(1, keepdim=True)
            bits = ek.draw24(seed, call, ek.ST_SAMPLE, (torch.arange(N, device=enc.device) + row0) * 9 + i)
            u = ((bits.double() + 0.5) / 16777216.0).unsqueeze(1)
            idx = (cdf < u).sum(1)
            last = T - 1 - torch.flip(e > 0, [1]).int().argmax(1)
            idx = torch.where(idx < T, idx.clamp(max=T - 1), last)
            margins = torch.minimum(margins, (cdf - u).abs().min(1).values)
        path[:, i] = idx
        idxs.append(idx)
        inp = enc[rows, idx]
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
