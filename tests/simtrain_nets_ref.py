"""Shared by the backbone training tests (dnn, widedeep, lstm, adversarial_slate): the valid (net, head) pairs, weights,
samples, the float64 autograd reference of a pair's gradient (the torch twin on a float64 copy of the flat parameters, with
the lstm kink margin), and a restatement of each net's parameter count and scratch layout."""
import numpy as np
import torch

import simtrain_ref as R
import simtrain_slate_ref as SR
from rl4rs_b200 import simtrain

NETS = (1, 2, 3, 4)
PAIRS = [(net, head) for net in (1, 2, 3) for head in (0, 1, 2)] + [(4, 3)]
NAMES = {(net, head): simtrain.NET_NAMES[net] + ("", "_slate", "_slate_multiclass")[head] for net in (1, 2, 3) for head in (0, 1, 2)}
NAMES[(4, 3)] = "adversarial_slate"
# the lstm parity cases hold only where every hard-sigmoid argument is this far from a kink (in float64): closer, the f32
# kernel and the f64 reference may sit on different sides of it and take different slopes
KINK_MARGIN = 1e-5


def cfg(H, head):
    return {"category_hash_size": H, "class_num": simtrain.CLASSES[head]}


def make_samples(n_records, H, head, seed=0, edge=False):
    s = R.make_edge_samples(n_records, H, seed=seed) if edge else R.make_samples(n_records, H, seed=seed)
    return simtrain.SlateSamples.view(s) if head else s


def make_weights(net, H, head, kind="default"):
    """default: Keras initialisers; stress: kernels x2 and bias noise 0.1; saturate (lstm): GRU kernels x2.5 and biases
    N(0, 1.5), which clips about a quarter of the gates."""
    c = cfg(H, head)
    if kind == "default":
        return simtrain.net_weights(c, net, head, seed=21)
    if kind == "saturate":
        return simtrain.net_weights(c, net, head, seed=23, gru_stress=2.5, gru_bias_noise=1.5)
    return simtrain.net_weights(c, net, head, seed=22, stress=2.0, bias_noise=0.1)


def compact(samples, idx, head):
    return SR.compact(samples, idx) if head else R.compact(samples, idx)


def compact_weights(w, ids):
    return dict(w, **{k: w[k][ids] for k in ("emb_cat", "emb_seq") if k in w})


def _loss_rows(head, z, y):
    if head:
        return simtrain.loss_rows(head, z, y)
    p = torch.softmax(z, -1)
    yy = torch.nn.functional.one_hot(torch.as_tensor(y, device=z.device), 2).to(z.dtype)
    pc = p.clamp(simtrain.CLIP, 1.0 - simtrain.CLIP)
    return -(yy * torch.log(pc) + (1.0 - yy) * torch.log(1.0 - pc)).mean(1)


def ref_grad(net, head, config, flat, samples, idx, keep=None, rate=simtrain.DROPOUT, device="cpu", chunk=512):
    """float64 autograd of the pair's mean loss at flat over the samples idx -> (loss, grad f64[np], probs f64[n, C],
    margin: the smallest distance of an lstm hard-sigmoid argument from a kink, inf for the other nets)."""
    idx = np.asarray(idx, np.int64)
    n = len(idx)
    tw = simtrain.twin(config, net, np.asarray(flat, np.float64), torch.float64, head=head).to(device)
    loss, probs, margin = 0.0, [], np.inf
    for b in range(0, n, chunk):
        cat, dense, seq, y = samples.features(idx[b:b + chunk])
        z, _ = tw.logits(cat, dense, seq, None if keep is None else keep[b:b + chunk], rate)
        margin = min(margin, getattr(tw, "margin", np.inf))
        lc = _loss_rows(head, z, y).sum() / n
        lc.backward()
        loss += float(lc.detach())
        probs.append((torch.sigmoid(z) if head in (1, 3) else torch.softmax(z, -1)).detach().cpu().numpy())
    return loss, tw.flat.grad.cpu().numpy(), np.concatenate(probs), margin


@torch.no_grad()
def ref_probs(net, head, config, flat, samples, idx, device="cpu", chunk=1024):
    idx = np.asarray(idx, np.int64)
    tw = simtrain.twin(config, net, np.asarray(flat, np.float64), torch.float64, head=head).to(device)
    return np.concatenate([tw(*samples.features(idx[b:b + chunk])[:3])[0].cpu().numpy() for b in range(0, len(idx), chunk)])


def num_params(net, H, head):
    return sum(int(np.prod(s)) for _, s in simtrain.layer_plan(cfg(H, head), net))


def scratch_cuts(net, n, head):
    """The planes r4st::make_nplanes cuts, in floats, in order."""
    C = simtrain.CLASSES[head]
    FA = {1: 256, 2: 256, 3: 3200, 4: 512}[net]
    FO = {1: 256, 2: 3072, 3: 256, 4: 0}[net]
    cuts = [n * 21, n * 432, n * 256, n * 128, n * 128, n * 128, n * FA, n * FA]
    if net in (1, 2):
        cuts += [n * 256, n * 256]
    if FO:
        cuts += [n * FO, n * FO]
    cuts += [n * C, n * C, n * 128, n * 128, n * 21 * 128, n * 2]
    if net != 1:
        cuts += [n * 64 * 128] * 2
    if net == 3:
        for nt in (21, 64, 64):
            r = n * nt
            cuts += [r * 128, r * 384, r * 128, r * 256, r * 128, r * 128, r * 256, r * 128]
        cuts += [3 * 257 * 384]
    ns = nslots(net)
    return cuts + [n * ns] * 4


def nslots(net):
    return {1: 21, 2: 21 + 128, 3: 21 + 128, 4: 20 + 128}[net]


def scratch_bytes(net, n, head):
    return sum((4 * k + 255) // 256 * 256 for k in scratch_cuts(net, n, head)) + (4 << 20) + 16 * n * nslots(net)
