"""Shared by the slate-head training tests: slate samples with teacher labels, the float64 autograd reference of the slate
heads' gradient (SimulatorNet with head 1 / 2 on a float64 copy of the flat parameters), the batch compacted to the ids it
touches, and a restatement of the slate heads' parameter count and scratch layout."""
import numpy as np
import torch

import simtrain_ref as R
from rl4rs_b200 import simtrain

HEADS = (1, 2)
NAMES = {1: "dien_slate", 2: "dien_slate_multiclass"}


def cfg(H, head):
    return {"category_hash_size": H, "class_num": simtrain.CLASSES[head]}


def make_samples(n_records, hash_size, seed=0, edge=False):
    s = R.make_edge_samples(n_records, hash_size, seed=seed) if edge else R.make_samples(n_records, hash_size, seed=seed)
    return simtrain.SlateSamples.view(s)


def make_weights(H, head, kind="default"):
    c = cfg(H, head)
    if kind == "default":
        return simtrain.head_weights(c, head, seed=21, bounded_scores=True)
    return simtrain.head_weights(c, head, seed=22, stress=2.0, bias_noise=0.1, bounded_scores=True)


def teacher_labels(samples, H, seed=7, stress=3.0, label_seed=1, draw=True):
    """Replace the clicks by draws from a teacher dien_slate's 9 column probabilities (float64 twin, no dropout), or
    with draw=False by the teacher's decisions p > 0.5 (a click pattern the features determine)."""
    c = cfg(H, 1)
    w = simtrain.head_weights(c, 1, seed=seed, stress=stress, bias_noise=0.2, bounded_scores=True)
    net = simtrain.SimulatorNet(c, simtrain.flatten(w, c), torch.float64, head=1)
    p = []
    with torch.no_grad():
        for b in range(0, len(samples), 512):
            cat, dense, seq, _ = samples.features(np.arange(b, min(len(samples), b + 512)))
            p.append(net(cat, dense, seq)[0].numpy())
    p = np.concatenate(p)
    u = np.random.RandomState(label_seed).random_sample(p.shape) if draw else np.full(p.shape, 0.5)
    samples.feedback = (u < p).astype(np.uint8)
    return p


def ref_grad(head, config, flat, samples, idx, keep=None, rate=simtrain.DROPOUT, device="cpu", chunk=512):
    """float64 autograd of the head's mean loss at flat over the records idx -> (loss, grad f64[np], probs f64[n, C])."""
    idx = np.asarray(idx, np.int64)
    n = len(idx)
    net = simtrain.SimulatorNet(config, np.asarray(flat, np.float64), torch.float64, head=head).to(device)
    loss, probs = 0.0, []
    for b in range(0, n, chunk):
        cat, dense, seq, y = samples.features(idx[b:b + chunk])
        z, _ = net.logits(cat, dense, seq, None if keep is None else keep[b:b + chunk], rate)
        lc = simtrain.loss_rows(head, z, y).sum() / n
        lc.backward()
        loss += float(lc.detach())
        probs.append((torch.sigmoid(z) if head == 1 else torch.softmax(z, -1)).detach().cpu().numpy())
    return loss, net.flat.grad.cpu().numpy(), np.concatenate(probs)


@torch.no_grad()
def ref_probs(head, config, flat, samples, idx, device="cpu", chunk=2048):
    idx = np.asarray(idx, np.int64)
    net = simtrain.SimulatorNet(config, np.asarray(flat, np.float64), torch.float64, head=head).to(device)
    return np.concatenate([net(*samples.features(idx[b:b + chunk])[:3])[0].cpu().numpy() for b in range(0, len(idx), chunk)])


def compact(samples, idx):
    """R.compact for slate samples: the records idx over the ids they read, the pad id 0 (cat slot 20, a query slot)
    included -> (ids, SlateSamples', idx')."""
    idx = np.asarray(idx, np.int64)
    recs, inv = np.unique(idx, return_inverse=True)
    ids = np.unique(np.concatenate([[0], samples.user_cat[recs].ravel(), samples.sequence_id[recs], samples.items[recs].ravel(),
                                    samples.seq[recs].ravel()]).astype(np.int64))

    def remap(a):
        return np.searchsorted(ids, a).astype(np.int32)
    s = simtrain.SlateSamples(
        len(ids), user_cat=remap(samples.user_cat[recs]), user_dense=samples.user_dense[recs],
        sequence_id=remap(samples.sequence_id[recs]), items=remap(samples.items[recs]), feedback=samples.feedback[recs],
        item_feature=samples.item_feature[recs], seq=remap(samples.seq[recs]))
    return ids, s, inv.astype(np.int64)


def num_params(H, head):
    return sum(int(np.prod(s)) for _, s in simtrain.layer_plan(cfg(H, head)))


def scratch_cuts(n, head):
    """R.scratch_cuts with the head's logits planes Z and dZ ([n][C]) in place of the item head's [n][2]."""
    cuts = R.scratch_cuts(n)
    cuts[10] = cuts[11] = n * simtrain.CLASSES[head]
    return cuts


def scratch_bytes(n, head):
    return sum((4 * k + 255) // 256 * 256 for k in scratch_cuts(n, head)) + R.cub_reserve(n)


def host_metrics(head, probs, labels, loss_rows):
    m = simtrain.METRICS[head]()
    m.add(probs, labels, loss_rows)
    return m

