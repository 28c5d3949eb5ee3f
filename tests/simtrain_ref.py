"""Shared by the simulator-training tests: synthetic item samples with teacher labels, and the float64 autograd reference of
the kernels' gradient (the torch twin SimulatorNet on a float64 copy of the flat parameters, as learner_ref64.py does for the
learners)."""
import numpy as np
import torch

from rl4rs_b200 import simtrain, synth


def make_samples(n_records, hash_size, seed=0, pages=True):
    """ItemSamples of n_records random page records: ids in [0, hash_size), histories of 1..80 ids (pre-padded), page numbers
    1..4 with the earlier pages' items as the second sequence."""
    rs = np.random.RandomState(seed)
    N = n_records
    seq = np.zeros((N, 2, 64), np.int32)
    sid = rs.randint(1, 5, N).astype(np.int32) if pages else np.ones(N, np.int32)
    for r in range(N):
        L = rs.randint(1, 81)
        h = rs.randint(1, hash_size, L)[-64:]
        seq[r, 0, 64 - len(h):] = h
        k = 9 * (sid[r] - 1)
        if k:
            seq[r, 1, 64 - k:] = rs.randint(1, hash_size, k)
    return simtrain.ItemSamples(
        hash_size, user_cat=rs.randint(0, hash_size, (N, 10)).astype(np.int32),
        user_dense=np.round(np.maximum(0.0, rs.normal(1.0, 1.0, (N, 32))), 3).astype(np.float32),
        sequence_id=sid, items=rs.randint(1, hash_size, (N, 9)).astype(np.int32),
        feedback=(rs.random_sample((N, 9)) < 0.35).astype(np.uint8),
        item_feature=np.round(rs.normal(0.0, 1.0, (N, 360)), 4).astype(np.float32), seq=seq)


def teacher_labels(samples, config, seed=7, stress=3.0, label_seed=1):
    """Replace the labels by draws from a teacher DIEN's click probabilities (float64 twin, no dropout)."""
    w = synth.make_weights(config, seed=seed, stress=stress, bias_noise=0.2, bounded_scores=True)
    net = simtrain.SimulatorNet(config, simtrain.flatten(w, config), torch.float64)
    idx = np.arange(len(samples))
    p = []
    with torch.no_grad():
        for b in range(0, len(idx), 512):
            cat, dense, seq, _ = samples.features(idx[b:b + 512])
            p.append(net(cat, dense, seq)[0][:, 1].numpy())
    p = np.concatenate(p)
    rs = np.random.RandomState(label_seed)
    samples.feedback = (rs.random_sample(p.shape) < p).astype(np.uint8).reshape(-1, 9)
    return p


def ref_grad(config, flat, samples, idx, keep=None, rate=simtrain.DROPOUT):
    """float64 autograd of the mean loss at flat over samples idx -> (loss, grad f64[np], probs f64[n, 2])."""
    net = simtrain.SimulatorNet(config, np.asarray(flat, np.float64), torch.float64)
    cat, dense, seq, y = samples.features(idx)
    probs, _ = net(cat, dense, seq, keep, rate)
    loss = simtrain.keras_bce(probs, y)
    loss.backward()
    return float(loss.detach()), net.flat.grad.numpy().copy(), probs.detach().numpy()


def constant_loss(labels):
    """The loss of the best constant predictor (the label mean)."""
    m = float(np.mean(labels))
    return -(m * np.log(m) + (1 - m) * np.log(1 - m))
