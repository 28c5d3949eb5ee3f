"""A float64 autograd reference for the MDP checker's transformer: the restatement in rl4rs_b200/mdpchecker/transformer.py
(forward, loss_fn) run in float64 on the CPU, with the same dropout draws, so the kernels' gradients are held to it
tensor by tensor.  relu_keep hands it the kernels' relu decisions (a pre-activation within roundoff of 0 could otherwise
be decided differently in float32 and float64)."""
import numpy as np
import torch

from rl4rs_b200.mdpchecker import transformer as tf

CLIP = 1e-7


def grad64(flat, cfg, enc, dec, target, seed=0, call=0, rate=0.0, relu_keep=None):
    """(loss, flat gradient, probabilities [n, Tt, Vt]) in float64 at the float32 weights flat."""
    p = flat.detach().cpu().double().requires_grad_(True)
    enc, dec, target = (torch.as_tensor(np.asarray(a), dtype=torch.int64) for a in (enc, dec, target))
    keep = None if relu_keep is None else [torch.as_tensor(k, dtype=torch.float64) for k in relu_keep]
    logits = tf.forward(tf.unflatten(p, cfg), cfg, enc, dec, seed, call, rate, relu_keep=keep)
    loss = tf.loss_fn(logits, dec, target)
    loss.backward()
    return float(loss.detach()), p.grad.detach(), torch.softmax(logits.detach(), -1).numpy()


def clip_edge_rows(probs, dec, rel=1e-3):
    """Loss positions (decoder input != 0) holding a probability within rel of a clip edge (1e-7 or 1 - 1e-7), where
    float32 and float64 may pass or stop the gradient differently."""
    near = (np.abs(probs - CLIP) < rel * CLIP) | (np.abs(probs - (1 - CLIP)) < rel * CLIP)
    return int((near.any(-1) & (np.asarray(dec) != 0)).sum())


def probs64(flat, cfg, enc, dec):
    with torch.no_grad():
        w = tf.unflatten(flat.detach().cpu().double(), cfg)
        enc, dec = (torch.as_tensor(np.asarray(a), dtype=torch.int64) for a in (enc, dec))
        return torch.softmax(tf.forward(w, cfg, enc, dec), -1).numpy()
