"""Float64 restatements of the learners' optimiser steps, and the fp32 rounding bounds the GPU tests hold them to.

Every rule takes the float32 inputs and the float32 values of its hyper-parameters (the C-ABI takes them as float, so a
learning rate of 1e-3 is float32(1e-3) on both sides) and computes in float64:

  adam            torch.optim.Adam as csrc/r4_ppo.cuh adam_update documents it: m = b1 m + (1 - b1) g,
                  v = b2 v + (1 - b2) g^2, p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps), t the 1-based step
  global_clip     k_adam's clip: g = grad * grad_scale, then g *= c where c = clip / (||grad|| grad_scale + 1e-6) < 1
                  (torch.nn.utils.clip_grad_norm_ applied after the 1/world scale); clip <= 0: off
  clip_per_tensor k_rainbow_apply's (and PA-DQN's) minimize_and_clip: each tensor's g *= clip / ||g|| where ||g|| > clip
  ddpg_apply      k_ddpg_apply: g = grad * grad_scale + l2 p on the w1 / w2 / w3 kernels of every net (never a bias),
                  the actor's Adam at actor_lr and actor_step (0: its params, m and v stay as they are), the critics' at
                  critic_lr and critic_step, then target = tau p + (1 - tau) target over the whole buffer
  bq_apply        k_bq_apply: Adam, then target[:ntgt] = params[:ntgt] when copy_target
  conti groups    the Adam groups of CQL-conti and BCQ-conti (include/rl4rs_b200.h's layouts): each group's parameter
                  range, learning-rate field and the target range its soft update writes

Bounds (u = 2^-24, the fp32 unit roundoff).  Each term of the kernel's arithmetic is rounded once; the bound of a result
is the sum of the rounding of every term it is made of, so it scales with the terms and not with the (possibly cancelled)
result:
  effective gradient  rel_g = 2u for the grad_scale and clip products, plus, where a clip engages, the relative error of
                      its factor: a sum of squares of positive terms added L at a time in a thread and then over a
                      log2(T)-level tree is within (L + log2 T) u of exact, its sqrt halves that, and the sqrt, the
                      scale, the + 1e-6 and the division add 4u: rel_c = ((L + log2 T) / 2 + 4) u
  m                   4u |b1 m0| + (4u + rel_g) |(1 - b1) g|
  v                   4u |b2 v0| + (5u + 2 rel_g) |(1 - b2) g^2|
  bias corrections    powf(b, t) is within 4 ulp (8u relative) of b^t, so 1 - b^t is within 8u b^t / (1 - b^t) of itself
  param               one ulp of the larger of |p| and |p'|, plus the step lr / bc1 * m / denom evaluated with m and v
                      at their bounds, the bias corrections at theirs and 4u for the division, sqrt and products
  soft target         tau p + (1 - tau) t with p the kernel's own new parameter: 3u (|tau p| + |(1 - tau) t|)
On an H100 the kernels stay within 0.66 of them (tests/test_gpu_optim_shapes.py).  A wrong step count, torch's eps
placed as TF1 places it, a clip factor missing or applied twice, l2 on a bias, swapped learning rates, tau swapped with
1 - tau, or a dropped grad_scale moves at least one element of that module's cases by more than 100x its bound.
"""
import math

import numpy as np

U = 2.0 ** -24
B1, B2 = float(np.float32(0.9)), float(np.float32(0.999))
EPS = float(np.float32(1e-8))
CLIP_EPS = float(np.float32(1e-6))          # k_adam's + 1e-6 in the clip's denominator


def f32(x):
    """The float32 value of a hyper-parameter, as the C-ABI receives it."""
    return float(np.float32(x))


def _d(x):
    return np.asarray(x, dtype=np.float64)


def ulp(p):
    """One ulp of float32 p (the spacing at |p|; the smallest normal's at 0)."""
    p = np.abs(np.asarray(p, dtype=np.float32))
    return (np.nextafter(np.maximum(p, np.float32(2.0 ** -126)), np.float32(np.inf)) -
            np.maximum(p, np.float32(2.0 ** -126))).astype(np.float64)


def sumsq_rel(n, threads):
    """rel_c of a clip factor whose norm sums n squares, ceil(n / threads) per thread, then over `threads` in a tree."""
    return ((math.ceil(n / threads) + math.log2(threads)) / 2 + 4) * U


def carried(n, seed, steps=3):
    """float32 (g, m, v): m and v carried from `steps` earlier gradients, so that the update depends on the gradient's
    magnitude and not only on its sign; magnitudes over six decades, about 5 % exact zeros, and a sixth of the elements at
    |g| ~ 1e-8, where sqrt(v_hat) is near eps."""
    rs = np.random.RandomState(seed)
    mag = 10.0 ** rs.uniform(-6, 0, n)
    tiny = rs.rand(n) < 1 / 6
    mag[tiny] = 10.0 ** rs.uniform(-8.5, -7.5, tiny.sum())
    m, v = np.zeros(n), np.zeros(n)
    for _ in range(steps):
        gk = rs.randn(n) * mag
        m = 0.9 * m + 0.1 * gk
        v = 0.999 * v + 0.001 * gk * gk
    g = rs.randn(n) * mag
    g[rs.rand(n) < 0.05] = 0.0
    return g.astype(np.float32), m.astype(np.float32), v.astype(np.float32)


# ---- the update rules -----------------------------------------------------------------------------------------------
class Step(object):
    """The result of one rule: p, m, v (float64 arrays) and the bounds bp, bm, bv of each element."""

    def __init__(self, p, m, v, bp, bm, bv):
        self.p, self.m, self.v, self.bp, self.bm, self.bv = p, m, v, bp, bm, bv


def adam(p, g, m, v, step, lr, b1=B1, b2=B2, eps=EPS, rel_g=2 * U):
    """torch.optim.Adam on float32 p, m, v and the effective gradient g (float64) -> Step.  rel_g: the relative error the
    kernel may carry in g (see the module docstring)."""
    p, g, m0, v0 = _d(p), _d(g), _d(m), _d(v)
    lr, b1, b2, eps = f32(lr), f32(b1), f32(b2), f32(eps)
    m1 = b1 * m0 + (1 - b1) * g
    v1 = b2 * v0 + (1 - b2) * g * g
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    sv = np.sqrt(v1) / math.sqrt(bc2)
    den = sv + eps
    upd = (lr / bc1) * m1 / den
    bm = 4 * U * np.abs(b1 * m0) + (4 * U + rel_g) * np.abs((1 - b1) * g)
    bv = 4 * U * np.abs(b2 * v0) + (5 * U + 2 * rel_g) * np.abs((1 - b2) * g * g)
    rbc1, rbc2 = 8 * U * b1 ** step / bc1, 8 * U * b2 ** step / bc2
    # the denominator's relative error: sqrt(v) carries half of v's, sqrt(bc2) half of bc2's, 2u for the sqrt and division
    rden = (0.5 * bv / np.maximum(v1, 1e-300) + 0.5 * rbc2 + 2 * U) * sv / den + U
    bstep = (lr / bc1) * bm / den + np.abs(upd) * (rden + rbc1 + 4 * U)
    return Step(p - upd, m1, v1, ulp(np.maximum(np.abs(p), np.abs(p - upd))) + bstep, bm, bv)


def global_clip(grad, grad_scale, clip):
    """k_adam's effective gradient -> (g float64, c the clip factor or 1, engaged)."""
    g = _d(grad) * f32(grad_scale)
    if not clip > 0:
        return g, 1.0, False
    gn = math.sqrt(float((_d(grad) ** 2).sum())) * f32(grad_scale)
    c = f32(clip) / (gn + CLIP_EPS)
    return (g * c, c, True) if c < 1 else (g, 1.0, False)


def clip_per_tensor(grad, slices, clip):
    """minimize_and_clip: every tensor [lo, hi) whose norm exceeds clip scaled to norm clip on its own -> (g float64,
    [(lo, hi, engaged)])."""
    g = np.array(grad, dtype=np.float64)
    out = []
    for lo, hi in slices:
        nrm = math.sqrt(float((g[lo:hi] ** 2).sum()))
        on = clip > 0 and nrm > f32(clip)
        if on:
            g[lo:hi] *= f32(clip) / nrm
        out.append((lo, hi, on))
    return g, out


def soft_target(p_new, t, tau):
    """tau p + (1 - tau) t, (1 - tau) rounded to float32 as the kernels form it -> (target, bound)."""
    tau = f32(tau)
    omt = f32(1.0 - tau)
    a, b = tau * _d(p_new), omt * _d(t)
    return a + b, 3 * U * (np.abs(a) + np.abs(b))


# ---- DDPG / TD3 -----------------------------------------------------------------------------------------------------
H1, H2, OBS = 400, 300, 256


def ddpg_nets(D, twin):
    """[(name, offset, [(tensor, lo, hi, is_kernel)])] of the actor and the critic(s), include/rl4rs_b200.h's layout."""
    out, off = [], 0
    for name, K, N3 in [("a_", OBS, D), ("q1_", OBS + D, 1)] + ([("q2_", OBS + D, 1)] if twin else []):
        ts = []
        for t, k, kern in (("w1", K * H1, True), ("b1", H1, False), ("w2", H1 * H2, True), ("b2", H2, False),
                           ("w3", H2 * N3, True), ("b3", N3, False)):
            ts.append((name + t, off, off + k, kern))
            off += k
        out.append((name, ts))
    return out, off


def ddpg_layout(D, twin):
    """-> (n_params, n_actor, kernel mask bool [n_params])."""
    nets, n = ddpg_nets(D, twin)
    mask = np.zeros(n, dtype=bool)
    for _, ts in nets:
        for _, lo, hi, kern in ts:
            mask[lo:hi] = kern
    return n, nets[0][1][-1][2], mask


def ddpg_apply(p, t, grad, m, v, D, twin, actor_step, critic_step, actor_lr, critic_lr, l2, tau, grad_scale):
    """k_ddpg_apply -> (Step over the whole buffer, actor range end).  The actor's part of Step is p, m, v unchanged (bounds
    0: bit-identical) when actor_step == 0."""
    n, na, kern = ddpg_layout(D, twin)
    p32 = _d(p)
    g = _d(grad) * f32(grad_scale)
    rel_g = np.full(n, 2 * U)
    g = np.where(kern, g + f32(l2) * p32, g)
    out = Step(*(np.zeros(n) for _ in range(6)))
    for lo, hi, s, lr in ((0, na, actor_step, actor_lr), (na, n, critic_step, critic_lr)):
        if s == 0:
            out.p[lo:hi], out.m[lo:hi], out.v[lo:hi] = p32[lo:hi], _d(m)[lo:hi], _d(v)[lo:hi]
            continue
        st = adam(p32[lo:hi], g[lo:hi], m[lo:hi], v[lo:hi], s, lr, rel_g=rel_g[lo:hi])
        # the l2 term is one more fp32 product and sum: its rounding joins the gradient's
        extra = np.where(kern[lo:hi], 2 * U * np.abs(f32(l2) * p32[lo:hi]), 0.0)
        st.bm += (1 - B1) * extra
        st.bv += (1 - B2) * 2 * np.abs(g[lo:hi]) * extra
        for k in ("p", "m", "v", "bp", "bm", "bv"):
            getattr(out, k)[lo:hi] = getattr(st, k)
    return out, na


# ---- discrete batch RL ----------------------------------------------------------------------------------------------
BQ_E = 32        # the masked encoder's item-embedding width


def bq_layout(algo, K, A):
    """-> (n_params, target_size) of include/rl4rs_b200.h's batch-RL layout (masked net: w1[K,256] b1[256] emb[A,32]
    w2[576,A] b2[A] w3[A,A] b3[A]; plain net: w1[K,256] b1 w2[256,256] b2 w3[256,A] b3; BC masked imitator, BCQ masked Q |
    masked imitator, CQL plain; the target holds the Q part)."""
    masked = K * 256 + 256 + A * BQ_E + (256 + 10 * BQ_E) * A + A + A * A + A
    plain = K * 256 + 256 + 256 * 256 + 256 + 256 * A + A
    return {"BC": (masked, 0), "BCQ": (2 * masked, masked), "CQL": (plain, plain)}[algo]


def bq_apply(p, t, grad, m, v, ntgt, step, lr, eps, copy_target):
    """k_bq_apply -> (Step, the new target float64 or None when it is not copied)."""
    st = adam(p, grad, m, v, step, lr, eps=eps)
    return st, (st.p[:ntgt] if copy_target else None)


# ---- continuous batch RL: the Adam groups of one SGD step -----------------------------------------------------------
CH = 256         # hidden width of every continuous batch-RL net


def _net(off, K, N):
    return off + K * CH + CH + CH * CH + CH + CH * N + N


def cqlc_groups(K, D):
    """CQL-conti's groups in update order: (name, params [lo, hi), the r4_cqlc_hyper lr field, target [lo, hi) of the
    soft update or None).  Layout: actor (K -> 2D) | critic 0 (K+D -> 1) | critic 1 | log_temp | log_alpha; the target is
    [critic 0 | critic 1], indexed from the first critic's w1 (target[k] follows params[t0 + k])."""
    a = _net(0, K, 2 * D)
    c1 = _net(_net(a, K + D, 1), K + D, 1)
    return [("temp", (c1, c1 + 1), "lr_temp", None), ("alpha", (c1 + 1, c1 + 2), "lr_alpha", None),
            ("critic", (a, c1), "lr_critic", (0, c1 - a)), ("actor", (0, a), "lr_actor", None)]


def cqlc_sizes(K, D):
    """-> (n_params, target_size, t0)."""
    g = dict((x[0], x) for x in cqlc_groups(K, D))
    return g["alpha"][1][1], g["critic"][3][1], g["critic"][1][0]


def bcqc_groups(K, D, Lat):
    """BCQ-conti's groups in update order (as cqlc_groups).  Layout: actor (K+D -> D) | critic 0 (K+D -> 1) | critic 1 |
    VAE encoder (K+D -> 2 Lat) | decoder (K+Lat -> D); the target is [actor | critic 0 | critic 1], indexed from 0 (the
    critics' soft update writes target[c0:c1], the actor's target[0:a])."""
    a = _net(0, K + D, D)
    c1 = _net(_net(a, K + D, 1), K + D, 1)
    dec = _net(_net(c1, K + D, 2 * Lat), K + Lat, D)
    return [("imitator", (c1, dec), "lr_imitator", None), ("critic", (a, c1), "lr_critic", (a, c1)),
            ("actor", (0, a), "lr_actor", (0, a))]


def bcqc_sizes(K, D, Lat):
    """-> (n_params, target_size)."""
    g = bcqc_groups(K, D, Lat)
    return g[0][1][1], g[1][1][1]
