"""Float64 references of the learner kernels (csrc/r4_ppo.cuh, r4_gauss.cuh, r4_ddpg.cuh, r4_rainbow.cuh, r4_batchrl.cuh).

Each function takes the flat float32 parameter vector in the layout include/rl4rs_b200.h documents, and the batch, and
returns a `Ref`: the loss, the per-sample rows (loss terms or td), the statistics the kernel reports, the gradient by
float64 autograd, and `margin` [n], each row's smallest distance to a discrete decision, divided by that decision's scale.
A row whose margin is small may take the other branch in float32 (a relu kink, an argmax, the huber knee, a clip edge,
BCQ's threshold), which moves whole weight columns by O(1/n); the GPU tests keep only rows with a clear margin.

The twins of rl4rs_b200/policy.py run the forward passes: a shallow copy of the twin gets a float64 `flat` leaf (and
target), so the reference is the twin's own operation in float64.  Two things stay in float32 on purpose:
  * RAINBOW's support z and the projection's r + gamma_n (1 - done) z, b, floor and ceil are formed in float32, as the
    twin (policy.py, DistributionalQNetwork.__init__) and the kernel form them, so both pick the same atoms bit for bit;
    the probabilities they move are float64.
  * CQL's reward scaler (r - mean) / den is applied in float32, as the kernel applies it.

Decisions and their scales (`margin` is the minimum over a row of distance / scale):
  relu pre-activations on the backward path   |x| / (rms of the row's layer * sqrt(max(1, K / 256))), K the dot-product
                                               length (forward-only relus -- target nets, the
                                               networks that pick a* -- are continuous in value and are not decisions)
  argmax (double-Q a*, BCQ's filtered a*,      (top1 - top2) / max(max |value| of the row, 1e-3)
    CQL a*)
  huber knee                                   ||td| - 1|
  PPO ratio clip, value clip                   |ratio - (1 +- clip)|, ||v - v_old| - vf_clip| / max(1, vf_clip) and,
                                               where the value clip is active, |vf1 - vf2| / max(1, vf1, vf2)
  TD3 smoothing                                ||target_noise * noise| - noise_clip| and ||pi'(s') + noise| - 1|
  BCQ threshold                                |log pi - max log pi - log_flex| over every action of s'
"""
import copy
import math

import numpy as np
import torch

TIE = 1e-4            # a decision this close (relative to its scale) to its switch point is a tie
RELU_TIE = 1e-5       # relu kinks, in units of the row's layer rms times sqrt(max(1, K / 256)) for a K-term dot product.
# Basis (measured on the CPU, K-term sums of fp32 products added one by one in fp32, the worst order a kernel could use):
# the worst error over 64 x 256 pre-activations is 2.5e-6 of the row rms at K = 256, 2.9e-6 at K = 400 and 1.1e-5 at
# K = 4096, so the threshold (1.0e-5, 1.25e-5, 4.0e-5 of the rms) stays at least 3.7x above it at every K of these nets.
# A flat 1e-4 would drop about 21 % of TD3's rows (its backward paths cross thousands of relu units); this drops 2-3 %.


class Ref(object):
    def __init__(self, loss, rows, stats, grad, margin, relu_margin, **extra):
        self.loss, self.rows, self.stats, self.grad = loss, rows, stats, grad
        self.margin, self.relu_margin = margin, relu_margin
        self.__dict__.update(extra)

    def clear(self):
        """bool [n]: rows whose every decision is clear of its switch point."""
        return (self.margin > TIE) & (self.relu_margin > RELU_TIE)


def tensors(twin):
    """[(name, slice)] of every tensor of the twin's flat layout."""
    out, off = [], 0
    for name, shape in twin._shapes:
        k = math.prod(shape)
        out.append((name, slice(off, off + k)))
        off += k
    return out


def _f64(twin, flat, target=None):
    t = copy.copy(twin)
    t.flat = flat.detach().to(torch.float64).clone().requires_grad_(True)
    if target is not None:
        t.target = target.detach().to(torch.float64).clone()
    return t


def _d(x):
    return None if x is None else x.detach().to(torch.float64)


def _relu_dist(*layers):
    """[n]: min over the layers (z [n, H], K) of |z| / (rms(z row) sqrt(max(1, K / 256))), K the length of the dot
    products that formed z (the scale of their fp32 rounding grows with K; see RELU_TIE)."""
    out = None
    for z, K in layers:
        z = z.detach()
        d = (z.abs() / z.pow(2).mean(1, keepdim=True).sqrt().clamp_min(1e-30)).min(1).values / math.sqrt(max(1.0, K / 256))
        out = d if out is None else torch.minimum(out, d)
    return out


def argmax_margin(v):
    """[n]: (top1 - top2) / max(max |v| of the row, 1e-3) of v [n, A]."""
    v = v.detach()
    top = v.topk(2, 1).values
    return (top[:, 0] - top[:, 1]) / v.abs().max(1).values.clamp_min(1e-3)


def masked_argmax_margin(v, allowed):
    """[n]: argmax_margin of v [n, A] over the allowed entries only, so that a masking sentinel (float32.min, -2^15) sets
    neither the gap nor the scale.  One allowed entry: inf (no decision); none: 0 (never clear)."""
    v = v.detach()
    top = v.masked_fill(~allowed, -math.inf).topk(2, 1).values
    gap = torch.where(allowed.any(1), top[:, 0] - top[:, 1], torch.zeros_like(top[:, 0]))
    return gap / v.masked_fill(~allowed, 0.0).abs().max(1).values.clamp_min(1e-3)


def _inf(n, dev):
    return torch.full((n,), math.inf, dtype=torch.float64, device=dev)


# ---- PPO / A2C over the mask policy and the Gaussian policy ------------------------------------------------------------
def _pg(pol, inputs, mode, action, old_logp, old_dist, old_value, adv, target, hp, inv_n):
    d, value = pol.forward(*inputs)
    logp, kl, ent = pol.terms(d, action, _d(old_dist) if mode == 0 else None)
    adv, target = _d(adv), _d(target)
    n = adv.shape[0]
    margin = _inf(n, adv.device)
    if mode == 0:
        old_value = _d(old_value)
        ratio = torch.exp(logp - _d(old_logp))
        c = hp["clip"]
        surr = torch.min(adv * ratio, adv * torch.clamp(ratio, 1 - c, 1 + c))
        vf1 = (value - target) ** 2
        vc = hp["vf_clip"]
        vf2 = (old_value + torch.clamp(value - old_value, -vc, vc) - target) ** 2
        vf = torch.max(vf1, vf2)
        pi = -surr
        total = pi + hp["kl_coeff"] * kl + hp["vf_coeff"] * vf - hp["ent_coeff"] * ent
        r = ratio.detach()
        margin = torch.minimum((r - (1 - c)).abs(), (r - (1 + c)).abs())
        margin = torch.minimum(margin, ((value - old_value).detach().abs() - vc).abs() / max(1.0, vc))
        clipped = (value - old_value).detach().abs() > vc           # inside the clip vf2 is vf1: no decision
        gap = (vf1 - vf2).detach().abs() / torch.max(vf1, vf2).detach().clamp_min(1.0)
        margin = torch.minimum(margin, torch.where(clipped, gap, torch.full_like(gap, math.inf)))
    else:
        pi = -(logp * adv)
        vf = 0.5 * (value - target) ** 2
        kl = torch.zeros_like(pi)
        total = pi + hp["vf_coeff"] * vf - hp["ent_coeff"] * ent
    loss = total.sum() * inv_n
    loss.backward()
    rows = torch.stack([pi, vf, kl, ent, total], 1).detach()
    return loss.detach(), rows, pol.flat.grad.detach(), margin, value.detach(), d.detach()


def policy_grad(twin, flat, mode, obs, mask, action, old_logp, old_logits, old_value, adv, target, hp, inv_n):
    """r4_policy_grad: mode 0 PPO surrogate, mode 1 A2C, loss = sum of the per-sample totals * inv_n.  stats = the
    column sums of rows {policy loss, vf loss, kl, entropy, total}; the kernel reports them times its stat_scale."""
    pol = _f64(twin, flat)
    loss, rows, grad, margin, value, logits = _pg(pol, (_d(obs), mask), mode, action.long(), old_logp, old_logits,
                                                  old_value, adv, target, hp, inv_n)
    return Ref(loss, rows, rows.sum(0), grad, margin, _inf(len(margin), margin.device))


def policy_act(twin, flat, obs, mask):
    """r4_policy_act with explore off -> (masked logits, value, logp of the argmax, argmax, argmax margin over the allowed
    actions)."""
    pol = _f64(twin, flat)
    with torch.no_grad():
        logits, value = pol.forward(_d(obs), mask)
        lp = torch.log_softmax(logits, -1)
        a = logits.argmax(1)
        m = masked_argmax_margin(logits, mask.bool())
    return logits, value, lp.gather(1, a.unsqueeze(1)).squeeze(1), a, m


def gauss_grad(twin, flat, mode, obs, action, old_logp, old_dist, old_value, adv, target, hp, inv_n):
    """r4_gauss_grad, as policy_grad over the DiagGaussian (tanh layers only: the decisions are PPO's clips)."""
    pol = _f64(twin, flat)
    loss, rows, grad, margin, value, d = _pg(pol, (_d(obs),), mode, _d(action), old_logp, old_dist, old_value, adv,
                                             target, hp, inv_n)
    return Ref(loss, rows, rows.sum(0), grad, margin, _inf(len(margin), margin.device))


def gauss_act(twin, flat, obs):
    pol = _f64(twin, flat)
    with torch.no_grad():
        return pol.forward(_d(obs))


# ---- DDPG / TD3 ---------------------------------------------------------------------------------------------------
def _mlp(p, pre, x):
    z1 = x @ p[pre + "w1"] + p[pre + "b1"]
    z2 = torch.relu(z1) @ p[pre + "w2"] + p[pre + "b2"]
    return torch.relu(z2) @ p[pre + "w3"] + p[pre + "b3"], ((z1, x.shape[1]), (z2, z1.shape[1]))


def ddpg_grad(twin, flat, target, obs, action, reward, new_obs, done, weights, noise, gamma, target_noise, noise_clip, inv_n):
    """r4_ddpg_grad: critic loss sum w (td1^2 + td2^2) / 2 * inv_n and actor loss -sum Q1(s, pi(s)) * inv_n (critic weights
    frozen) -> rows = td1, stats = {critic loss, actor loss, sum Q1(s, pi(s)) * inv_n}."""
    pol = _f64(twin, flat, target)
    obs, new_obs, action = _d(obs), _d(new_obs), _d(action)
    n = obs.shape[0]
    P, T = pol.params(pol.flat), pol.params(pol.target)
    w = torch.ones(n, dtype=torch.float64, device=obs.device) if weights is None else _d(weights)
    margin = _inf(n, obs.device)
    with torch.no_grad():
        a2 = torch.tanh(_mlp(T, "a_", new_obs)[0])
        if noise is not None:
            tn = target_noise * _d(noise)
            margin = torch.minimum(margin, (tn.abs() - noise_clip).abs().min(1).values)
            a2 = a2 + tn.clamp(-noise_clip, noise_clip)
            margin = torch.minimum(margin, (a2.abs() - 1.0).abs().min(1).values)
            a2 = a2.clamp(-1.0, 1.0)
        x2 = torch.cat([new_obs, a2], 1)
        qt = _mlp(T, "q1_", x2)[0].squeeze(-1)
        if pol.twin:
            qt = torch.min(qt, _mlp(T, "q2_", x2)[0].squeeze(-1))
        y = _d(reward) + gamma * (1.0 - done.to(torch.float64)) * qt
    xa = torch.cat([obs, action], 1)
    q1, z_q1 = _mlp(P, "q1_", xa)
    td1 = q1.squeeze(-1) - y
    err = 0.5 * td1 ** 2
    zs = list(z_q1)
    if pol.twin:
        q2, z_q2 = _mlp(P, "q2_", xa)
        err = err + 0.5 * (q2.squeeze(-1) - y) ** 2
        zs += list(z_q2)
    critic = (w * err).sum() * inv_n
    pre, z_a = _mlp(P, "a_", obs)
    frozen = {k: v.detach() for k, v in P.items()}
    qpi, z_qpi = _mlp(frozen, "q1_", torch.cat([obs, torch.tanh(pre)], 1))
    actor = -qpi.sum() * inv_n
    (critic + actor).backward()
    stats = torch.stack([critic.detach(), actor.detach(), -actor.detach()])
    return Ref(critic.detach() + actor.detach(), td1.detach(), stats, pol.flat.grad.detach(), margin,
               _relu_dist(*zs, *z_a, *z_qpi))


def ddpg_act(twin, flat, obs):
    pol = _f64(twin, flat)
    with torch.no_grad():
        return torch.tanh(_mlp(pol.params(pol.flat), "a_", _d(obs))[0])


# ---- RAINBOW ------------------------------------------------------------------------------------------------------
def rainbow_grad(twin, flat, target, obs, action, reward, new_obs, done, weights, gamma_n, inv_n):
    """r4_rainbow_grad through the twin's loss in float64 (projection indices in float32, see the module docstring) ->
    rows = td, stats = {loss, sum td * inv_n, sum Q(s, a) * inv_n}."""
    pol = _f64(twin, flat, target)
    obs, new_obs = _d(obs), _d(new_obs)
    n = obs.shape[0]
    w = None if weights is None else _d(weights)
    loss, td = pol.loss(obs, action, reward, new_obs, done, w, gamma_n, inv_n)
    loss.backward()
    p = pol.params(pol.flat)
    with torch.no_grad():
        rows = torch.arange(n, device=obs.device)
        q = pol.forward(obs)[1][rows, action.long()]
        h = torch.tanh(torch.tanh(obs @ p["w1"] + p["b1"]) @ p["w2"] + p["b2"])
        relu = _relu_dist((h @ p["aw1"] + p["ab1"], h.shape[1]), (h @ p["sw1"] + p["sb1"], h.shape[1]))
        margin = argmax_margin(pol.forward(new_obs)[1])
    stats = torch.stack([loss.detach(), td.sum() * inv_n, q.sum() * inv_n])
    return Ref(loss.detach(), td, stats, pol.flat.grad.detach(), margin, relu)


def rainbow_act(twin, flat, obs):
    pol = _f64(twin, flat)
    with torch.no_grad():
        return pol.forward(_d(obs))[1]


# ---- BC / BCQ / CQL -----------------------------------------------------------------------------------------------
def batchrl_grad(twin, flat, target, obs, action, reward, next_obs, terminal, hp):
    """r4_batchrl_grad through the twin's loss in float64 -> stats {loss, td or nll, Q(s, a) or the imitator's mean z^2}
    (minibatch means).  rows: None (the kernel reports no per-sample rows)."""
    net = _f64(twin, flat, target if twin.n_target else None)
    obs, next_obs = _d(obs), _d(next_obs)
    n = obs.shape[0]
    if net.algo == "CQL":        # the reward scaler in float32, as the kernel applies it
        reward = ((reward.to(torch.float32) - hp["reward_mean"]) / hp["reward_den"])
        hp = dict(hp, reward_mean=0.0, reward_den=1.0)
    loss, st = net.loss(obs, action, reward, next_obs, terminal, hp)
    loss.backward()
    p = net.params(net.flat)
    margin = _inf(n, obs.device)
    with torch.no_grad():
        if net.algo == "CQL":
            z1 = obs @ p["w1"] + p["b1"]
            relu = _relu_dist((z1, obs.shape[1]), (torch.relu(z1) @ p["w2"] + p["b2"], z1.shape[1]))
        else:
            pres = ("i_",) if net.algo == "BC" else ("q_", "i_")
            relu = _relu_dist(*[(obs @ p[q + "w1"] + p[q + "b1"], obs.shape[1]) for q in pres])
        if net.algo != "BC":
            rows = torch.arange(n, device=obs.device)
            if net.algo == "BCQ":
                lp = torch.log_softmax(net.imitator(next_obs), 1)
                thr = (lp - lp.max(1, keepdim=True).values - hp["log_flex"]).abs().min(1).values
                margin = torch.minimum(thr, argmax_margin(net.bcq_filtered(next_obs, hp["log_flex"])))
                a_star = net.bcq_filtered(next_obs, hp["log_flex"]).argmax(1)
                r = _d(reward)
            else:
                margin = argmax_margin(net.q(next_obs))
                a_star = net.q(next_obs).argmax(1)
                r = _d(reward)
            y = r + hp["gamma"] * (1.0 - terminal.to(torch.float64)) * net.q(next_obs, net.target)[rows, a_star]
            td = net.q(obs)[rows, action.long()] - y
            margin = torch.minimum(margin, (td.abs() - 1.0).abs())
    return Ref(loss.detach(), None, st, net.flat.grad.detach(), margin, relu)


def batchrl_act(twin, flat, obs, log_flex):
    """r4_batchrl_act in float64 -> (raw output, action_probs, keep, [(pick, margin) of mode 0, of mode 1]).  Mode 0's
    margin is taken over the items keep allows (the -2^15 sentinel is not a value); mode 1's includes, for BCQ, the
    imitator threshold |log pi - max log pi - log_flex| over every action of the row."""
    net = _f64(twin, flat)
    x = _d(obs)
    with torch.no_grad():
        raw = net.imitator(x) if net.algo == "BC" else net.q(x)
        probs = torch.log_softmax(raw, 1) if net.algo == "BC" else torch.softmax(raw, 1)
        keep = net.keep(x)
        pick0 = torch.where(keep, probs, torch.full_like(probs, -2.0 ** 15))
        pick1 = net.bcq_filtered(x, log_flex) if net.algo == "BCQ" else probs
        m1 = argmax_margin(pick1)
        if net.algo == "BCQ":
            lp = torch.log_softmax(net.imitator(x), 1)
            m1 = torch.minimum(m1, (lp - lp.max(1, keepdim=True).values - log_flex).abs().min(1).values)
    return raw, probs, keep, [(pick0, masked_argmax_margin(probs, keep)), (pick1, m1)]


# ---- synthetic batches of the learner tests (tests/test_learner_ref64_cpu.py on the CPU, test_gpu_learner_shapes.py) ----
def mask_batch(pol, P, A, dev, seed):
    """P rows of a PPO / A2C batch over the mask policy: masks with one allowed action, every action, or a random half;
    the value clip (PG_HP, 1.0) active on about half the rows."""
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(P, 256, generator=g).to(dev)
    mask = (torch.rand(P, A, generator=g) < 0.5).to(torch.uint8)
    for i in range(P):                                  # one allowed action, every action, a random half
        if i % 3 == 0:
            mask[i].zero_()
            mask[i, int(torch.randint(0, A, (1,), generator=g))] = 1
        elif i % 3 == 1:
            mask[i].fill_(1)
        elif int(mask[i].sum()) == 0:
            mask[i, 0] = 1
    mask = mask.to(dev)
    act = torch.multinomial(mask.double(), 1, generator=torch.Generator(device=dev).manual_seed(seed)).squeeze(1)
    with torch.no_grad():
        logits, value = pol.forward(obs, mask)
    ok = mask.bool()
    old_logits = torch.where(ok, logits + 0.3 * torch.randn(P, A, generator=g).to(dev), logits).contiguous()
    old_logp = torch.log_softmax(old_logits, -1).gather(1, act.unsqueeze(1)).squeeze(1).contiguous()
    old_v = (value + 1.5 * torch.randn(P, generator=g).to(dev)).contiguous()    # both sides of vf_clip = 1
    adv = torch.randn(P, generator=g).to(dev)
    tgt = (old_v + 3 * torch.randn(P, generator=g).to(dev)).contiguous()
    return obs, mask, act, old_logp, old_logits, old_v, adv, tgt


PG_HP = {0: {"clip": 0.3, "vf_clip": 1.0, "vf_coeff": 0.5, "kl_coeff": 0.2, "ent_coeff": 0.01},
         1: {"clip": 0.0, "vf_clip": 0.0, "vf_coeff": 0.5, "kl_coeff": 0.0, "ent_coeff": 0.01}}


def gauss_batch(pol, P, D, dev, seed):
    """P rows of a PPO / A2C batch over the Gaussian policy, actions drawn from a perturbed old distribution."""
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(P, 256, generator=g).to(dev)
    with torch.no_grad():
        d, v = pol.forward(obs)
    old_d = (d + 0.2 * torch.randn(P, 2 * D, generator=g).to(dev)).contiguous()
    act = (old_d[:, :D] + old_d[:, D:].exp() * torch.randn(P, D, generator=g).to(dev)).contiguous()
    old_lp = pol.logp(old_d, act).contiguous()
    old_v = (v + 1.5 * torch.randn(P, generator=g).to(dev)).contiguous()
    adv = torch.randn(P, generator=g).to(dev)
    tgt = (old_v + 3 * torch.randn(P, generator=g).to(dev)).contiguous()
    return obs, act, old_lp, old_d, old_v, adv, tgt


def rb_rewards(P, Z, v_min, v_max, g):
    """Rewards on the atoms, on and beyond the clip edges, and in between."""
    dz = np.float32(np.float32(v_max) - np.float32(v_min)) / np.float32(Z - 1)
    atoms = np.float32(v_min) + np.arange(Z, dtype=np.float32) * dz
    r = (torch.rand(P, generator=g).double().numpy() * (v_max - v_min) * 0.3).astype(np.float32)
    kind = np.arange(P) % 5
    r[kind == 0] = atoms[np.arange(P)[kind == 0] % Z]
    r[kind == 1] = np.where(np.arange(P)[kind == 1] % 2 == 0, np.float32(v_max), np.float32(v_min))
    r[kind == 2] = np.where(np.arange(P)[kind == 2] % 2 == 0, np.float32(v_max + 5), np.float32(v_min - 5))
    return torch.as_tensor(r)


def bq_net(algo, K, A, dev):
    """BatchRLNet with a synthetic location mask (about 70 % allowed per page layer, item A - 1 in every layer) and special
    items (A // 20 of them, at least one, never A - 1), the target moved off the Q weights."""
    from rl4rs_b200.policy import BatchRLNet
    rs = np.random.RandomState(K + A)
    lm = (rs.rand(4, A) < 0.7).astype(np.float32)
    lm[:, A - 1] = 1.0              # bq_data never logs item A - 1 as a previous action: every row keeps at least it
    special = sorted(set(rs.choice(A, max(1, A // 20), replace=False).tolist()) - {A - 1}) or [0]
    net = BatchRLNet(algo, K, lm, special, A, dev, seed=1)
    if net.n_target:
        with torch.no_grad():
            net.target.add_(0.05 * torch.randn(net.n_target, generator=torch.Generator().manual_seed(3)).to(dev))
    return net


def bq_data(K, A, P, dev, seed):
    """A logged dataset of 10-entry episodes with at least P transitions: random observations, valid item ids in the
    last 10 columns, the DeviceDataset on `dev`."""
    from rl4rs_b200.batchrl import DeviceDataset
    L = 10
    E = P // (L - 1) + 2
    rs = np.random.RandomState(seed)
    obs = rs.randn(E, L, K).astype(np.float32)
    obs[:, :, K - 10:K - 1] = rs.randint(0, A - 1, (E, L, 9))     # item A - 1 stays out: see bq_net
    # Slate and SeqSlate cur_steps; the encoder embeds cur_steps with the item table, so it stays below A
    obs[:, :, K - 1] = (np.arange(L)[None] + 9 * (np.arange(E)[:, None] % 4)) % A
    ds = {"observations": obs.reshape(-1, K), "actions": rs.randint(0, A, E * L).reshape(-1, 1).astype(np.float32),
          "rewards": rs.rand(E * L).astype(np.float32), "terminals": np.tile(np.r_[np.zeros(L - 1), 1.0], E)}
    return DeviceDataset(ds, dev)


# the kernels take these as float32: the values are float32 numbers, so the float64 reference uses the same ones
BQ_HP = {"gamma": float(np.float32(0.99)), "beta": 0.5, "alpha": 1.0, "log_flex": float(np.float32(math.log(0.3))),
         "reward_mean": 0.375, "reward_den": 0.3125}


def bq_hyper(algo):
    """The hyper-parameters of one algorithm (the reward scaler is CQL's only, beta BCQ's)."""
    h = dict(BQ_HP, beta=0.0 if algo == "BC" else 0.5)
    if algo != "CQL":
        h.update(reward_mean=0.0, reward_den=1.0)
    return h
