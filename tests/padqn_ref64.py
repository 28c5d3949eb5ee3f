"""Float64 NumPy reference of PA-DQN (csrc/r4_padqn.cuh, policy.ParametricQNetwork): the masked Q over every (row, item)
pair, the double-Q target with done and masked next states, the Huber loss and every tensor's gradient, the per-tensor clip
with torch.optim.Adam and the hard target copy, and the SoftQ / argmax rule on given uniforms."""
import numpy as np

import optim_ref64

OBS, H = 256, 256
FLOAT_MIN = float(np.finfo(np.float32).min)
NAMES = ("w1", "b1", "w2", "b2", "w3", "b3")


def shapes(D):
    return [("w1", (OBS + D, H)), ("b1", (H,)), ("w2", (H, H)), ("b2", (H,)), ("w3", (H, 1)), ("b3", (1,))]


def slices(D):
    out, off = [], 0
    for _, s in shapes(D):
        k = int(np.prod(s))
        out.append((off, off + k))
        off += k
    return out


def params(flat, D):
    flat = np.asarray(flat, dtype=np.float64)
    return {name: flat[lo:hi].reshape(s) for (name, s), (lo, hi) in zip(shapes(D), slices(D))}


def q_pairs(p, obs, emb, action):
    """Q(s, a) [n] and the forward planes of the n taken pairs."""
    x = np.concatenate([obs, emb[action]], 1)
    h1 = np.tanh(x @ p["w1"] + p["b1"])
    h2 = np.tanh(h1 @ p["w2"] + p["b2"])
    return (h2 @ p["w3"] + p["b3"])[:, 0], (x, h1, h2)


def qm(p, obs, mask, emb, chunk=32):
    """Qm [n, A]: Q(s, a) where mask[s, a] != 0, float32.min where it is 0."""
    n, A = mask.shape
    out = np.empty((n, A))
    P = emb @ p["w1"][OBS:]
    for i in range(0, n, chunk):
        S = obs[i:i + chunk] @ p["w1"][:OBS] + p["b1"]
        h = np.tanh(np.tanh(S[:, None, :] + P[None]) @ p["w2"] + p["b2"])
        out[i:i + chunk] = (h @ p["w3"])[..., 0] + p["b3"][0]
    return np.where(np.asarray(mask) != 0, out, FLOAT_MIN)


def target(p_on, p_tg, new_obs, next_mask, reward, done, gamma, emb):
    """(a* [n], y [n]): a* the first argmax of the online Qm(s', .), y = r + gamma (1 - done) Qm_target(s', a*)."""
    a_star = qm(p_on, new_obs, next_mask, emb).argmax(1)
    qt = qm(p_tg, new_obs, next_mask, emb)[np.arange(len(a_star)), a_star]
    return a_star, reward + gamma * (1.0 - done) * qt


def loss_and_grads(p, p_tg, emb, obs, action, reward, new_obs, done, next_mask, weights=None, gamma=1.0, inv_n=None):
    """-> (loss, td [n], Q(s, a) [n], {tensor: gradient}) of sum_i w_i huber(td_i) inv_n."""
    n = obs.shape[0]
    inv_n = 1.0 / n if inv_n is None else inv_n
    w = np.ones(n) if weights is None else np.asarray(weights, dtype=np.float64)
    _, y = target(p, p_tg, new_obs, next_mask, reward, done, gamma, emb)
    q, (x, h1, h2) = q_pairs(p, obs, emb, action)
    td = q - y
    hub = np.where(np.abs(td) <= 1.0, 0.5 * td * td, np.abs(td) - 0.5)
    dq = w * np.clip(td, -1.0, 1.0) * inv_n
    d2 = dq[:, None] * p["w3"][:, 0][None] * (1 - h2 ** 2)
    d1 = (d2 @ p["w2"].T) * (1 - h1 ** 2)
    g = {"w1": x.T @ d1, "b1": d1.sum(0), "w2": h1.T @ d2, "b2": d2.sum(0), "w3": h2.T @ dq[:, None], "b3": dq.sum(0, keepdims=True)}
    return (w * hub).sum() * inv_n, td, q, g


def flat_grad(g, D):
    return np.concatenate([g[k].reshape(-1) for k in NAMES])


def apply(flat, target_flat, grad, m, v, step, D, lr=5e-4, eps=1e-8, clip=40.0, copy_target=False):
    """Per-tensor clip (minimize_and_clip), torch.optim.Adam (betas 0.9 / 0.999) at the 1-based step, then the hard copy ->
    (flat, target, m, v)."""
    g, _ = optim_ref64.clip_per_tensor(grad, slices(D), clip)
    m = 0.9 * m + 0.1 * g
    v = 0.999 * v + 0.001 * g * g
    denom = np.sqrt(v) / np.sqrt(1 - 0.999 ** step) + eps
    flat = flat - (lr / (1 - 0.9 ** step)) * m / denom
    return flat, (flat.copy() if copy_target else np.array(target_flat, dtype=np.float64)), m, v


def act(q, u=None):
    """The first argmax of Qm [n, A] (u None), or SoftQ: the first a whose cumulative softmax exceeds u [n] in [0, 1)."""
    if u is None:
        return q.argmax(1)
    e = np.exp(q - q.max(1, keepdims=True))
    cdf = np.cumsum(e, 1)
    return np.minimum((cdf <= (np.asarray(u) * cdf[:, -1])[:, None]).sum(1), q.shape[1] - 1)


def uniforms(seed, counter, n):
    """The act kernel's uniform per row: the top 24 bits of r4ddpg::draw(seed, counter, row, 0) / 2^24."""
    from rl4rs_b200.policy import counter_draws
    return (counter_draws(seed, counter, n, 1)[0][:, 0] + 1.0) / 2.0


def env_like_masks(n, A, seed=0, keep=0.3):
    """Masks shaped like the env's location masks: a random contiguous window of items per row (at least one)."""
    rng = np.random.default_rng(seed)
    m = np.zeros((n, A), dtype=np.uint8)
    w = max(1, int(A * keep))
    for i in range(n):
        lo = rng.integers(0, A - w + 1)
        m[i, lo:lo + w] = 1
    return m


def planted_masks(n, A, seed=0):
    """Sparse masks (1 to 3 items per row) with every 5th row all masked."""
    rng = np.random.default_rng(seed)
    m = np.zeros((n, A), dtype=np.uint8)
    for i in range(n):
        if i % 5 == 4:
            continue
        m[i, rng.choice(A, size=min(A, int(rng.integers(1, 4))), replace=False)] = 1
    return m


def tie_pairs(A):
    """The item pairs item_vectors(..., dup=True) gives identical vectors: (a, a + 1) in neighbouring lanes of the act
    kernel's warp (both ends of the row), and (a, a + 32) in one lane when A > 34."""
    out = [(1, 2), (A - 2, A - 1)] if A >= 4 else [(0, 1)]
    if A > 34:
        out.append((3, 35))
    return out


def item_vectors(A, D, seed=0, onehot=False, dup=False):
    """The env's item vectors: row 0 zeros, the rest L2-normalised (or the identity under one-hot actions).  dup: the
    second item of every tie_pairs(A) pair copies the first's vector, so their Q values are bitwise equal in the kernel and
    in qm_t."""
    if onehot:
        return np.eye(A)
    rng = np.random.default_rng(seed)
    e = rng.standard_normal((A, D))
    e /= np.linalg.norm(e, axis=1, keepdims=True)
    e[0] = 0.0
    if dup:
        for a, b in tie_pairs(A):
            e[b] = e[a]
    return e


def plant_ties(mask, A, every=11):
    """Rows i = 3 mod `every` keep only one tie_pairs(A) pair (taken in turn), so their first argmax is decided by a tie."""
    pairs = tie_pairs(A)
    for k, i in enumerate(range(3, mask.shape[0], every)):
        mask[i] = 0
        mask[i, list(pairs[k % len(pairs)])] = 1
    return mask


# ---- the float64 reference in torch, on any device, in row chunks -----------------------------------------------------
def params_t(flat, D, device):
    """{tensor: float64 torch tensor on device} of a flat f32 / f64 buffer (torch or NumPy)."""
    import torch
    flat = torch.as_tensor(flat).detach().to(device=device, dtype=torch.float64)
    return {name: flat[lo:hi].reshape(s) for (name, s), (lo, hi) in zip(shapes(D), slices(D))}


def qm_t(p, obs, mask, emb, plane=1 << 24):
    """qm() in float64 torch on obs's device, in row chunks of at most `plane` hidden values.  Q is evaluated once per
    distinct item vector, so items with equal vectors get bitwise-equal values."""
    import torch
    dev = p["w1"].device
    obs, emb = torch.as_tensor(obs).to(dev, torch.float64), torch.as_tensor(emb).to(dev, torch.float64)
    uniq, inv = torch.unique(emb, dim=0, return_inverse=True)
    P = uniq @ p["w1"][OBS:]
    n, U = obs.shape[0], uniq.shape[0]
    chunk = max(1, plane // (U * H))
    out = []
    for i in range(0, n, chunk):
        S = obs[i:i + chunk] @ p["w1"][:OBS] + p["b1"]
        h = torch.tanh(torch.tanh(S[:, None, :] + P[None]) @ p["w2"] + p["b2"])
        out.append((h @ p["w3"])[..., 0] + p["b3"][0])
    q = (torch.cat(out) if out else obs.new_zeros(0, U))[:, inv]
    return torch.where(torch.as_tensor(mask).to(dev).bool(), q, torch.full_like(q, FLOAT_MIN))


def top_gap(q):
    """Per row: the row's max minus the largest value strictly below it (inf when every value is equal), so exact ties
    do not count as near decisions."""
    import torch
    m = q.max(1, keepdim=True).values
    below = torch.where(q < m, q, torch.full_like(q, -float("inf"))).max(1).values
    return m[:, 0] - below


def q_pairs_t(p, obs, emb, action):
    """q_pairs() in float64 torch: Q(s, a) [n] and the forward planes of the taken pairs."""
    import torch
    x = torch.cat([obs.double(), torch.as_tensor(emb).to(obs.device, torch.float64)[action.long()]], 1)
    h1 = torch.tanh(x @ p["w1"] + p["b1"])
    h2 = torch.tanh(h1 @ p["w2"] + p["b2"])
    return (h2 @ p["w3"] + p["b3"])[:, 0], (x, h1, h2)


def target_t(p_on, p_tg, new_obs, next_mask, emb):
    """(a* [n], Qm_target(s', a*) [n], the online top-two gap [n]) in float64 torch."""
    import torch
    q_on = qm_t(p_on, new_obs, next_mask, emb)
    a_star = q_on.argmax(1)
    qt = qm_t(p_tg, new_obs, next_mask, emb)[torch.arange(len(a_star), device=a_star.device), a_star]
    return a_star, qt, top_gap(q_on)


def loss_and_grads_t(p, p_tg, emb, obs, action, reward, new_obs, done, next_mask, weights=None, gamma=1.0, inv_n=None):
    """loss_and_grads() in float64 torch -> dict of loss, the per-sample td, q, hub, a*, gap (the online Qm(s', .) top-two
    gap that decides a*), kink (| |td| - 1 |, the distance from the Huber kink) and grads {tensor: gradient}."""
    import torch
    n = obs.shape[0]
    inv_n = 1.0 / n if inv_n is None else inv_n
    w = torch.ones(n, dtype=torch.float64, device=obs.device) if weights is None else weights.double()
    a_star, qt, gap = target_t(p, p_tg, new_obs, next_mask, emb)
    y = reward.double() + gamma * (1.0 - done.double()) * qt
    q, (x, h1, h2) = q_pairs_t(p, obs, emb, action)
    td = q - y
    hub = torch.where(td.abs() <= 1.0, 0.5 * td * td, td.abs() - 0.5)
    dq = w * td.clamp(-1.0, 1.0) * inv_n
    d2 = dq[:, None] * p["w3"][:, 0][None] * (1 - h2 ** 2)
    d1 = (d2 @ p["w2"].T) * (1 - h1 ** 2)
    g = {"w1": x.T @ d1, "b1": d1.sum(0), "w2": h1.T @ d2, "b2": d2.sum(0), "w3": h2.T @ dq[:, None],
         "b3": dq.sum(0, keepdim=True)}
    return {"loss": (w * hub).sum() * inv_n, "td": td, "q": q, "hub": hub, "a_star": a_star, "gap": gap,
            "kink": (td.abs() - 1.0).abs(), "grads": g, "stats": torch.stack([(w * hub).sum(), td.sum(), q.sum()]) * inv_n}


def td_plan(n, seed):
    """Planned td errors [n]: even rows +-(0.25, 0.9) (the quadratic Huber branch), odd rows +-(1.1, 3) (the linear one),
    every row at least 0.1 from the kink.  The quadratic branch's gradient is proportional to td, so |td| stays well above
    the float32 error of Q (~1e-6 of |Q| through k_padqn_rows, ~3e-6 through the pair scorer) that it inherits."""
    rng = np.random.default_rng(seed)
    inner = rng.choice([-1.0, 1.0], n) * rng.uniform(0.25, 0.9, n)
    outer = rng.choice([-1.0, 1.0], n) * rng.uniform(1.1, 3.0, n)
    return np.where(np.arange(n) % 2 == 0, inner, outer)


# ---- gradient cases: a replay pool, rewards that place every td on a planned Huber branch, and the clear rows -----------
TIE = 2e-4          # the online Qm(s', .) top-two gap below which a* is a near decision (|Q| of order 1 in the tests)
KINK = 1e-3         # | |td| - 1 | below which the Huber branch is a near decision
MAX_DROP = 0.08     # the share of a pool the two filters may drop


def pool_size(n):
    return max(256, n + n // 10 + 16)


def grad_case(flat, target, emb, n, gamma, weighted, seed, inv_n=None, dead_next=False):
    """A replay pool of pool_size(n) rows on emb's device and the n sampled rows of one r4_padqn_grad call.

    Next-state masks are env_like_masks with plant_ties rows; rows 5 mod 13 have every next action masked, and are
    terminal unless dead_next (then y = r + gamma Qm_target = r + gamma float32.min).  Every third row is terminal.  The
    rewards are r = Q(s, a) - gamma (1 - done) Qm_target(s', a*) - td_plan, rounded to float32, so both Huber branches
    are populated and every td is clear of the kink.  idx = the first n pool rows whose a* gap clears TIE and whose td
    clears KINK, after asserting the filter dropped less than MAX_DROP of the pool.
    -> dict of the pool tensors (obs, action, reward, new_obs, done, next_mask), idx, weights [n] or None, inv_n, the
    float64 reference over the n rows (`ref`, loss_and_grads_t's dict) and the dropped share."""
    import torch
    dev = emb.device
    A, D = emb.shape
    N = pool_size(n)
    g = torch.Generator().manual_seed(seed)
    obs, new_obs = torch.randn(N, OBS, generator=g).to(dev), torch.randn(N, OBS, generator=g).to(dev)
    action = torch.randint(0, A, (N,), generator=g, dtype=torch.int32).to(dev)
    nm = plant_ties(env_like_masks(N, A, seed), A)
    rows = np.arange(N)
    nm[rows % 13 == 5] = 0
    done = (rows % 3 == 0) | ((rows % 13 == 5) & (not dead_next))
    next_mask, done = torch.as_tensor(nm).to(dev), torch.as_tensor(done.astype(np.uint8)).to(dev)
    p, pt = params_t(flat, D, dev), params_t(target, D, dev)
    _, qt, _ = target_t(p, pt, new_obs, next_mask, emb)
    q, _ = q_pairs_t(p, obs, emb, action)
    plan = torch.as_tensor(td_plan(N, seed), device=dev)
    live = (done == 1) | next_mask.bool().any(1)
    noise = torch.randn(N, generator=g, dtype=torch.float64).to(dev)
    reward = torch.where(live, q - gamma * (1.0 - done.double()) * torch.where(live, qt, 0.0) - plan, noise).float()
    w = (torch.rand(N, generator=g) + 0.5).to(dev) if weighted else None
    pool = loss_and_grads_t(p, pt, emb, obs, action, reward, new_obs, done, next_mask, w, gamma)
    clear = (pool["gap"] > TIE) & (pool["kink"] > KINK)
    drop = 1.0 - float(clear.double().mean())
    assert drop < MAX_DROP, "the tie filter dropped %.1f %% of the pool" % (100 * drop)
    idx = torch.nonzero(clear).reshape(-1)[:n]
    assert idx.numel() == n
    ws = w[idx] if weighted else None
    inv_n = 1.0 / n if inv_n is None else inv_n
    ref = loss_and_grads_t(p, pt, emb, obs[idx], action[idx], reward[idx], new_obs[idx], done[idx], next_mask[idx], ws,
                           gamma, inv_n)
    return {"obs": obs, "action": action, "reward": reward, "new_obs": new_obs, "done": done, "next_mask": next_mask,
            "idx": idx, "weights": ws, "inv_n": inv_n, "ref": ref, "drop": drop, "clear": clear}
