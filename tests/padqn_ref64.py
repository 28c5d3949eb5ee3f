"""Float64 NumPy reference of PA-DQN (csrc/r4_padqn.cuh, policy.ParametricQNetwork): the masked Q over every (row, item)
pair, the double-Q target with done and masked next states, the Huber loss and every tensor's gradient, the per-tensor clip
with torch.optim.Adam and the hard target copy, and the SoftQ / argmax rule on given uniforms."""
import numpy as np

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
    g = np.array(grad, dtype=np.float64)
    for lo, hi in slices(D):
        nrm = np.sqrt((g[lo:hi] ** 2).sum())
        if clip > 0 and nrm > clip:
            g[lo:hi] *= clip / nrm
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
        m[i, rng.choice(A, size=int(rng.integers(1, 4)), replace=False)] = 1
    return m


def item_vectors(A, D, seed=0, onehot=False):
    """The env's item vectors: row 0 zeros, the rest L2-normalised (or the identity under one-hot actions)."""
    if onehot:
        return np.eye(A)
    rng = np.random.default_rng(seed)
    e = rng.standard_normal((A, D))
    e /= np.linalg.norm(e, axis=1, keepdims=True)
    e[0] = 0.0
    return e
