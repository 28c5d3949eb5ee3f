"""The policy the reference trains on this env: RLlib's MyMaskActionsModel
(rl4rs/nets/rllib/rllib_mask_model.py:7-64): obs(256) -> FC 64 tanh -> 284 logits
+ max(log(action_mask), float32.min); the value head shares the 64-d hidden (vf_share_layers).

Exploration is RLlib SoftQ with temperature 1 = sample from softmax(logits)
(modelfree_train.py:398-402); evaluation uses argmax (explore=False, :412-414).
Parameters live in one flat f32 buffer so the data-parallel gradient all-reduce is ONE NCCL call
(SURVEY.md section 8e: 34 973 parameters ~ 140 KB).
"""
import math

import torch

OBS, HID = 256, 64
FLOAT_MIN = torch.finfo(torch.float32).min


class MaskedPolicy(object):
    def __init__(self, action_size=284, device="cuda", seed=0):
        self.A = action_size
        self.device = torch.device(device)
        shapes = [("w1", (OBS, HID)), ("b1", (HID,)), ("w2", (HID, action_size)), ("b2", (action_size,)),
                  ("wv", (HID, 1)), ("bv", (1,))]
        n = sum(math.prod(s) for _, s in shapes)
        g = torch.Generator(device="cpu").manual_seed(seed)
        self.flat = torch.zeros(n, dtype=torch.float32, device=self.device, requires_grad=True)
        self.views, off = {}, 0
        with torch.no_grad():
            for name, shape in shapes:
                k = math.prod(shape)
                v = self.flat[off:off + k].view(shape)
                if len(shape) == 2:       # RLlib normc_initializer(1.0) (0.01 for the output layers)
                    w = torch.randn(shape, generator=g)
                    std = 0.01 if name in ("w2", "wv") else 1.0
                    w = w * std / w.pow(2).sum(0, keepdim=True).sqrt()
                    v.copy_(w.to(self.device))
                off += k
        self._shapes, self.n_params = shapes, n

    def params(self):
        out, off = {}, 0
        for name, shape in self._shapes:
            k = math.prod(shape)
            out[name] = self.flat[off:off + k].view(shape)
            off += k
        return out

    def forward(self, obs, mask):
        """obs f32 [B,256], mask {0,1} [B,A] -> (masked logits [B,A], value [B])."""
        p = self.params()
        h = torch.tanh(obs @ p["w1"] + p["b1"])
        logits = h @ p["w2"] + p["b2"]
        inf_mask = torch.clamp(torch.log(mask.to(torch.float32)), min=FLOAT_MIN)   # rllib_mask_model.py:55-58
        value = (h @ p["wv"] + p["bv"]).squeeze(-1)
        return logits + inf_mask, value

    def inputs(self, obs):
        """env observation {'obs', 'action_mask'} -> the inputs of forward()."""
        return obs["obs"], obs["action_mask"]

    def terms(self, logits, action, old_logits=None):
        """Categorical over masked logits -> (logp(action), KL(old || new) or None without old_logits, entropy) per sample."""
        logp_all = torch.log_softmax(logits, -1)
        logp = logp_all.gather(1, action.unsqueeze(1)).squeeze(1)
        kl = None
        if old_logits is not None:
            old_logp_all = torch.log_softmax(old_logits, -1)
            kl = (old_logp_all.exp() * (old_logp_all - logp_all)).sum(-1)
        return logp, kl, -(logp_all.exp() * logp_all).sum(-1)

    @torch.no_grad()
    def act(self, obs, mask, explore=True):
        """-> (action i32 [B], logp [B], value [B], masked logits [B,A])."""
        logits, value = self.forward(obs, mask)
        logp_all = torch.log_softmax(logits, dim=-1)
        if explore:
            a = torch.multinomial(logp_all.exp(), 1).squeeze(-1)
        else:
            a = logits.argmax(dim=-1)
        return a.to(torch.int32), logp_all.gather(1, a.long().unsqueeze(1)).squeeze(1), value, logits


class GaussianPolicy(object):
    """The policy RLlib builds for the continuous-action env (`PPO_conti` / `A2C_conti`, modelfree_train.py:46-48): the default
    FullyConnectedNetwork (fcnet_hiddens [256, 256], tanh, vf_share_layers off) over obs(256):
        fc_1 256 tanh -> fc_2 256 tanh -> fc_out 2D = mean | log_std      (DiagGaussian dist inputs, free_log_std off)
        fc_value_1 256 tanh -> fc_value_2 256 tanh -> value_out 1
    normc_initializer(1.0) for the hidden kernels, 0.01 for fc_out and value_out, zero biases.  Exploration is
    StochasticSampling (a = mean + std * N(0, 1)); evaluation takes the mean.  The env receives clip(a, -1, 1)
    (clip_actions), the sample batch stores a.  The flat layout is csrc/r4_gauss.cuh's; this torch twin is the CPU path and
    the autograd cross-check of those kernels (tests/test_gpu_trainer_conti.py)."""

    def __init__(self, action_dim=32, device="cuda", seed=0):
        self.D = action_dim
        self.device = torch.device(device)
        D2 = 2 * action_dim
        shapes = [("w1", (OBS, 256)), ("b1", (256,)), ("w2", (256, 256)), ("b2", (256,)), ("wo", (256, D2)), ("bo", (D2,)),
                  ("vw1", (OBS, 256)), ("vb1", (256,)), ("vw2", (256, 256)), ("vb2", (256,)), ("vwo", (256, 1)), ("vbo", (1,))]
        n = sum(math.prod(s) for _, s in shapes)
        g = torch.Generator(device="cpu").manual_seed(seed)
        self.flat = torch.zeros(n, dtype=torch.float32, device=self.device, requires_grad=True)
        off = 0
        with torch.no_grad():
            for name, shape in shapes:
                k = math.prod(shape)
                if len(shape) == 2:       # normc_initializer
                    w = torch.randn(shape, generator=g)
                    std = 0.01 if name in ("wo", "vwo") else 1.0
                    self.flat[off:off + k].view(shape).copy_((w * std / w.pow(2).sum(0, keepdim=True).sqrt()).to(self.device))
                off += k
        self._shapes, self.n_params = shapes, n

    params = MaskedPolicy.params

    def forward(self, obs):
        """obs f32 [n,256] -> (dist inputs [n,2D] = mean | log_std, value [n])."""
        p = self.params()
        h = torch.tanh(torch.tanh(obs @ p["w1"] + p["b1"]) @ p["w2"] + p["b2"])
        g = torch.tanh(torch.tanh(obs @ p["vw1"] + p["vb1"]) @ p["vw2"] + p["vb2"])
        return h @ p["wo"] + p["bo"], (g @ p["vwo"] + p["vbo"]).squeeze(-1)

    def inputs(self, obs):
        """env observation (the obs vector, or {'obs': ...}) -> the inputs of forward()."""
        return (obs["obs"] if isinstance(obs, dict) else obs,)

    def terms(self, dist_inputs, action, old_dist=None):
        """-> (logp(action), KL(old || new) or None without old_dist, entropy) per sample."""
        return self.logp(dist_inputs, action), None if old_dist is None else self.kl(old_dist, dist_inputs), self.entropy(dist_inputs)

    @staticmethod
    def logp(dist_inputs, action):
        """DiagGaussian log-likelihood summed over the action dimensions."""
        mu, ls = dist_inputs.chunk(2, dim=-1)
        return (-0.5 * ((action - mu) / ls.exp()) ** 2 - ls - 0.5 * math.log(2 * math.pi)).sum(-1)

    @staticmethod
    def entropy(dist_inputs):
        ls = dist_inputs.chunk(2, dim=-1)[1]
        return (ls + 0.5 * math.log(2 * math.pi * math.e)).sum(-1)

    @staticmethod
    def kl(old_inputs, new_inputs):
        """KL(old || new) of two DiagGaussians (RLlib TorchDiagGaussian.kl)."""
        mo, lo = old_inputs.chunk(2, dim=-1)
        mn, ln = new_inputs.chunk(2, dim=-1)
        return (ln - lo + ((2 * lo).exp() + (mo - mn) ** 2) / (2 * (2 * ln).exp()) - 0.5).sum(-1)

    @torch.no_grad()
    def act(self, obs, explore=True):
        """-> (action [n,D] unclipped, env action [n,D] = clip(action, -1, 1), logp [n], value [n], dist inputs [n,2D])."""
        d, value = self.forward(obs)
        mu, ls = d.chunk(2, dim=-1)
        a = mu + ls.exp() * torch.randn(mu.shape, device=mu.device) if explore else mu.clone()
        return a, a.clamp(-1.0, 1.0), self.logp(d, a), value, d


def _splitmix64(x):
    """csrc/r4_ppo.cuh splitmix64 over a uint64 array (wrapping arithmetic)."""
    import numpy as np
    x = x + np.uint64(0x9E3779B97F4A7C15)
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def counter_draws(seed, counter, rows, dims):
    """The exploration draws of csrc/r4_ddpg.cuh for rows 0..rows-1 and dims 0..dims-1, keyed by (seed, counter):
    -> (uniform in [-1, 1), standard normal), both float64 [rows, dims]."""
    import numpy as np
    with np.errstate(over="ignore"):
        r = np.arange(rows, dtype=np.uint64)[:, None]
        d = np.arange(dims, dtype=np.uint64)[None, :]
        key = ((np.uint64(counter) + r) << np.uint64(6)) + d
        x = _splitmix64(np.uint64(seed) ^ _splitmix64(key))
    hi = (x >> np.uint64(40)).astype(np.float64)
    u1 = (hi + 0.5) / 16777216.0
    u2 = ((x >> np.uint64(16)) & np.uint64(0xFFFFFF)).astype(np.float64) / 16777216.0
    return hi * (2.0 / 16777216.0) - 1.0, np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


class DeterministicActorCritic(object):
    """The networks RLlib 1.5 builds for DDPG / TD3 (modelfree_trainer.py:25-28, actor_hiddens = critic_hiddens = [400, 300],
    relu): an actor obs(256) -> 400 -> 300 -> D squashed to Box(-1, 1) by (high - low) sigmoid(2x) + low = tanh(x), and a
    critic concat(obs, a) -> 400 -> 300 -> 1; TD3 (twin) adds a second critic.  Keras glorot-uniform kernels, zero biases.
    One flat buffer [actor | critic | twin] (csrc/r4_ddpg.cuh's layout) and a target copy of it (hard copy at construction).
    This torch twin is the CPU path of DDPGTrainer / TD3Trainer and the autograd cross-check of the kernels
    (tests/test_gpu_trainer_ddpg.py)."""

    H1, H2 = 400, 300

    def __init__(self, action_dim=32, device="cuda", seed=0, twin=False):
        self.D, self.twin = action_dim, bool(twin)
        self.device = torch.device(device)
        D, H1, H2 = action_dim, self.H1, self.H2

        def net(p, K, N3):
            return [(p + "w1", (K, H1)), (p + "b1", (H1,)), (p + "w2", (H1, H2)), (p + "b2", (H2,)), (p + "w3", (H2, N3)),
                    (p + "b3", (N3,))]
        shapes = net("a_", OBS, D) + net("q1_", OBS + D, 1) + (net("q2_", OBS + D, 1) if twin else [])
        n = sum(math.prod(s) for _, s in shapes)
        g = torch.Generator(device="cpu").manual_seed(seed)
        self.flat = torch.zeros(n, dtype=torch.float32, device=self.device, requires_grad=True)
        off = 0
        with torch.no_grad():
            for name, shape in shapes:
                k = math.prod(shape)
                if len(shape) == 2:       # glorot uniform
                    lim = math.sqrt(6.0 / (shape[0] + shape[1]))
                    self.flat[off:off + k].view(shape).copy_(((torch.rand(shape, generator=g) * 2 - 1) * lim).to(self.device))
                off += k
        self._shapes, self.n_params = shapes, n
        self.n_actor = sum(math.prod(s) for name, s in shapes if name.startswith("a_"))
        self.target = self.flat.detach().clone()
        mask = torch.zeros(n, dtype=torch.bool)
        off = 0
        for name, shape in shapes:
            k = math.prod(shape)
            mask[off:off + k] = len(shape) == 2
            off += k
        self.kernel_mask = mask.to(self.device)      # the l2 terms cover the kernels, not the biases

    def params(self, flat=None):
        flat = self.flat if flat is None else flat
        out, off = {}, 0
        for name, shape in self._shapes:
            k = math.prod(shape)
            out[name] = flat[off:off + k].view(shape)
            off += k
        return out

    @staticmethod
    def _mlp(p, pre, x):
        return torch.relu(torch.relu(x @ p[pre + "w1"] + p[pre + "b1"]) @ p[pre + "w2"] + p[pre + "b2"]) @ p[pre + "w3"] + p[pre + "b3"]

    def actor(self, obs, flat=None):
        """obs f32 [n,256] -> the deterministic action [n,D] in (-1, 1)."""
        return torch.tanh(self._mlp(self.params(flat), "a_", obs))

    def critic(self, obs, a, k=1, flat=None):
        """Q_k(obs, a) [n] (k = 1, or 2 for the twin)."""
        return self._mlp(self.params(flat), "q%d_" % k, torch.cat([obs, a], dim=1)).squeeze(-1)

    def inputs(self, obs):
        return (obs["obs"] if isinstance(obs, dict) else obs,)

    def losses(self, obs, action, reward, new_obs, done, weights=None, smooth_noise=None, gamma=1.0, target_noise=0.2,
               noise_clip=0.5, inv_n=None):
        """The RLlib DDPG / TD3 losses without the l2 terms (r4_ddpg_grad's definition), as sums over the batch times inv_n
        (default 1/n): -> (critic loss, actor loss, td1 [n]).  The actor loss reads the critic with its weights detached,
        so its gradient reaches the actor weights only."""
        n = obs.shape[0]
        inv_n = 1.0 / n if inv_n is None else inv_n
        w = torch.ones(n, device=obs.device) if weights is None else weights
        with torch.no_grad():
            a2 = self.actor(new_obs, self.target)
            if smooth_noise is not None:
                a2 = (a2 + (target_noise * smooth_noise).clamp(-noise_clip, noise_clip)).clamp(-1.0, 1.0)
            qt = self.critic(new_obs, a2, 1, self.target)
            if self.twin:
                qt = torch.min(qt, self.critic(new_obs, a2, 2, self.target))
            y = reward + gamma * (1.0 - done.to(torch.float32)) * qt
        td1 = self.critic(obs, action, 1) - y
        err = 0.5 * td1 ** 2
        if self.twin:
            err = err + 0.5 * (self.critic(obs, action, 2) - y) ** 2
        critic_loss = (w * err).sum() * inv_n
        frozen = self.flat.detach()
        actor_loss = -self.critic(obs, self.actor(obs), 1, frozen).sum() * inv_n
        return critic_loss, actor_loss, td1.detach()

    def l2_loss(self, l2):
        """l2 * sum(w^2) / 2 over the kernels of the actor and of the critic(s) (the two losses' l2 terms added)."""
        return l2 * 0.5 * (self.flat[self.kernel_mask] ** 2).sum()

    @torch.no_grad()
    def soft_update(self, tau):
        """target = tau * online + (1 - tau) * target."""
        self.target.copy_(tau * self.flat.detach() + (1.0 - tau) * self.target)


class DistributionalQNetwork(object):
    """The Q network RLlib 1.5 builds for RAINBOW on the plain 256-d observation (modelfree_train.py:146-178, no custom
    model): the default FullyConnectedNetwork with no_final_linear, obs(256) -> 256 tanh -> 256 tanh (normc(1.0) kernels,
    zero biases), and the dueling distributional head (hiddens [128], Keras glorot-uniform kernels, zero biases):
        advantage   256 -> 128 relu -> A * atoms          state score   256 -> 128 relu -> atoms
        logits[a][k] = score[k] + (adv[a][k] - mean_a adv[a][k]),  Q(s, a) = sum_k z_k softmax(logits[a])_k,
    z = v_min + k dz, dz = (v_max - v_min) / (atoms - 1) in float32.  One flat buffer (csrc/r4_rainbow.cuh's layout) and a
    target copy of it (hard copy at construction).  This torch twin is the CPU path of RainbowTrainer and the autograd
    cross-check of the kernels (tests/test_gpu_trainer_rainbow.py)."""

    HT, HQ = 256, 128

    def __init__(self, action_size=284, device="cuda", seed=0, num_atoms=8, v_min=0.0, v_max=1000.0):
        import numpy as np
        self.A, self.atoms, self.v_min, self.v_max = action_size, num_atoms, float(v_min), float(v_max)
        self.device = torch.device(device)
        A, Z, HT, HQ = action_size, num_atoms, self.HT, self.HQ
        shapes = [("w1", (OBS, HT)), ("b1", (HT,)), ("w2", (HT, HT)), ("b2", (HT,)),
                  ("aw1", (HT, HQ)), ("ab1", (HQ,)), ("aw2", (HQ, A * Z)), ("ab2", (A * Z,)),
                  ("sw1", (HT, HQ)), ("sb1", (HQ,)), ("sw2", (HQ, Z)), ("sb2", (Z,))]
        n = sum(math.prod(s) for _, s in shapes)
        g = torch.Generator(device="cpu").manual_seed(seed)
        self.flat = torch.zeros(n, dtype=torch.float32, device=self.device, requires_grad=True)
        self.slices, off = [], 0
        with torch.no_grad():
            for name, shape in shapes:
                k = math.prod(shape)
                v = self.flat[off:off + k].view(shape)
                if name in ("w1", "w2"):               # normc_initializer(1.0)
                    w = torch.randn(shape, generator=g)
                    v.copy_((w / w.pow(2).sum(0, keepdim=True).sqrt()).to(self.device))
                elif len(shape) == 2:                  # glorot uniform
                    lim = math.sqrt(6.0 / (shape[0] + shape[1]))
                    v.copy_(((torch.rand(shape, generator=g) * 2 - 1) * lim).to(self.device))
                self.slices.append((off, off + k))
                off += k
        self._shapes, self.n_params = shapes, n
        self.target = self.flat.detach().clone()
        # the support in float32, formed as the kernels form it (the projection's floor / ceil must agree bit for bit)
        dz = np.float32(np.float32(self.v_max) - np.float32(self.v_min)) / np.float32(Z - 1)
        self.dz = torch.tensor(dz, dtype=torch.float32, device=self.device)
        self.z = torch.tensor(np.float32(self.v_min), device=self.device) + torch.arange(Z, dtype=torch.float32,
                                                                                          device=self.device) * self.dz

    params = DeterministicActorCritic.params

    def forward(self, obs, flat=None):
        """obs f32 [n,256] -> (support logits [n, A, atoms], Q [n, A])."""
        p = self.params(flat)
        h = torch.tanh(torch.tanh(obs @ p["w1"] + p["b1"]) @ p["w2"] + p["b2"])
        adv = (torch.relu(h @ p["aw1"] + p["ab1"]) @ p["aw2"] + p["ab2"]).view(-1, self.A, self.atoms)
        score = torch.relu(h @ p["sw1"] + p["sb1"]) @ p["sw2"] + p["sb2"]
        logits = score.unsqueeze(1) + (adv - adv.mean(1, keepdim=True))
        return logits, (torch.softmax(logits, -1) * self.z).sum(-1)

    def inputs(self, obs):
        return (obs["obs"] if isinstance(obs, dict) else obs,)

    def project(self, reward, done, probs, gamma_n):
        """RLlib QLoss's categorical projection: the target distribution probs [n, atoms] moved to r + gamma_n (1 - done) z,
        clipped to [v_min, v_max], split over the neighbouring atoms -> m [n, atoms].  Mass on an index off the support is
        dropped, as tf.one_hot drops it."""
        Z = self.atoms
        nd = gamma_n * (1.0 - done.to(torch.float32))
        rt = (reward.to(torch.float32).unsqueeze(1) + nd.unsqueeze(1) * self.z).clamp(self.v_min, self.v_max)
        b = (rt - self.v_min) / self.dz
        lb, ub = torch.floor(b), torch.ceil(b)
        feq = (ub - lb < 0.5).to(torch.float32)
        ml, mu = probs * (ub - b + feq), probs * (b - lb)
        m = torch.zeros_like(probs)
        for j in range(Z):                             # in atom order, as the kernel adds them
            for i, w in ((lb[:, j].long(), ml[:, j]), (ub[:, j].long(), mu[:, j])):
                ok = (i >= 0) & (i < Z)
                m.scatter_add_(1, i.clamp(0, Z - 1).unsqueeze(1), torch.where(ok, w, torch.zeros_like(w)).unsqueeze(1))
        return m

    def loss(self, obs, action, reward, new_obs, done, weights=None, gamma_n=1.0, inv_n=None):
        """The distributional double-Q loss sum_i w_i td_i * inv_n (default 1/n), td = softmax cross entropy of the projected
        target (labels) and the taken action's logits -> (loss, td [n])."""
        n = obs.shape[0]
        inv_n = 1.0 / n if inv_n is None else inv_n
        rows = torch.arange(n, device=obs.device)
        with torch.no_grad():
            a_star = self.forward(new_obs)[1].argmax(1)
            pt = torch.softmax(self.forward(new_obs, self.target)[0][rows, a_star], -1)
            m = self.project(reward, done, pt, gamma_n)
        logits = self.forward(obs)[0][rows, action.long()]
        td = -(m * torch.log_softmax(logits, -1)).sum(-1)
        w = torch.ones(n, device=obs.device) if weights is None else weights
        return (w * td).sum() * inv_n, td.detach()

    @torch.no_grad()
    def clip_per_tensor(self, grad, clip):
        """RLlib's minimize_and_clip: every tensor's gradient whose norm exceeds clip is scaled to norm clip, on its own."""
        if clip:
            for lo, hi in self.slices:
                g = grad[lo:hi]
                norm = g.norm()
                if float(norm) > clip:
                    g.mul_(clip / norm)

    @torch.no_grad()
    def act(self, obs, explore, seed=0, counter=0):
        """-> (action i32 [n], Q [n, A]): argmax Q, or SoftQ (a ~ softmax(Q)) over csrc/r4_rainbow.cuh's uniform per row."""
        import numpy as np
        q = self.forward(obs)[1]
        if not explore:
            return q.argmax(1).to(torch.int32), q
        u = (counter_draws(seed, counter, q.shape[0], 1)[0][:, 0] + 1.0) / 2.0       # the top 24 bits / 2^24
        cdf = np.cumsum(torch.softmax(q.double(), 1).cpu().numpy(), 1)
        a = np.minimum((cdf <= (u * cdf[:, -1])[:, None]).sum(1), self.A - 1)
        return torch.as_tensor(a, dtype=torch.int32, device=q.device), q


class RawStatePolicy(object):
    """RLlib 'mask_model_rawstate' (rl4rs/nets/rllib/rllib_mask_model.py:67-115 over rllib_rawstate_model.py:25-86): the
    policy reads the RAW state -- category ids [21], dense features [432], sequence ids [2,64] (`rawstate_as_obs`,
    slate.py:246-253) -- through its own embedding tables:
        category = mean_t E_c[cat]            (utils.id_input_processing, nets/utils.py:7-14)
        dense    = ELU(ELU(x W1 + b1) W2 + b2) (nets/utils.py:48-54; the Dropout layers are inactive outside Keras fit)
        sequence = [mean_t E_s[seq_0] | mean_t E_s[seq_1]]   (nets/utils.py:56-77: ONE table for both sequences)
        context  = ELU([sequence | dense | category] Wc + bc)   (256)
        logits   = context Wo + bo + max(log(mask), float32.min) ;  value = context Wv + bv
    This is the functional twin for `*_rawstate` algorithms: plain torch ops + autograd (no hand-written kernel -- it is not
    on the benchmarked path; the 25.6 M-parameter embedding tables make its SGD step an HBM-bound dense Adam update).
    Observations travel through the trainer as ONE packed f32 row [cat 21 | dense 432 | seq 128] (ids < 2^24 are exact)."""

    def __init__(self, action_size=284, device="cuda", seed=0, config=None):
        cfg = config or {}
        self.A = action_size
        self.device = torch.device(device)
        self.H, self.E, self.U = cfg.get("category_hash_size", 100000), cfg.get("emb_size", 128), cfg.get("hidden_units", 128)
        self.C, self.D = cfg.get("category_feature_num", 21), cfg.get("dense_feature_num", 432)
        self.S, self.L = cfg.get("seq_num", 2), cfg.get("maxlen", 64)
        self.obs_dim = self.C + self.D + self.S * self.L
        E, U = self.E, self.U
        shapes = [("emb_cat", (self.H, E)), ("emb_seq", (self.H, E)), ("dw1", (self.D, U)), ("db1", (U,)), ("dw2", (U, U)),
                  ("db2", (U,)), ("wc", (self.S * E + U + E, 256)), ("bc", (256,)), ("w2", (256, action_size)),
                  ("b2", (action_size,)), ("wv", (256, 1)), ("bv", (1,))]
        n = sum(math.prod(s) for _, s in shapes)
        g = torch.Generator(device="cpu").manual_seed(seed)
        self.flat = torch.zeros(n, dtype=torch.float32, device=self.device, requires_grad=True)
        off = 0
        with torch.no_grad():
            for name, shape in shapes:
                k = math.prod(shape)
                v = self.flat[off:off + k].view(shape)
                if name.startswith("emb_"):            # Keras Embedding: uniform(-0.05, 0.05)
                    v.copy_(((torch.rand(shape, generator=g) - 0.5) * 0.1).to(self.device))
                elif name in ("w2", "wv"):             # normc_initializer(0.01)
                    w = torch.randn(shape, generator=g)
                    v.copy_((w * 0.01 / w.pow(2).sum(0, keepdim=True).sqrt()).to(self.device))
                elif len(shape) == 2:                  # Keras Dense: glorot uniform
                    lim = math.sqrt(6.0 / (shape[0] + shape[1]))
                    v.copy_(((torch.rand(shape, generator=g) * 2 - 1) * lim).to(self.device))
                off += k
        self._shapes, self.n_params = shapes, n

    params = MaskedPolicy.params

    def pack(self, obs):
        """env observation dict (rawstate_as_obs, torch format) -> packed f32 [B, 581]."""
        B = obs["category_feature"].shape[0]
        return torch.cat([obs["category_feature"].reshape(B, -1).to(torch.float32), obs["dense_feature"].reshape(B, -1).to(torch.float32),
                          obs["sequence_feature"].reshape(B, -1).to(torch.float32)], dim=1)

    def inputs(self, obs):
        return self.pack(obs), obs["action_mask"]

    def forward(self, obs, mask):
        p = self.params()
        C, D = self.C, self.D
        cat = obs[:, :C].long()
        dense = obs[:, C:C + D]
        seq = obs[:, C + D:].long().view(-1, self.S, self.L)
        elu = torch.nn.functional.elu
        cfeat = torch.nn.functional.embedding(cat, p["emb_cat"]).mean(dim=1)
        x = elu(elu(dense @ p["dw1"] + p["db1"]) @ p["dw2"] + p["db2"])
        sfeat = torch.cat([torch.nn.functional.embedding(seq[:, i], p["emb_seq"]).mean(dim=1) for i in range(self.S)], dim=1)
        ctx = elu(torch.cat([sfeat, x, cfeat], dim=1) @ p["wc"] + p["bc"])
        logits = ctx @ p["w2"] + p["b2"]
        inf_mask = torch.clamp(torch.log(mask.to(torch.float32)), min=FLOAT_MIN)
        return logits + inf_mask, (ctx @ p["wv"] + p["bv"]).squeeze(-1)

    act, terms = MaskedPolicy.act, MaskedPolicy.terms
