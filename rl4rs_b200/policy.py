"""The policy the reference trains on this env: RLlib's MyMaskActionsModel
(rl4rs/nets/rllib/rllib_mask_model.py:7-64): obs(256) -> FC 64 tanh -> 284 logits
+ max(log(action_mask), float32.min); the value head shares the 64-d hidden (vf_share_layers).

Exploration is RLlib SoftQ with temperature 1 = sample from softmax(logits)
(modelfree_train.py:398-402); evaluation uses argmax (explore=False, :412-414).
Parameters live in one flat f32 buffer so the data-parallel gradient all-reduce is ONE NCCL call
(SURVEY.md section 8e: 34 973 parameters ~ 140 KB).
"""
import math

import numpy as np
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


class ParametricQNetwork(object):
    """The parametric-action Q network of PA-DQN: for a row s and an item a the input is x = [obs(s) (256) | e(a) (D)], e(a)
    row a of the env's fixed item vectors emb [A, D] (engine.action_emb), through RLlib's default fcnet
    (fcnet_hiddens [256, 256], tanh): Dense 256 tanh -> Dense 256 tanh -> Dense 1; normc(1.0) hidden kernels, normc(0.01)
    output kernel, zero biases.  The masked values are Qm(s, a) = Q(s, a) where the mask is set and float32.min where it is
    not (MyMaskActionsModel's Q + max(log mask, float32.min), as a select).  One flat buffer (csrc/r4_padqn.cuh's layout)
    and a target copy of it.  This torch twin is the CPU path of PADQNTrainer and the autograd cross-check of the kernels
    (tests/test_gpu_trainer_padqn.py)."""

    H = 256

    def __init__(self, emb, device="cuda", seed=0):
        self.device = torch.device(device)
        self.emb = torch.as_tensor(emb, dtype=torch.float32).to(self.device).contiguous()
        self.A, self.D = self.emb.shape
        H, K = self.H, OBS + self.D
        shapes = [("w1", (K, H)), ("b1", (H,)), ("w2", (H, H)), ("b2", (H,)), ("w3", (H, 1)), ("b3", (1,))]
        n = sum(math.prod(s) for _, s in shapes)
        g = torch.Generator(device="cpu").manual_seed(seed)
        self.flat = torch.zeros(n, dtype=torch.float32, device=self.device, requires_grad=True)
        self.slices, off = [], 0
        with torch.no_grad():
            for name, shape in shapes:
                k = math.prod(shape)
                if len(shape) == 2:                    # normc_initializer(1.0), 0.01 for the output layer
                    w = torch.randn(shape, generator=g)
                    std = 0.01 if name == "w3" else 1.0
                    self.flat[off:off + k].view(shape).copy_((w * std / w.pow(2).sum(0, keepdim=True).sqrt()).to(self.device))
                self.slices.append((off, off + k))
                off += k
        self._shapes, self.n_params = shapes, n
        self.target = self.flat.detach().clone()

    params = DeterministicActorCritic.params
    clip_per_tensor = DistributionalQNetwork.clip_per_tensor

    def inputs(self, obs):
        """env observation {'obs', 'action_mask'} -> (obs, mask)."""
        return obs["obs"], obs["action_mask"]

    def q_pairs(self, obs, action, flat=None):
        """Q(s, a) [n] of the n pairs (obs [n, 256], action [n])."""
        p = self.params(flat)
        x = torch.cat([obs, self.emb[action.long()]], dim=1)
        h = torch.tanh(torch.tanh(x @ p["w1"] + p["b1"]) @ p["w2"] + p["b2"])
        return (h @ p["w3"] + p["b3"]).squeeze(-1)

    def forward(self, obs, mask, flat=None):
        """obs f32 [n, 256], mask {0, 1} [n, A] -> Qm [n, A], through the split first layer (S[s] + P[a]) in row chunks."""
        p = self.params(flat)
        S = obs @ p["w1"][:OBS] + p["b1"]
        P = self.emb @ p["w1"][OBS:]
        out = []
        for i in range(0, obs.shape[0], 64):
            h = torch.tanh(torch.tanh(S[i:i + 64, None, :] + P[None]) @ p["w2"] + p["b2"])
            out.append((h @ p["w3"] + p["b3"]).squeeze(-1))
        q = torch.cat(out) if out else S.new_zeros(0, self.A)
        return torch.where(mask.to(torch.bool), q, torch.full_like(q, FLOAT_MIN))

    def loss(self, obs, action, reward, new_obs, done, next_mask, weights=None, gamma=1.0, inv_n=None):
        """The double-Q Huber loss sum_i w_i huber(td_i) * inv_n (default 1/n), td = Q(s, a) - (r + gamma (1 - done)
        Qm_target(s', argmax Qm_online(s', .))) -> (loss, td [n], Q(s, a) [n])."""
        n = obs.shape[0]
        inv_n = 1.0 / n if inv_n is None else inv_n
        rows = torch.arange(n, device=obs.device)
        with torch.no_grad():
            a_star = self.forward(new_obs, next_mask).argmax(1)
            qt = self.forward(new_obs, next_mask, self.target)[rows, a_star]
            y = reward.to(torch.float32) + gamma * (1.0 - done.to(torch.float32)) * qt
        q = self.q_pairs(obs, action)
        td = q - y
        w = torch.ones(n, device=obs.device) if weights is None else weights
        hub = torch.where(td.abs() <= 1.0, 0.5 * td * td, td.abs() - 0.5)
        return (w * hub).sum() * inv_n, td.detach(), q.detach()

    @torch.no_grad()
    def act(self, obs, mask, explore, seed=0, counter=0):
        """-> (action i32 [n], Qm [n, A]): the first argmax of Qm, or SoftQ over csrc/r4_padqn.cuh's uniform per row."""
        import numpy as np
        q = self.forward(obs, mask)
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


class BatchRLFlat(object):
    """The flat parameter vector of the batch-RL twins, in their kernels' layout, and its named views."""

    def _init_flat(self, shapes, seed, fixed=None):
        """self.flat for `shapes` [(name, shape)] in layout order, drawn from a CPU generator seeded with `seed`: a name in
        `fixed` is filled with its value and draws nothing, a name ending in 'emb' is drawn N(0, 1) (torch's Embedding),
        the rest torch's default U(+-1/sqrt(fan_in)) (Linear), a bias with the fan of the weight before it."""
        fixed = fixed or {}
        n = sum(math.prod(s) for _, s in shapes)
        g = torch.Generator(device="cpu").manual_seed(seed)
        self.flat = torch.zeros(n, dtype=torch.float32, device=self.device, requires_grad=True)
        off, fan = 0, 1
        with torch.no_grad():
            for name, shape in shapes:
                k = math.prod(shape)
                v = self.flat[off:off + k].view(shape)
                if name in fixed:
                    v.fill_(fixed[name])
                elif name.endswith("emb"):
                    v.copy_(torch.randn(shape, generator=g).to(self.device))
                else:
                    fan = shape[0] if len(shape) == 2 else fan          # a bias follows its weight
                    bound = 1.0 / math.sqrt(fan)
                    v.copy_(((torch.rand(shape, generator=g) * 2 - 1) * bound).to(self.device))
                off += k
        self._shapes, self.n_params = shapes, n

    def params(self, flat=None):
        """name -> its view of flat (default self.flat); a shorter vector (BCQ's target) gives the names it holds."""
        flat = self.flat if flat is None else flat
        out, off = {}, 0
        for name, shape in self._shapes:
            k = math.prod(shape)
            if off + k > flat.numel():
                break
            out[name] = flat[off:off + k].view(shape)
            off += k
        return out


class BatchRLNet(BatchRLFlat):
    """The networks of the discrete batch-RL learners (script/batchrl_trainer.py:34-90, d3rlpy 0.91 as the script configures
    it), in csrc/r4_batchrl.cuh's flat layout.  The masked net M (BC's imitator; BCQ's Q function and, separately, its
    imitator) is rl4rs/nets/cql/encoder.py CustomVectorEncoder with_q plus d3rlpy's Linear(A, A) head:
        h = relu(x W1 + b1) [256] ; e = flatten(Emb[x[:, -10:]]) [10 x 32] (the 9 prev actions and cur_steps)
        f = ([h | e] W2 + b2), set to 0 where keep is 0 ; z = f W3 + b3
    keep: location_mask[cur_steps % 9 // 3], 0 for the 9 prev actions, and 0 for every special item of a row whose prev
    actions hold one.  CQL's plain net is d3rlpy's default encoder (256 relu, 256 relu) and Linear(256, A).  Init is torch's
    default (Linear: U(+-1/sqrt(fan_in)) for weight and bias; Embedding: N(0, 1)).  The target is a copy of the Q part
    (BCQ: its Q net; CQL: the whole net; BC has none).  This twin is the CPU path of rl4rs_b200.batchrl and the autograd
    cross-check of the kernels (tests/test_gpu_batchrl.py)."""

    H, E, W, PW = 256, 32, 10, 9
    ALGOS = ("BC", "BCQ", "CQL")

    def __init__(self, algo, obs_dim, location_mask, special_items, action_size=284, device="cuda", seed=0):
        assert algo in self.ALGOS
        self.algo, self.K, self.A = algo, int(obs_dim), int(action_size)
        self.device = torch.device(device)
        K, A, H, E, W = self.K, self.A, self.H, self.E, self.W

        def mnet(p):
            return [(p + "w1", (K, H)), (p + "b1", (H,)), (p + "emb", (A, E)), (p + "w2", (H + W * E, A)), (p + "b2", (A,)),
                    (p + "w3", (A, A)), (p + "b3", (A,))]
        cnet = [("w1", (K, H)), ("b1", (H,)), ("w2", (H, H)), ("b2", (H,)), ("w3", (H, A)), ("b3", (A,))]
        self._init_flat({"BC": mnet("i_"), "BCQ": mnet("q_") + mnet("i_"), "CQL": cnet}[algo], seed)
        self.n_target = {"BC": 0, "BCQ": self.n_params // 2, "CQL": self.n_params}[algo]
        self.target = self.flat.detach()[:self.n_target].clone()
        lm = torch.as_tensor(np.asarray(location_mask)[:3] >= 0.01, dtype=torch.uint8)
        self.location_mask = lm.to(self.device)
        sp = torch.zeros(A, dtype=torch.uint8)
        sp[torch.as_tensor(np.asarray(list(special_items), dtype=np.int64))] = 1
        self.special = sp.to(self.device)

    def keep(self, x):
        """bool [n, A]: the custom encoder's mask (encoder.py:43-65), the same as the eval rule's (policy_model.py:24-33)."""
        prev = x[:, -self.W:-1].to(torch.long)
        layer = x[:, -1].to(torch.long) % self.PW // 3
        mask = self.location_mask[layer].clone()
        mask.scatter_(1, prev, 0)
        has = self.special[prev].bool().any(1)
        mask[has.unsqueeze(1) & self.special.bool().unsqueeze(0)] = 0
        return mask.bool()

    def features(self, x, prefix, flat=None, keep=None):
        """The custom encoder's output (encoder.py:42-67 with_q): the masked features f [n, A] of the masked net."""
        p = self.params(flat)
        keep = self.keep(x) if keep is None else keep
        h = torch.relu(x @ p[prefix + "w1"] + p[prefix + "b1"])
        e = torch.nn.functional.embedding(x[:, -self.W:].to(torch.long), p[prefix + "emb"]).flatten(1)
        f = torch.cat([h, e], 1) @ p[prefix + "w2"] + p[prefix + "b2"]
        return torch.where(keep, f, torch.zeros_like(f))

    def mnet(self, x, prefix, flat=None, keep=None):
        """The masked net on x [n, K] -> z [n, A] (d3rlpy's Linear head on the encoder's features)."""
        p = self.params(flat)
        return self.features(x, prefix, flat, keep) @ p[prefix + "w3"] + p[prefix + "b3"]

    def cnet(self, x, flat=None):
        p = self.params(flat)
        h = torch.relu(torch.relu(x @ p["w1"] + p["b1"]) @ p["w2"] + p["b2"])
        return h @ p["w3"] + p["b3"]

    def q(self, x, flat=None):
        """The Q function (BCQ, CQL) [n, A]."""
        return self.cnet(x, flat) if self.algo == "CQL" else self.mnet(x, "q_", flat)

    def imitator(self, x, flat=None):
        """The imitator's logits (BC, BCQ) [n, A]."""
        return self.mnet(x, "i_", flat)

    def bcq_filtered(self, x, log_flex):
        """d3rlpy DiscreteBCQ's action rule: (Q - min Q) * [log pi - max log pi > log_flex] (first argmax picks)."""
        lp = torch.log_softmax(self.imitator(x), 1)
        mask = ((lp - lp.max(1, keepdim=True).values) > log_flex).to(torch.float32)
        q = self.q(x)
        return (q - q.min(1, keepdim=True).values) * mask

    def loss(self, obs, action, reward, next_obs, terminal, hp):
        """The minibatch loss of the algorithm -> (loss, stats [3]) in r4_batchrl_grad's statistics order.  hp: gamma, beta,
        alpha, log_flex, reward_mean, reward_den."""
        n = obs.shape[0]
        rows = torch.arange(n, device=obs.device)
        a = action.long()

        def huber(d):
            return torch.where(d.abs() < 1.0, 0.5 * d * d, d.abs() - 0.5)

        def bc_terms(z):
            nll = -torch.log_softmax(z, 1)[rows, a]
            pen = (z * z).mean(1)
            return nll + hp["beta"] * pen, nll, pen
        if self.algo == "BC":
            tot, nll, pen = bc_terms(self.imitator(obs))
            return tot.mean(), torch.stack([tot.mean(), nll.mean(), pen.mean()]).detach()
        with torch.no_grad():
            if self.algo == "BCQ":
                a_star = self.bcq_filtered(next_obs, hp["log_flex"]).argmax(1)
                r = reward
            else:
                a_star = self.q(next_obs).argmax(1)
                r = (reward - hp["reward_mean"]) / hp["reward_den"]
            qt = self.q(next_obs, self.target)[rows, a_star]
            y = r + hp["gamma"] * (1.0 - terminal.to(torch.float32)) * qt
        q = self.q(obs)
        qa = q[rows, a]
        td = huber(qa - y)
        if self.algo == "BCQ":
            tot = td + bc_terms(self.imitator(obs))[0]
        else:
            tot = td + hp["alpha"] * (torch.logsumexp(q, 1) - qa)
        return tot.mean(), torch.stack([tot.mean(), td.mean(), qa.mean()]).detach()

    @torch.no_grad()
    def act(self, obs, mode=0, log_flex=math.log(0.3)):
        """r4_batchrl_act's rule -> (action i32 [n], action_probs [n, A], raw output [n, A]).  mode 0: predict_with_mask
        (policy_model.py:17-36); mode 1: d3rlpy's predict."""
        x = obs.to(torch.float32)
        raw = self.imitator(x) if self.algo == "BC" else self.q(x)
        probs = torch.log_softmax(raw, 1) if self.algo == "BC" else torch.softmax(raw, 1)
        if mode == 0:
            pick = torch.where(self.keep(x), probs, torch.full_like(probs, -2.0 ** 15))
        elif self.algo == "BCQ":
            pick = self.bcq_filtered(x, log_flex)
        else:
            pick = probs
        return pick.argmax(1).to(torch.int32), probs, raw


def cqlc_draws(seed, counter, stream, rows, samples, dims, uniform=None):
    """The noise of csrc/r4_cqlconti.cuh for one stream of one step: splitmix64(splitmix64(seed ^ splitmix64(counter << 3 |
    stream)) ^ (row << 24 | sample << 12 | dim)) -> float64 [rows, samples, dims]: uniform in [-1, 1) for the uniform
    streams (2 and 4), else standard normal (Box-Muller on (2 hi + 1) / 2^25, hi the top 24 bits, and bits 16..39)."""
    import numpy as np
    assert samples <= 4096 and dims <= 4096
    with np.errstate(over="ignore"):
        base = _splitmix64(np.uint64(seed) ^ _splitmix64(np.uint64((int(counter) << 3) | int(stream))))
        r = np.arange(rows, dtype=np.uint64)[:, None, None] << np.uint64(24)
        s = np.arange(samples, dtype=np.uint64)[None, :, None] << np.uint64(12)
        d = np.arange(dims, dtype=np.uint64)[None, None, :]
        x = _splitmix64(base ^ (r | s | d))
    hi = (x >> np.uint64(40)).astype(np.float64)
    if (stream in (2, 4)) if uniform is None else uniform:
        return hi * (2.0 / 16777216.0) - 1.0
    u1 = (2.0 * hi + 1.0) / 33554432.0
    u2 = ((x >> np.uint64(16)) & np.uint64(0xFFFFFF)).astype(np.float64) / 16777216.0
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


class BatchRLContiNet(BatchRLFlat):
    """The networks of continuous-action CQL (script/batchrl_trainer.py:61-73 'CQL-conti', d3rlpy 0.91 CQL with its default
    VectorEncoderFactory), in csrc/r4_cqlconti.cuh's flat layout:
        actor     obs [K] -> 256 relu -> 256 relu -> [mu | logstd] [2D]   (SquashedNormalPolicy; logstd clamped to [-20, 2])
        critic k  [obs | action] [K + D] -> 256 relu -> 256 relu -> Q [1]   (k = 0, 1)
        log_temp, log_alpha   (initial temperature and alpha 1.0)
    Init is torch's default (Linear: U(+-1/sqrt(fan_in)) for weight and bias).  The target is a copy of both critics.
    The noise enters explicitly (cqlc_draws), so the same draws drive this twin and the kernels.  This twin is the CPU
    path of rl4rs_b200.batchrl.ContinuousCQL and the autograd cross-check of the kernels (tests/test_gpu_batchrl_conti.py)."""

    H = 256
    STREAMS = ("temp", "alpha_policy", "alpha_uniform", "critic_policy", "critic_uniform", "actor")

    def __init__(self, obs_dim, action_dim, device="cuda", seed=0, initial_temperature=1.0, initial_alpha=1.0):
        self.K, self.D = int(obs_dim), int(action_dim)
        self.device = torch.device(device)
        K, D, H = self.K, self.D, self.H

        def net(p, n_in, n_out):
            return [(p + "w1", (n_in, H)), (p + "b1", (H,)), (p + "w2", (H, H)), (p + "b2", (H,)), (p + "w3", (H, n_out)),
                    (p + "b3", (n_out,))]
        shapes = net("a_", K, 2 * D) + net("q0_", K + D, 1) + net("q1_", K + D, 1) + [("log_temp", (1,)),
                                                                                        ("log_alpha", (1,))]
        self._init_flat(shapes, seed, {"log_temp": math.log(initial_temperature), "log_alpha": math.log(initial_alpha)})
        n = self.n_params
        size = {name: math.prod(s) for name, s in shapes}
        self.n_actor = sum(v for k, v in size.items() if k.startswith("a_"))
        self.n_critic = sum(v for k, v in size.items() if k.startswith("q0_"))
        self.t0, self.n_target = self.n_actor, 2 * self.n_critic
        self.lt, self.la = n - 2, n - 1
        self.target = self.flat.detach()[self.t0:self.t0 + self.n_target].clone()

    def target_params(self, target=None, dtype=None):
        """The target critics as a params() dict (q0_*, q1_*)."""
        t = self.target if target is None else target
        full = torch.zeros(self.n_params, dtype=dtype or t.dtype, device=t.device)
        full[self.t0:self.t0 + self.n_target] = t.to(full.dtype)
        return self.params(full)

    @staticmethod
    def _mlp(p, pre, x):
        h = torch.relu(x @ p[pre + "w1"] + p[pre + "b1"])
        return torch.relu(h @ p[pre + "w2"] + p[pre + "b2"]) @ p[pre + "w3"] + p[pre + "b3"]

    def actor(self, x, p):
        """-> (mu, the raw logstd), each [..., D]."""
        o = self._mlp(p, "a_", x)
        return o[..., :self.D], o[..., self.D:]

    @staticmethod
    def sample(mu, ls_raw, eps):
        """SquashedNormalPolicy.sample_with_log_prob with the given normal draws: -> (tanh(u), log pi [...]), u = mu +
        exp(clamp(logstd, -20, 2)) eps; log pi = Normal(mu, std).log_prob(u) - 2 (log 2 - u - softplus(-2 u)), summed."""
        ls = ls_raw.clamp(-20.0, 2.0)
        std = ls.exp()
        u = mu + std * eps
        logp = -((u - mu) ** 2) / (2 * std * std) - ls - 0.5 * math.log(2 * math.pi)
        jacob = 2 * (math.log(2) - u - torch.nn.functional.softplus(-2 * u))
        return torch.tanh(u), (logp - jacob).sum(-1)

    def critic(self, x, a, k, p):
        return self._mlp(p, "q%d_" % k, torch.cat([x, a], -1)).squeeze(-1)

    def predict(self, x, flat=None):
        """d3rlpy predict: tanh(mu) [n, D]."""
        return torch.tanh(self.actor(x, self.params(flat))[0])

    def predict_value(self, x, a, flat=None):
        """d3rlpy predict_value: the mean of the two critics [n]."""
        p = self.params(flat)
        return 0.5 * (self.critic(x, a, 0, p) + self.critic(x, a, 1, p))

    def noise(self, seed, step, n, S, dtype=torch.float32):
        """The six draws of step `step` (kernel streams 0..5) as tensors: temp and actor [n, D], the others [n, S, D]."""
        out = {}
        for st, name in enumerate(self.STREAMS):
            one = name in ("temp", "actor")
            d = cqlc_draws(seed, step, st, n, 1 if one else S, self.D)
            t = torch.from_numpy(d[:, 0] if one else d)
            out[name] = t.to(device=self.device, dtype=dtype)
        return out

    def conservative(self, p, obs, act, mu, ls, eps_p, unif, hp):
        """clamp(exp(log_alpha), 0, 1e6) mean_i sum_k (w (lse - Q_k(s, a)) - threshold) with lse the max-subtracted
        logsumexp over the S policy samples (minus their log-probs; mu and ls carry no gradient) and the S uniform ones
        (minus D log 0.5).  -> (the term, the per-row sum over critics before alpha)."""
        n, S = eps_p.shape[:2]
        a_p, lp_p = self.sample(mu[:, None], ls[:, None], eps_p)
        xr = obs[:, None].expand(n, S, obs.shape[-1])
        lrand = math.log(0.5 ** self.D)
        rows = 0
        for k in (0, 1):
            qp, qu, qd = self.critic(xr, a_p, k, p), self.critic(xr, unif, k, p), self.critic(obs, act, k, p)
            tv = torch.cat([qp - lp_p, qu - lrand], 1)
            mx = tv.max(1, keepdim=True).values.detach()
            lse = mx.squeeze(1) + torch.log(torch.exp(tv - mx).sum(1))
            rows = rows + hp["conservative_weight"] * (lse - qd) - hp["alpha_threshold"]
        alpha = p["log_alpha"][0].exp().clamp(0.0, 1e6)
        return alpha * rows.mean(), rows

    def losses(self, batch, noise, hp, flat=None, target=None):
        """The four losses of one step at one parameter vector (r4_cqlc_grad's definition): -> ({'temp', 'alpha', 'critic',
        'actor'} losses, stats [5]).  Each loss is to be differentiated for its own group only."""
        obs, act, rew, nobs, term = batch
        flat = self.flat if flat is None else flat
        p = self.params(flat)
        dt = flat.dtype
        obs, act, nobs = obs.to(dt), act.to(dt), nobs.to(dt)
        nz = {k: v.to(dt) for k, v in noise.items()}
        mu, ls = self.actor(obs, p)
        with torch.no_grad():
            _, lp_t = self.sample(mu, ls, nz["temp"])
        temp_loss = -(p["log_temp"][0].exp() * (lp_t - self.D)).mean()
        mu_d, ls_d = mu.detach(), ls.detach()
        cons_a, _ = self.conservative(p, obs, act, mu_d, ls_d, nz["alpha_policy"], nz["alpha_uniform"], hp)
        alpha_loss = -cons_a
        with torch.no_grad():
            tp = self.target_params(target, dt)
            a2 = torch.tanh(self.actor(nobs, p)[0])
            qt = torch.min(self.critic(nobs, a2, 0, tp), self.critic(nobs, a2, 1, tp))
            r = (rew.to(dt) - hp["reward_mean"]) / hp["reward_den"]
            y = r + hp["gamma"] * (1.0 - term.to(dt)) * qt
        q0 = self.critic(obs, act, 0, p)
        td = ((q0 - y) ** 2).mean() + ((self.critic(obs, act, 1, p) - y) ** 2).mean()
        cons_c, _ = self.conservative(p, obs, act, mu_d, ls_d, nz["critic_policy"], nz["critic_uniform"], hp)
        critic_loss = td + cons_c
        a_pi, lp_pi = self.sample(mu, ls, nz["actor"])
        qmin = torch.stack([self.critic(obs, a_pi, 0, p), self.critic(obs, a_pi, 1, p)]).min(0).values
        actor_loss = (p["log_temp"][0].exp() * lp_pi - qmin).mean()
        st = torch.stack([critic_loss, actor_loss, temp_loss, alpha_loss, q0.mean()]).detach()
        return {"temp": temp_loss, "alpha": alpha_loss, "critic": critic_loss, "actor": actor_loss}, st

    def group(self, name):
        """The slice of the flat vector the loss `name` updates."""
        return {"actor": slice(0, self.n_actor), "critic": slice(self.t0, self.t0 + self.n_target),
                "temp": slice(self.lt, self.lt + 1), "alpha": slice(self.la, self.la + 1)}[name]

    def grads(self, batch, noise, hp, flat=None, target=None):
        """r4_cqlc_grad: every group's gradient of its own loss at one parameter vector -> (grad [n_params], stats)."""
        flat = self.flat if flat is None else flat
        if not flat.requires_grad:
            flat = flat.detach().requires_grad_(True)
        losses, st = self.losses(batch, noise, hp, flat, target)
        g = torch.zeros_like(flat.detach())
        for name, loss in losses.items():
            sl = self.group(name)
            g[sl] = torch.autograd.grad(loss, flat, retain_graph=True)[0][sl]
        return g, st

    @torch.no_grad()
    def soft_update(self, tau):
        """target = tau * critics + (1 - tau) * target."""
        c = self.flat.detach()[self.t0:self.t0 + self.n_target]
        self.target.copy_(tau * c + (1.0 - tau) * self.target)


class BatchRLContiBCQNet(BatchRLContiNet):
    """The networks of continuous-action BCQ (script/batchrl_trainer.py:61-73 'BCQ-conti', d3rlpy 0.91 BCQ with its default
    VectorEncoderFactory), in csrc/r4_bcqconti.cuh's flat layout (each net 256 relu -> 256 relu -> out):
        actor     [obs | a] -> f [D];  pi(s, a) = clamp(a + flex tanh(f), -1, 1)   (DeterministicResidualPolicy)
        critic k  [obs | a] -> Q [1]   (k = 0, 1)
        encoder   [obs | a] -> [mu | logstd] [2 L] (logstd clamped to [-20, 2]);  decoder  [obs | z] -> tanh [D]
    Torch default init.  The target is a copy of [actor | critic 0 | critic 1].  The noise enters explicitly."""

    STREAMS = ("vae", "target", "actor")

    def __init__(self, obs_dim, action_dim, device="cuda", seed=0, latent_size=32):
        self.K, self.D, self.L = int(obs_dim), int(action_dim), int(latent_size)
        self.device = torch.device(device)
        K, D, L, H = self.K, self.D, self.L, self.H

        def net(p, n_in, n_out):
            return [(p + "w1", (n_in, H)), (p + "b1", (H,)), (p + "w2", (H, H)), (p + "b2", (H,)), (p + "w3", (H, n_out)),
                    (p + "b3", (n_out,))]
        shapes = net("a_", K + D, D) + net("q0_", K + D, 1) + net("q1_", K + D, 1) + net("e_", K + D, 2 * L) + \
            net("d_", K + L, D)
        self._init_flat(shapes, seed)
        size = {name: math.prod(s) for name, s in shapes}
        part = lambda pre: sum(v for k, v in size.items() if k.startswith(pre))
        self.n_actor, self.n_critic = part("a_"), part("q0_")
        self.t0, self.n_target = 0, self.n_actor + 2 * self.n_critic
        self.target = self.flat.detach()[:self.n_target].clone()

    def group(self, name):
        return {"actor": slice(0, self.n_actor), "critic": slice(self.n_actor, self.n_target),
                "imitator": slice(self.n_target, self.n_params)}[name]

    def perturb(self, p, pre, x, a, flex):
        """pi(x, a) = clamp(a + flex tanh(f([x | a])), -1, 1)."""
        return (a + flex * torch.tanh(self._mlp(p, pre, torch.cat([x, a], -1)))).clamp(-1.0, 1.0)

    def decode(self, p, x, z):
        return torch.tanh(self._mlp(p, "d_", torch.cat([x, z], -1)))

    def candidates(self, p, x, z, flex, tp=None):
        """The S perturbed, decoded actions of rows x [n, K] for latent draws z [n, S, L] (clamped to +-0.5), with the actor
        of tp (default p) -> [n, S, D]."""
        xr = x[:, None].expand(x.shape[0], z.shape[1], x.shape[1])
        a = self.decode(p, xr, z.clamp(-0.5, 0.5))
        return self.perturb(p if tp is None else tp, "a_", xr, a, flex)

    def noise(self, seed, step, n, S, dtype=torch.float32):
        out = {}
        for st, name in enumerate(self.STREAMS):
            d = cqlc_draws(seed, step, st, n, S if name == "target" else 1, self.L, uniform=False)
            out[name] = torch.from_numpy(d if name == "target" else d[:, 0]).to(device=self.device, dtype=dtype)
        return out

    def predict_noise(self, seed, counter, n, S, dtype=torch.float32):
        """The latent draws of one predict call (kernel stream 3) [n, S, L]."""
        return torch.from_numpy(cqlc_draws(seed, counter, 3, n, S, self.L, uniform=False)).to(self.device, dtype)

    def predict(self, x, z, hp, flat=None):
        """d3rlpy BCQ predict: the candidate with the largest Q_0 (the first on ties) -> [n, D]."""
        p = self.params(flat)
        c = self.candidates(p, x, z.to(x.dtype), hp["action_flexibility"])
        xr = x[:, None].expand(x.shape[0], c.shape[1], x.shape[1])
        q = self.critic(xr, c, 0, p)
        return c[torch.arange(x.shape[0], device=x.device), q.argmax(1)]

    def losses(self, batch, noise, hp, flat=None, target=None):
        """The three losses of one step at one parameter vector (r4_bcqc_grad's definition): -> ({'imitator', 'critic',
        'actor'}, stats [5] = imitator loss, critic loss, actor loss, mean Q_0(s, a), reconstruction mse)."""
        obs, act, rew, nobs, term = batch
        flat = self.flat if flat is None else flat
        p, dt = self.params(flat), flat.dtype
        obs, act, nobs = obs.to(dt), act.to(dt), nobs.to(dt)
        nz = {k: v.to(dt) for k, v in noise.items()}
        L, flex = self.L, hp["action_flexibility"]
        e = self._mlp(p, "e_", torch.cat([obs, act], -1))
        mu, ls = e[:, :L], e[:, L:].clamp(-20.0, 2.0)
        recon = self.decode(p, obs, mu + ls.exp() * nz["vae"])
        mse = ((recon - act) ** 2).mean()
        kl = (-ls + 0.5 * ((2 * ls).exp() + mu * mu) - 0.5).mean()
        imitator = mse + hp["beta"] * kl
        with torch.no_grad():
            tp = self.target_params(target, dt)
            c = self.candidates(p, nobs, nz["target"], flex, tp)
            xr = nobs[:, None].expand(nobs.shape[0], c.shape[1], nobs.shape[1])
            qa, qb = self.critic(xr, c, 0, tp), self.critic(xr, c, 1, tp)
            v = hp["lam"] * torch.minimum(qa, qb) + (1 - hp["lam"]) * torch.maximum(qa, qb)
            r = (rew.to(dt) - hp["reward_mean"]) / hp["reward_den"]
            y = r + hp["gamma"] * (1.0 - term.to(dt)) * v.max(1).values
        q0 = self.critic(obs, act, 0, p)
        critic = ((q0 - y) ** 2).mean() + ((self.critic(obs, act, 1, p) - y) ** 2).mean()
        with torch.no_grad():
            a_s = self.decode(p, obs, nz["actor"].clamp(-0.5, 0.5))
        actor = -self.critic(obs, self.perturb(p, "a_", obs, a_s, flex), 0, p).mean()
        st = torch.stack([imitator, critic, actor, q0.mean(), mse]).detach()
        return {"imitator": imitator, "critic": critic, "actor": actor}, st

    @torch.no_grad()
    def soft_update(self, tau):
        """target = tau * [actor | critics] + (1 - tau) * target."""
        self.target.copy_(tau * self.flat.detach()[:self.n_target] + (1.0 - tau) * self.target)
