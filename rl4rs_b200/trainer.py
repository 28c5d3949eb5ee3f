"""Model-free trainers over the GPU-resident env: PPO and A2C (the two algorithms of BASELINE
configs 2, 3 and 5), mirroring ``script/modelfree_trainer.py:get_rl_model`` + the hyper-parameters of
``script/modelfree_train.py:179-217`` (PPO), ``:248-304`` (A2C), ``:394-417`` (common).

Differences from the reference, by design (north_star):
  * rollouts never leave the GPU: obs / mask / action / logp / value / reward live in
    [T, B, ...] device buffers (no HTTP vector env, no Ray object store);
  * data parallel over env rows: every rank rolls its own shard and ONE ``all_reduce`` over the flat
    34 973-parameter gradient (~140 KB) per optimizer step is the only collective
    (NCCL over NVLink on GPUs; gloo in the CPU tests).
On a CUDA device the policy forward + sampling, the loss gradients (hand-derived backward) and Adam
are the library's own kernels (csrc/r4_ppo.cuh through the C-ABI: r4_policy_act / r4_policy_grad /
r4_adam_step), 2 launches per SGD step; the torch implementation below is kept as the CPU path of
the tests and as the autograd cross-check of the kernels (tests/test_gpu_trainer.py).

RLlib semantics kept: gamma = 1, GAE(lambda = 1) advantages from complete episodes, SoftQ(T=1)
exploration = sampling from softmax(masked logits), argmax for evaluation; PPO: standardised
advantages, clip 0.3, vf clip 500, vf coeff 0.5, adaptive KL (0.2 / target 0.01), minibatch 256,
one SGD epoch, Adam 1e-4; A2C: summed losses, vf coeff 0.5, entropy 0.01, grad-norm clip 10.
"""
import os

import ctypes as C

import torch
import torch.distributed as dist

from .policy import MaskedPolicy, RawStatePolicy


def _p(t, byte_offset=0):
    return C.c_void_p(t.data_ptr() + byte_offset) if t is not None else C.c_void_p(0)


class KernelOps(object):
    """ctypes front of the K12 kernels (include/rl4rs_b200.h: r4_policy_act / r4_policy_grad / r4_adam_step)."""

    def __init__(self, A, device, n_params):
        from . import _capi
        self.capi = _capi
        self.lib = _capi.load_library()
        self.A, self.device, self.n = A, device, n_params
        assert self.lib.r4_policy_num_params(A) == n_params
        z = lambda k: torch.zeros(k, dtype=torch.float32, device=device)
        self.m, self.v, self.grad, self.stats, self.norm = z(n_params), z(n_params), z(n_params), z(5), z(1)
        self.sms = torch.cuda.get_device_properties(device).multi_processor_count   # grid cap of the learner kernels
        self.scratch = z(self.sms * (n_params + 5))
        self.step = 0
        self.counter = 0
        self.launches = 0                # kernels launched through this object (bench.py: gpu_launches)

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _check(self, rc, what):
        if rc != 0:
            raise self.capi.R4Error("%s failed (%d): %s" % (what, rc, (self.lib.r4_last_error(None) or b"?").decode()))

    def act(self, flat, obs, mask, explore, seed, action_i32, logp, value, logits):
        n = obs.shape[0]
        rc = self.lib.r4_policy_act(_p(flat), _p(obs), _p(mask), n, self.A, int(bool(explore)), seed, self.counter,
                                    _p(action_i32), _p(logp), _p(value), _p(logits), self._stream())
        self._check(rc, "r4_policy_act")
        self.counter += n
        self.launches += 1

    def policy_grad(self, mode, flat, data, idx, idx_offset, n, hp, inv_n, stat_scale, G=None):
        obs, mask, act, logp, logits, val, adv, target = data
        G = G or max(1, min((n + 3) // 4, self.sms))          # 4 samples per CTA tile (r4_ppo.cuh: TS)
        rc = self.lib.r4_policy_grad(mode, _p(flat), _p(obs), _p(mask), _p(act), _p(logp), _p(logits), _p(val), _p(adv),
                                     _p(target), _p(idx, idx_offset * 8) if idx is not None else C.c_void_p(0), n, self.A,
                                     hp["clip"], hp["vf_clip"], hp["vf_coeff"], hp["kl_coeff"], hp["ent_coeff"], inv_n,
                                     _p(self.scratch), G, _p(self.grad), _p(self.stats), stat_scale, self._stream())
        self._check(rc, "r4_policy_grad")
        self.launches += 2               # k_policy_grad + k_grad_reduce

    def ppo_epoch(self, flat, data, perm, n, mb, hp, lr, clip):
        """All minibatch steps of one SGD epoch in ONE library call (single-GPU learner)."""
        obs, mask, act, logp, logits, val, adv, target = data
        rc = self.lib.r4_ppo_epoch(_p(flat), _p(obs), _p(mask), _p(act), _p(logp), _p(logits), _p(val), _p(adv), _p(target),
                                   _p(perm), n, mb, self.A, hp["clip"], hp["vf_clip"], hp["vf_coeff"], hp["kl_coeff"],
                                   hp["ent_coeff"], _p(self.scratch), _p(self.grad), _p(self.stats), _p(self.m), _p(self.v),
                                   self.step, lr, 0.9, 0.999, 1e-8, float(clip or 0.0), _p(self.norm), self._stream())
        if rc < 0:
            self._check(rc, "r4_ppo_epoch")
        self.step += rc
        self.launches += rc * (4 if clip else 2)   # k_policy_grad + k_reduce_adam, or + k_grad_reduce, k_sumsq, k_adam
        return rc

    def ppo_epoch_dist(self, comm, flat, data, perm, n, mb_local, hp, lr):
        """All minibatch steps of one SGD epoch of a data-parallel learner in ONE library call: per step the gradient
        kernel + the fused peer-memory exchange / Adam kernel (csrc/r4_comm.cuh); no NCCL, no host round trip."""
        obs, mask, act, logp, logits, val, adv, target = data
        rc = self.lib.r4_ppo_epoch_dist(comm.h, _p(flat), _p(obs), _p(mask), _p(act), _p(logp), _p(logits), _p(val), _p(adv),
                                        _p(target), _p(perm), n, mb_local, self.A, hp["clip"], hp["vf_clip"], hp["vf_coeff"],
                                        hp["kl_coeff"], hp["ent_coeff"], _p(self.scratch), _p(self.grad), _p(self.stats),
                                        _p(self.m), _p(self.v), self.step, lr, 0.9, 0.999, 1e-8, self._stream())
        if rc < 0:
            self._check(rc, "r4_ppo_epoch_dist")
        self.step += rc
        self.launches += rc * 2          # k_policy_grad + k_exchange_adam
        return rc

    def policy_grad_exchange(self, comm, mode, flat, data, n, hp, inv_n, stat_scale):
        """One gradient over n local samples, summed over the ranks through peer memory into self.grad (A2C)."""
        obs, mask, act, logp, logits, val, adv, target = data
        G = max(1, min((n + 3) // 4, self.sms))
        rc = self.lib.r4_policy_grad_partial(mode, _p(flat), _p(obs), _p(mask), _p(act), _p(logp), _p(logits), _p(val), _p(adv),
                                             _p(target), C.c_void_p(0), n, self.A, hp["clip"], hp["vf_clip"], hp["vf_coeff"],
                                             hp["kl_coeff"], hp["ent_coeff"], inv_n, _p(self.scratch), G, self._stream())
        self._check(rc, "r4_policy_grad_partial")
        rc = self.lib.r4_grad_exchange(comm.h, _p(self.scratch), G, self.A, _p(self.grad), _p(self.stats), stat_scale, self._stream())
        self._check(rc, "r4_grad_exchange")
        self.launches += 2

    def gae(self, reward, value, gamma, lam):
        """-> (target, adv) of a [T, B] rollout in one launch (r4_gae)."""
        adv, target = torch.empty_like(reward), torch.empty_like(reward)
        rc = self.lib.r4_gae(_p(reward), _p(value), reward.shape[0], reward.shape[1], gamma, gamma * lam, _p(adv), _p(target), self._stream())
        self._check(rc, "r4_gae")
        self.launches += 1
        return target, adv

    def adam(self, flat, lr, grad_scale, clip):
        self.step += 1
        rc = self.lib.r4_adam_step(_p(flat), _p(self.grad), _p(self.m), _p(self.v), self.n, self.step, lr, 0.9, 0.999,
                                   1e-8, grad_scale, float(clip or 0.0), _p(self.norm), self._stream())
        self._check(rc, "r4_adam_step")
        self.launches += 2 if clip else 1

class PeerComm(object):
    """The learner's gradient exchange over NVLink peer memory (include/rl4rs_b200.h: r4_comm_*).  Every rank exports
    its inbox with cudaIpcGetMemHandle; the 64-byte handles are all-gathered ONCE through torch.distributed; after that
    the SGD steps use no host-side collective.  ``ok`` is False (on every rank) when peer mapping is not possible on this
    box -- the trainer then keeps the NCCL all-reduce per step and says so."""

    def __init__(self, n_params, device):
        from . import _capi
        self.lib = _capi.load_library()
        self.h, self.ok, self.why = None, False, ""
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() < 2 or device.type != "cuda":
            return
        rank, world = dist.get_rank(), dist.get_world_size()
        if os.environ.get("R4_NO_PEER_COMM"):
            self.why = "disabled by R4_NO_PEER_COMM"
            return
        h = C.c_void_p()
        good = self.lib.r4_comm_create(rank, world, n_params, C.byref(h)) == 0
        buf = (C.c_uint8 * 64)()
        good = good and self.lib.r4_comm_handle(h, buf) == 0
        mine = torch.tensor(list(buf), dtype=torch.uint8, device=device)
        every = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(every, mine)
        if good:
            blob = torch.cat(every).cpu().numpy().tobytes()
            good = self.lib.r4_comm_open(h, blob, world) == 0
        if not good:
            self.why = (self.lib.r4_last_error(None) or b"?").decode()
        flag = torch.tensor([1 if good else 0], device=device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)            # all ranks take the same path
        self.ok = bool(flag.item())
        if self.ok:
            self.h = h
        elif h:
            self.lib.r4_comm_destroy(h)
        if not self.ok and rank == 0:
            import sys
            sys.stderr.write("rl4rs_b200: peer-memory gradient exchange unavailable (%s); using NCCL all-reduce per SGD step\n" % self.why)

    def close(self):
        if self.h:
            self.lib.r4_comm_destroy(self.h)
            self.h = None


PPO_DEFAULTS = {"gamma": 1.0, "lambda": 1.0, "kl_coeff": 0.2, "sgd_minibatch_size": 256, "num_sgd_iter": 1,
                "lr": 1e-4, "vf_loss_coeff": 0.5, "clip_param": 0.3, "vf_clip_param": 500.0, "kl_target": 0.01,
                "entropy_coeff": 0.0, "grad_clip": None, "shuffle_sequences": True}
A2C_DEFAULTS = {"gamma": 1.0, "lambda": 1.0, "grad_clip": 10.0, "lr": 1e-4, "vf_loss_coeff": 0.5,
                "entropy_coeff": 0.01}


def _world():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


class RolloutBuffer(object):
    """[T, B, ...] device-resident sample batch of one vector episode."""

    def __init__(self, T, B, A, device, obs_dim=256):
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        self.obs, self.mask = z(T, B, obs_dim), z(T, B, A, dt=torch.uint8)
        self.action, self.logp, self.value = z(T, B, dt=torch.int64), z(T, B), z(T, B)
        self.logits, self.reward = z(T, B, A), z(T, B)
        self.T, self.B = T, B

    def returns_and_advantages(self, gamma, lam):
        """GAE (RLlib compute_advantages, complete episodes => bootstrap value 0)."""
        T = self.T
        adv = torch.zeros_like(self.reward)
        last = torch.zeros_like(self.reward[0])
        for t in reversed(range(T)):
            nv = self.value[t + 1] if t + 1 < T else torch.zeros_like(self.value[0])
            delta = self.reward[t] + gamma * nv - self.value[t]
            last = delta + gamma * lam * last
            adv[t] = last
        return adv + self.value, adv


class _TrainerBase(object):
    algo = None

    def __init__(self, config, env, device=None, seed=0):
        """config: RLlib-style hyper-parameter dict (unknown keys ignored); env: a RecEnvBase built
        with output_format='torch' and support_rllib_mask=True (or any object with that protocol)."""
        self.config = dict(self.DEFAULTS, **{k: v for k, v in (config or {}).items() if k in self.DEFAULTS})
        self.env = env
        self.T = env.config["max_steps"]
        self.B = env.config["batch_size"]
        self.A = env.config["action_size"]
        self.device = torch.device(device) if device is not None else env.sim.engine.device
        # `*_rawstate` algorithms / rawstate_as_obs (modelfree_train.py:218,235-240,270,287-298): the policy embeds the raw
        # state itself ('mask_model_rawstate'); that twin is plain torch + autograd, the kernels serve the 256-d obs policy
        self.rawstate = bool(env.config.get("rawstate_as_obs", False))
        if self.rawstate:
            self.policy = RawStatePolicy(self.A, self.device, seed=seed, config=env.config)
        else:
            self.policy = MaskedPolicy(self.A, self.device, seed=seed)     # same init on every rank
        self.use_kernels = self.device.type == "cuda" and (config or {}).get("use_kernels", True) and not self.rawstate
        self.opt = torch.optim.Adam([self.policy.flat], lr=self.config["lr"])
        self.ops = KernelOps(self.A, self.device, self.policy.n_params) if self.use_kernels else None
        self.comm = PeerComm(self.policy.n_params, self.device) if self.use_kernels else None
        self._act_i32 = torch.zeros(self.B, dtype=torch.int32, device=self.device)
        # shared `seed` for the parameter init and the minibatch permutation; the exploration noise is per rank
        # (k_policy_act hashes seed ^ counter+row: the same seed would give rank r row i the noise of rank 0 row i)
        rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
        self._seed = (seed * 1000003 + rank) & 0x7fffffffffffffff
        if rank and not self.use_kernels:
            torch.manual_seed(seed * 1000003 + rank)
        self.buf = RolloutBuffer(self.T, self.B, self.A, self.device, obs_dim=self.policy.obs_dim if self.rawstate else 256)
        self.iteration = 0
        self.timesteps_total = 0

    # ---- rollout ------------------------------------------------------------------------------
    @torch.no_grad()
    def rollout(self, explore=True):
        env, buf = self.env, self.buf
        obs = env.reset()
        for t in range(self.T):
            buf.obs[t].copy_(self.policy.pack(obs) if self.rawstate else obs["obs"]); buf.mask[t].copy_(obs["action_mask"])
            if self.use_kernels:       # forward + sampling in ONE kernel, written straight into the rollout buffers
                a = self._act_i32
                self.ops.act(self.policy.flat, buf.obs[t], buf.mask[t], explore, self._seed, a,
                             buf.logp[t], buf.value[t], buf.logits[t])
                buf.action[t].copy_(a)
            else:
                a, logp, value, logits = self.policy.act(buf.obs[t], obs["action_mask"], explore=explore)
                buf.action[t].copy_(a); buf.logp[t].copy_(logp); buf.value[t].copy_(value); buf.logits[t].copy_(logits)
            obs, reward, done, info = env.step(a)
            buf.reward[t].copy_(reward)
        self.final_step = (obs, done)          # what the episode's last step returned
        return buf

    def _gae(self, buf):
        c = self.config
        lam = c.get("lambda", 1.0)
        if self.use_kernels and buf.reward.dtype == torch.float32 and buf.reward.is_contiguous() and buf.value.is_contiguous():
            return self.ops.gae(buf.reward, buf.value, c["gamma"], lam)
        return buf.returns_and_advantages(c["gamma"], lam)

    def _allreduce_grad(self, average):
        w = _world()
        if w > 1:
            dist.all_reduce(self.policy.flat.grad, op=dist.ReduceOp.SUM)     # the ONE collective
            if average:
                self.policy.flat.grad.div_(w)

    def _global_mean(self, x):
        x = x.detach().clone().to(torch.float64)
        if _world() > 1:
            dist.all_reduce(x, op=dist.ReduceOp.SUM)
            x /= _world()
        return float(x)

    def _global_means(self, named):
        """{name: 0-d tensor or float} -> {name: float mean over ranks}: ONE collective and ONE host synchronisation."""
        keys = list(named)
        x = torch.stack([torch.as_tensor(named[k], dtype=torch.float64, device=self.device).detach().reshape(()) for k in keys])
        if _world() > 1:
            dist.all_reduce(x, op=dist.ReduceOp.SUM)
            x /= _world()
        return dict(zip(keys, x.tolist()))

    def train(self):
        buf = self.rollout(explore=True)
        stats = self.learn(buf)
        self.iteration += 1
        self.timesteps_total += self.T * self.B * _world()
        ep_rew = stats.pop("_episode_reward_mean", None)
        if ep_rew is None:
            ep_rew = self._global_mean(buf.reward.sum(0).mean())
        stats.update({"episode_reward_mean": ep_rew, "training_iteration": self.iteration,
                      "timesteps_this_iter": self.T * self.B * _world(), "timesteps_total": self.timesteps_total,
                      "episodes_this_iter": self.B * _world()})
        return stats

    @torch.no_grad()
    def evaluate(self, episodes=1):
        """evaluation_config explore=False (modelfree_train.py:412-414): greedy episodes, mean reward."""
        tot = 0.0
        for _ in range(episodes):
            tot += float(self.rollout(explore=False).reward.sum(0).mean())
        return self._global_mean(torch.tensor(tot / episodes, device=self.device))

    @torch.no_grad()
    def compute_actions(self, obs, explore=False):
        """trainer.compute_actions (modelfree_train.py:454): obs = {'obs': [n,256], 'action_mask': [n,A]}
        (arrays or tensors) or RLlib's {i: {'obs':..,'action_mask':..}} dict."""
        import numpy as np
        if isinstance(obs, dict) and "action_mask" not in obs:      # RLlib's {env_id: observation} form
            keys = list(obs.keys())
            fields = [f for f in obs[keys[0]]]
            a = self.compute_actions({f: np.stack([np.asarray(obs[k][f]) for k in keys]) for f in fields}, explore)
            return dict(zip(keys, a.tolist()))
        if self.rawstate:
            o = self.policy.pack({k: torch.as_tensor(obs[k], device=self.device) for k in ("category_feature", "dense_feature", "sequence_feature")})
        else:
            o = torch.as_tensor(obs["obs"], dtype=torch.float32, device=self.device).contiguous()
        m = torch.as_tensor(obs["action_mask"], device=self.device)
        if self.use_kernels:
            n = o.shape[0]
            a = torch.empty(n, dtype=torch.int32, device=self.device)
            lp, v = torch.empty(n, device=self.device), torch.empty(n, device=self.device)
            self.ops.act(self.policy.flat, o, m.to(torch.uint8).contiguous(), explore, self._seed, a, lp, v, None)
            return a.cpu().numpy()
        a, _, _, _ = self.policy.act(o, m, explore=explore)
        return a.cpu().numpy()

    # ---- checkpoint / resume (trainer.save / restore, modelfree_train.py:421-435) -----------------
    def save(self, checkpoint_dir):
        os.makedirs(checkpoint_dir, exist_ok=True)
        path = os.path.join(checkpoint_dir, "checkpoint_%06d.pt" % self.iteration)
        kst = None
        if self.use_kernels:
            kst = {"m": self.ops.m.cpu(), "v": self.ops.v.cpu(), "step": self.ops.step}
        torch.save({"algo": self.algo, "flat": self.policy.flat.detach().cpu(), "opt": self.opt.state_dict(), "kernel_adam": kst,
                    "iteration": self.iteration, "timesteps_total": self.timesteps_total,
                    "extra": self._extra_state()}, path)
        return path

    def restore(self, path):
        st = torch.load(path, map_location="cpu")
        assert st["algo"] == self.algo
        with torch.no_grad():
            self.policy.flat.copy_(st["flat"].to(self.device))
        self.opt.load_state_dict(st["opt"])
        if self.use_kernels and st.get("kernel_adam"):
            k = st["kernel_adam"]
            self.ops.m.copy_(k["m"]); self.ops.v.copy_(k["v"]); self.ops.step = k["step"]
        self.iteration, self.timesteps_total = st["iteration"], st["timesteps_total"]
        self._load_extra_state(st["extra"])

    def _extra_state(self):
        return {}

    def _load_extra_state(self, s):
        pass


class PPOTrainer(_TrainerBase):
    algo = "PPO"
    DEFAULTS = PPO_DEFAULTS

    def __init__(self, config, env, device=None, seed=0):
        super().__init__(config, env, device, seed)
        self.kl_coeff = self.config["kl_coeff"]
        # minibatch permutations are drawn on the device the rollout lives on (a CPU randperm + copy stalled the GPU ~1 ms per epoch)
        self._gen = torch.Generator(device=self.device if self.device.type == "cuda" else "cpu").manual_seed(seed)

    def loss(self, obs, mask, action, old_logp, old_logits, old_value, adv, target):
        """RLlib 1.5 ppo_surrogate_loss."""
        c = self.config
        logits, value = self.policy.forward(obs, mask)
        logp_all = torch.log_softmax(logits, -1)
        logp = logp_all.gather(1, action.unsqueeze(1)).squeeze(1)
        old_logp_all = torch.log_softmax(old_logits, -1)
        p_old = old_logp_all.exp()
        kl = (p_old * (old_logp_all - logp_all)).sum(-1)
        entropy = -(logp_all.exp() * logp_all).sum(-1)
        ratio = torch.exp(logp - old_logp)
        surr = torch.min(adv * ratio, adv * torch.clamp(ratio, 1 - c["clip_param"], 1 + c["clip_param"]))
        vf1 = (value - target) ** 2
        vclip = old_value + torch.clamp(value - old_value, -c["vf_clip_param"], c["vf_clip_param"])
        vf = torch.max(vf1, (vclip - target) ** 2)
        total = (-surr + self.kl_coeff * kl + c["vf_loss_coeff"] * vf - c["entropy_coeff"] * entropy).mean()
        return total, {"policy_loss": (-surr).mean(), "vf_loss": vf.mean(), "kl": kl.mean(), "entropy": entropy.mean()}

    def learn(self, buf):
        c = self.config
        target, adv = self._gae(buf)
        n = buf.T * buf.B
        flat = lambda x: x.reshape((n,) + x.shape[2:])
        obs, mask, act = flat(buf.obs), flat(buf.mask), flat(buf.action)
        logp, logits, val = flat(buf.logp), flat(buf.logits), flat(buf.value)
        adv, target = flat(adv), flat(target)
        # StandardizeFields(["advantages"]) over the whole (global) train batch
        mean, sq = adv.mean(), (adv ** 2).mean()
        if _world() > 1:
            ms = torch.stack([mean, sq]); dist.all_reduce(ms); ms /= _world(); mean, sq = ms[0], ms[1]
        adv = (adv - mean) / torch.clamp((sq - mean ** 2).clamp_min(0).sqrt(), min=1e-4)
        # RLlib: sgd_minibatch_size is the TOTAL over devices; every rank contributes sgd_minibatch_size / world samples
        # of its own shard to each SGD step (multi-GPU tower semantics) and the loss is the mean over all of them
        mb = min(max(c["sgd_minibatch_size"] // _world(), 1), n)
        data = (obs, mask, act, logp, logits, val, adv, target)
        agg, steps = (self._sgd_kernels if self.use_kernels else self._sgd_eager)(data, n, mb)
        named = {k: v / max(steps, 1) for k, v in agg.items()}
        named["_episode_reward_mean"] = buf.reward.sum(0).mean()
        out = self._global_means(named)
        # adaptive KL (RLlib KLCoeffMixin.update_kl)
        if out.get("kl", 0.0) > 2.0 * c["kl_target"]:
            self.kl_coeff *= 1.5
        elif out.get("kl", 0.0) < 0.5 * c["kl_target"]:
            self.kl_coeff *= 0.5
        out.update({"cur_kl_coeff": self.kl_coeff, "sgd_steps": steps})
        return out

    def _perm(self, n, device):
        c = self.config
        if not c["shuffle_sequences"]:
            return torch.arange(n, device=device)
        return torch.randperm(n, generator=self._gen, device=self._gen.device).to(device)

    def _sgd_eager(self, data, n, mb):
        c = self.config
        agg, steps = {}, 0
        for _ in range(c["num_sgd_iter"]):
            perm = self._perm(n, data[0].device)
            for s in range(0, n - mb + 1, mb):
                idx = perm[s:s + mb]
                if self.policy.flat.grad is not None:
                    self.policy.flat.grad.zero_()
                total, st = self.loss(*[d[idx] for d in data])
                total.backward()
                self._allreduce_grad(average=True)
                if c["grad_clip"]:
                    torch.nn.utils.clip_grad_norm_([self.policy.flat], c["grad_clip"])
                self.opt.step()
                steps += 1
                for k, v in st.items():
                    agg[k] = agg.get(k, 0.0) + v.detach()
                agg["total_loss"] = agg.get("total_loss", 0.0) + total.detach()
        return agg, steps

    def _sgd_kernels(self, data, n, mb):
        """Per minibatch: the gradient kernel (forward, RLlib surrogate loss, hand-derived backward) and ONE kernel that
        reduces, exchanges over peer memory (N > 1) and applies Adam -- the whole epoch is one library call
        (r4_ppo_epoch / r4_ppo_epoch_dist).  Fallback without peer memory: NCCL all-reduce between two launches."""
        c = self.config
        ops = self.ops
        data = tuple(d.contiguous() for d in data)
        hp = {"clip": c["clip_param"], "vf_clip": c["vf_clip_param"], "vf_coeff": c["vf_loss_coeff"],
              "kl_coeff": float(self.kl_coeff), "ent_coeff": c["entropy_coeff"]}
        ops.stats.zero_()
        steps = 0
        w = _world()
        for _ in range(c["num_sgd_iter"]):
            perm = self._perm(n, data[0].device).contiguous()
            if w == 1:
                steps += ops.ppo_epoch(self.policy.flat, data, perm, n, mb, hp, c["lr"], c["grad_clip"])
                continue
            if self.comm is not None and self.comm.ok and not c["grad_clip"]:
                steps += ops.ppo_epoch_dist(self.comm, self.policy.flat, data, perm, n, mb, hp, c["lr"])
                continue
            for s in range(0, n - mb + 1, mb):
                ops.policy_grad(0, self.policy.flat, data, perm, s, mb, hp, 1.0 / mb, 1.0 / mb)
                if w > 1:
                    dist.all_reduce(ops.grad, op=dist.ReduceOp.SUM)           # the ONE collective
                ops.adam(self.policy.flat, c["lr"], 1.0 / w, c["grad_clip"])
                steps += 1
        st = ops.stats
        agg = {"policy_loss": st[0], "vf_loss": st[1], "kl": st[2], "entropy": st[3], "total_loss": st[4]}
        return agg, steps

    def _extra_state(self):
        return {"kl_coeff": self.kl_coeff}

    def _load_extra_state(self, s):
        self.kl_coeff = s.get("kl_coeff", self.kl_coeff)


class A2CTrainer(_TrainerBase):
    algo = "A2C"
    DEFAULTS = A2C_DEFAULTS

    def loss(self, obs, mask, action, adv, target):
        """RLlib 1.5 A3CLoss: summed terms."""
        c = self.config
        logits, value = self.policy.forward(obs, mask)
        logp_all = torch.log_softmax(logits, -1)
        logp = logp_all.gather(1, action.unsqueeze(1)).squeeze(1)
        pi_loss = -(logp * adv).sum()
        vf_loss = 0.5 * ((value - target) ** 2).sum()
        entropy = -(logp_all.exp() * logp_all).sum()
        total = pi_loss + c["vf_loss_coeff"] * vf_loss - c["entropy_coeff"] * entropy
        return total, {"policy_loss": pi_loss, "vf_loss": vf_loss, "entropy": entropy}

    def learn(self, buf):
        c = self.config
        target, adv = self._gae(buf)
        n = buf.T * buf.B
        flat = lambda x: x.reshape((n,) + x.shape[2:])
        if self.use_kernels:
            ops, w = self.ops, _world()
            data = (flat(buf.obs), flat(buf.mask), flat(buf.action), None, flat(buf.logits), None,
                    flat(adv).contiguous(), flat(target).contiguous())
            hp = {"clip": 0.0, "vf_clip": 0.0, "vf_coeff": c["vf_loss_coeff"], "kl_coeff": 0.0, "ent_coeff": c["entropy_coeff"]}
            ops.stats.zero_()
            if w > 1 and self.comm is not None and self.comm.ok:
                ops.policy_grad_exchange(self.comm, 1, self.policy.flat, data, n, hp, 1.0, 1.0)   # summed over the ranks
            else:
                ops.policy_grad(1, self.policy.flat, data, None, 0, n, hp, 1.0, 1.0)
                if w > 1:
                    dist.all_reduce(ops.grad, op=dist.ReduceOp.SUM)            # summed loss over the global batch
            gn = ops.grad.norm()
            ops.adam(self.policy.flat, c["lr"], 1.0, c["grad_clip"])
            st = ops.stats
            g = self._global_means({"policy_loss": st[0], "vf_loss": st[1], "entropy": st[3], "total_loss": st[4], "gn": gn,
                                    "_episode_reward_mean": buf.reward.sum(0).mean()})
            return {"policy_loss": g["policy_loss"] * w, "vf_loss": g["vf_loss"] * w, "entropy": g["entropy"] * w,
                    "total_loss": g["total_loss"] * w, "grad_gnorm": g["gn"], "sgd_steps": 1,
                    "_episode_reward_mean": g["_episode_reward_mean"]}
        if self.policy.flat.grad is not None:
            self.policy.flat.grad.zero_()
        total, st = self.loss(flat(buf.obs), flat(buf.mask), flat(buf.action), flat(adv), flat(target))
        total.backward()
        self._allreduce_grad(average=False)          # summed loss over the global batch
        gn = torch.nn.utils.clip_grad_norm_([self.policy.flat], c["grad_clip"]) if c["grad_clip"] else torch.zeros(())
        self.opt.step()
        out = {k: self._global_mean(v) * _world() for k, v in st.items()}
        out.update({"total_loss": self._global_mean(total) * _world(), "grad_gnorm": float(gn), "sgd_steps": 1})
        return out


def get_rl_model(algo, rllib_config, env=None, **kw):
    """script/modelfree_trainer.py:11-36.  Only the algorithms of the BASELINE configs are built."""
    if algo in ("PPO", "PPO_rawstate"):        # '*_rawstate' = the same trainer on an env built with rawstate_as_obs (modelfree_train.py:55-56)
        return PPOTrainer(rllib_config, env, **kw)
    if algo in ("A2C", "A2C_rawstate"):
        return A2CTrainer(rllib_config, env, **kw)
    algo = algo.replace("_rawstate", "")
    assert algo in ("PPO", "DQN", "A2C", "A3C", "PG", "IMPALA", "TD3", "RAINBOW", "SLATEQ", "DDPG")
    raise NotImplementedError("%s is outside the hot-path scope (SURVEY.md section 2, row 11)" % algo)
