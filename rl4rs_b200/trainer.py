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
the tests and as the autograd cross-check of the kernels (tests/test_gpu_trainer.py).  The Gaussian policy of the
continuous-action env (GaussPPOTrainer / GaussA2CTrainer) runs the same learner over csrc/r4_gauss.cuh (GaussKernelOps).

RLlib semantics kept: gamma = 1, GAE(lambda = 1) advantages from complete episodes, SoftQ(T=1)
exploration = sampling from softmax(masked logits), argmax for evaluation; PPO: standardised
advantages, clip 0.3, vf clip 500, vf coeff 0.5, adaptive KL (0.2 / target 0.01), minibatch 256,
one SGD epoch, Adam 1e-4; A2C: summed losses, vf coeff 0.5, entropy 0.01, grad-norm clip 10.
"""
import os

import ctypes as C

import torch
import torch.distributed as dist

from .policy import (DeterministicActorCritic, DistributionalQNetwork, GaussianPolicy, MaskedPolicy, RawStatePolicy,
                     counter_draws)


def _p(t, byte_offset=0):
    return C.c_void_p(t.data_ptr() + byte_offset) if t is not None else C.c_void_p(0)


def _hp(hp):
    """The loss hyper-parameters in the argument order of the gradient entry points."""
    return hp["clip"], hp["vf_clip"], hp["vf_coeff"], hp["kl_coeff"], hp["ent_coeff"]


class KernelOps(object):
    """ctypes front of the K12 kernels (include/rl4rs_b200.h: r4_policy_act / r4_policy_grad / r4_adam_step).  `data` is
    (obs, mask, action, logp, logits, value, adv, target), the argument order of the gradient entry points."""

    def __init__(self, A, device, n_params):
        self.A = A
        self._init(device, n_params)

    def _init(self, device, n_params):
        """The Adam, gradient and statistics buffers, the learner scratch and the counters, for either policy."""
        from . import _capi
        self.capi = _capi
        self.lib = _capi.load_library()
        self.device, self.n = device, n_params
        assert self._num_params() == n_params
        z = lambda k: torch.zeros(k, dtype=torch.float32, device=device)
        self.m, self.v, self.grad, self.stats, self.norm = z(n_params), z(n_params), z(n_params), z(5), z(1)
        self.sms = torch.cuda.get_device_properties(device).multi_processor_count   # grid cap of the learner kernels
        self.scratch = z(self._scratch_floats())
        self.step = 0
        self.counter = 0
        self.launches = 0                # kernels launched through this object (bench.py: gpu_launches)

    def _num_params(self):
        return self.lib.r4_policy_num_params(self.A)

    def _scratch_floats(self):
        return self.sms * (self.n + 5)   # one partial gradient + statistics per CTA

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
        G = G or max(1, min((n + 3) // 4, self.sms))          # 4 samples per CTA tile (r4_ppo.cuh: TS)
        rc = self.lib.r4_policy_grad(mode, _p(flat), *map(_p, data), _p(idx, idx_offset * 8), n, self.A, *_hp(hp), inv_n,
                                     _p(self.scratch), G, _p(self.grad), _p(self.stats), stat_scale, self._stream())
        self._check(rc, "r4_policy_grad")
        self.launches += 2               # k_policy_grad + k_grad_reduce

    def ppo_epoch(self, flat, data, perm, n, mb, hp, lr, clip):
        """All minibatch steps of one SGD epoch in ONE library call (single-GPU learner)."""
        rc = self._epoch("r4_ppo_epoch", (), self.A, flat, data, perm, n, mb, hp, lr, (float(clip or 0.0), _p(self.norm)))
        self.launches += rc * (4 if clip else 2)   # k_policy_grad + k_reduce_adam, or + k_grad_reduce, k_sumsq, k_adam
        return rc

    def ppo_epoch_dist(self, comm, flat, data, perm, n, mb_local, hp, lr):
        """All minibatch steps of one SGD epoch of a data-parallel learner in ONE library call: per step the gradient
        kernel + the fused peer-memory exchange / Adam kernel (csrc/r4_comm.cuh); no NCCL, no host round trip."""
        rc = self._epoch("r4_ppo_epoch_dist", (comm.h,), self.A, flat, data, perm, n, mb_local, hp, lr, ())
        self.launches += rc * 2          # k_policy_grad + k_exchange_adam
        return rc

    def _epoch(self, fn, head, dim, flat, data, perm, n, mb, hp, lr, tail):
        """One call of an epoch entry point (r4_ppo_epoch, r4_gauss_ppo_epoch and their _dist forms): the argument lists differ
        only in the leading communicator, the policy's columns and size, and the trailing gradient clip."""
        rc = getattr(self.lib, fn)(*head, _p(flat), *map(_p, data), _p(perm), n, mb, dim, *_hp(hp), _p(self.scratch),
                                   _p(self.grad), _p(self.stats), _p(self.m), _p(self.v), self.step, lr, 0.9, 0.999, 1e-8,
                                   *tail, self._stream())
        if rc < 0:
            self._check(rc, fn)
        self.step += rc
        return rc

    def policy_grad_exchange(self, comm, mode, flat, data, n, hp, inv_n, stat_scale):
        """One gradient over n local samples, summed over the ranks through peer memory into self.grad (A2C)."""
        G = max(1, min((n + 3) // 4, self.sms))
        rc = self.lib.r4_policy_grad_partial(mode, _p(flat), *map(_p, data), C.c_void_p(0), n, self.A, *_hp(hp), inv_n,
                                             _p(self.scratch), G, self._stream())
        self._check(rc, "r4_policy_grad_partial")
        self._exchange(comm, self.scratch, G, stat_scale)
        self.launches += 2

    def _exchange(self, comm, partial, G, stat_scale):
        """self.grad = the sum over the ranks of this rank's G partial gradients in `partial` (then their statistics)."""
        rc = self.lib.r4_grad_exchange_n(comm.h, _p(partial), G, self.n, _p(self.grad), _p(self.stats), stat_scale,
                                         self._stream())
        self._check(rc, "r4_grad_exchange_n")

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


class GaussKernelOps(KernelOps):
    """ctypes front of the Gaussian-policy kernels (include/rl4rs_b200.h: r4_gauss_*), with KernelOps's methods, so the
    same learner drives either; `data` is (obs, action, logp, dist_inputs, value, adv, target)."""

    def __init__(self, D, device, n_params):
        self.D = D
        self._init(device, n_params)
        # one rank's gradient + statistics, the partial r4_grad_exchange_n sums (A2C)
        self.gsum = torch.zeros(n_params + 5, dtype=torch.float32, device=device)

    def _num_params(self):
        return self.lib.r4_gauss_num_params(self.D)

    def _scratch_floats(self):
        return self.lib.r4_gauss_scratch_size(self.D)

    def act(self, flat, obs, explore, seed, action, env_action, logp, value, dist_inputs):
        n = obs.shape[0]
        rc = self.lib.r4_gauss_act(_p(flat), _p(obs), n, self.D, int(bool(explore)), seed, self.counter, _p(action),
                                   _p(env_action), _p(logp), _p(value), _p(dist_inputs), self._stream())
        self._check(rc, "r4_gauss_act")
        self.counter += n
        self.launches += 1

    def _chunks(self, n):
        return 2 * -(-n // 2048)         # k_gauss_rows + k_gauss_wgrad per chunk of 2048 samples (r4_gauss.cuh: CH)

    def policy_grad(self, mode, flat, data, idx, idx_offset, n, hp, inv_n, stat_scale, grad=None, stats=None):
        grad = self.grad if grad is None else grad
        stats = self.stats if stats is None else stats
        rc = self.lib.r4_gauss_grad(mode, _p(flat), *map(_p, data), _p(idx, idx_offset * 8), n, self.D, *_hp(hp), inv_n,
                                    _p(self.scratch), _p(grad), _p(stats), stat_scale, self._stream())
        self._check(rc, "r4_gauss_grad")
        self.launches += self._chunks(n)

    def ppo_epoch(self, flat, data, perm, n, mb, hp, lr, clip):
        rc = self._epoch("r4_gauss_ppo_epoch", (), self.D, flat, data, perm, n, mb, hp, lr, (float(clip or 0.0), _p(self.norm)))
        self.launches += rc * (self._chunks(mb) + (2 if clip else 1))
        return rc

    def ppo_epoch_dist(self, comm, flat, data, perm, n, mb_local, hp, lr):
        rc = self._epoch("r4_gauss_ppo_epoch_dist", (comm.h,), self.D, flat, data, perm, n, mb_local, hp, lr, ())
        self.launches += rc * (self._chunks(mb_local) + 1)
        return rc

    def policy_grad_exchange(self, comm, mode, flat, data, n, hp, inv_n, stat_scale):
        """One gradient over n local samples, summed over the ranks through peer memory into self.grad (A2C)."""
        self.gsum[self.n:].zero_()
        self.policy_grad(mode, flat, data, None, 0, n, hp, inv_n, 1.0, grad=self.gsum[:self.n], stats=self.gsum[self.n:])
        self._exchange(comm, self.gsum, 1, stat_scale)
        self.launches += 1


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
    """[T, B, ...] device-resident sample batch of one vector episode of the mask policy."""

    def __init__(self, T, B, A, device, obs_dim=256):
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        self.obs, self.mask = z(T, B, obs_dim), z(T, B, A, dt=torch.uint8)
        self.action, self.logp, self.value = z(T, B, dt=torch.int64), z(T, B), z(T, B)
        self.logits, self.reward = z(T, B, A), z(T, B)
        self.T, self.B = T, B

    def observe(self, t, obs, mask):
        """Stores the policy inputs of step t -> the stored copies."""
        self.obs[t].copy_(obs); self.mask[t].copy_(mask)
        return self.obs[t], self.mask[t]

    def _flat(self, *cols):
        n = self.T * self.B
        return tuple(x.reshape((n,) + x.shape[2:]) for x in cols)

    def columns(self):
        """The rollout as flat [n, ...] columns: the policy inputs, action, logp, dist inputs, value -- the order in which the
        losses and the gradient entry points take them before (adv, target)."""
        return self._flat(self.obs, self.mask, self.action, self.logp, self.logits, self.value)

    def a2c_columns(self):
        """columns() with what the A2C gradient does not read left out (r4_policy_grad reads the logits in every mode)."""
        obs, mask, action, _, logits, _ = self.columns()
        return obs, mask, action, None, logits, None

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


class GaussRolloutBuffer(RolloutBuffer):
    """[T, B, ...] device-resident sample batch of the continuous-action env: the unclipped action, the dist inputs
    (mean | log_std, RLlib's stored 'action_dist_inputs'), no mask and no logits."""

    def __init__(self, T, B, D, device, obs_dim=256):
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=device)
        self.obs, self.action, self.dist = z(T, B, obs_dim), z(T, B, D), z(T, B, 2 * D)
        self.logp, self.value, self.reward = z(T, B), z(T, B), z(T, B)
        self.T, self.B = T, B

    def observe(self, t, obs):
        self.obs[t].copy_(obs)
        return (self.obs[t],)

    def columns(self):
        return self._flat(self.obs, self.action, self.logp, self.dist, self.value)

    def a2c_columns(self):
        """No dist inputs: with them r4_gauss_grad would add a KL pass that A2C does not use."""
        obs, action = self.columns()[:2]
        return obs, action, None, None, None


class _TrainerBase(object):
    algo = None
    conti = False          # True: the Gaussian policy of the continuous-action env (PPO_conti / A2C_conti)

    def __init__(self, config, env, device=None, seed=0):
        """config: RLlib-style hyper-parameter dict (unknown keys ignored); env: a RecEnvBase built with output_format='torch'
        and support_rllib_mask=True, or with support_conti_env=True for the Gaussian policy (or any object with that protocol)."""
        self.config = dict(self.DEFAULTS, **{k: v for k, v in (config or {}).items() if k in self.DEFAULTS})
        self.env = env
        self.T = env.config["max_steps"]
        self.B = env.config["batch_size"]
        self.A = env.config["action_size"]
        self.device = torch.device(device) if device is not None else env.sim.engine.device
        # `*_rawstate` algorithms / rawstate_as_obs (modelfree_train.py:218,235-240,270,287-298): the policy embeds the raw
        # state itself ('mask_model_rawstate'); that twin is plain torch + autograd, the kernels serve the 256-d obs policy
        self.rawstate = not self.conti and bool(env.config.get("rawstate_as_obs", False))
        # same init on every rank; _env_action is what the act kernel hands the env: the sampled index, or clip(a, -1, 1)
        if self.conti:
            self.D = env.config.get("action_emb_size", 32)
            self.policy = GaussianPolicy(self.D, self.device, seed=seed)
            self.buf = GaussRolloutBuffer(self.T, self.B, self.D, self.device)
            self._env_action = torch.zeros(self.B, self.D, dtype=torch.float32, device=self.device)
        else:
            if self.rawstate:
                self.policy = RawStatePolicy(self.A, self.device, seed=seed, config=env.config)
            else:
                self.policy = MaskedPolicy(self.A, self.device, seed=seed)
            self.buf = RolloutBuffer(self.T, self.B, self.A, self.device, obs_dim=self.policy.obs_dim if self.rawstate else 256)
            self._env_action = torch.zeros(self.B, dtype=torch.int32, device=self.device)
        self.use_kernels = self.device.type == "cuda" and (config or {}).get("use_kernels", True) and not self.rawstate
        self.opt = torch.optim.Adam([self.policy.flat], lr=self.config["lr"])
        self.ops = None
        if self.use_kernels:
            self.ops = (GaussKernelOps(self.D, self.device, self.policy.n_params) if self.conti
                        else KernelOps(self.A, self.device, self.policy.n_params))
        self.comm = PeerComm(self.policy.n_params, self.device) if self.use_kernels else None
        # shared `seed` for the parameter init and the minibatch permutation; the exploration noise is per rank
        # (k_policy_act hashes seed ^ counter+row: the same seed would give rank r row i the noise of rank 0 row i)
        rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
        self._seed = (seed * 1000003 + rank) & 0x7fffffffffffffff
        if rank and not self.use_kernels:
            torch.manual_seed(seed * 1000003 + rank)
        self.iteration = 0
        self.timesteps_total = 0

    # ---- rollout ------------------------------------------------------------------------------
    @torch.no_grad()
    def rollout(self, explore=True):
        env, buf, flat = self.env, self.buf, self.policy.flat
        obs = env.reset()
        for t in range(self.T):
            inputs = buf.observe(t, *self.policy.inputs(obs))
            if self.use_kernels:       # forward + sampling in ONE kernel, written straight into the rollout buffers
                a = self._env_action
                if self.conti:
                    self.ops.act(flat, *inputs, explore, self._seed, buf.action[t], a, buf.logp[t], buf.value[t], buf.dist[t])
                else:
                    self.ops.act(flat, *inputs, explore, self._seed, a, buf.logp[t], buf.value[t], buf.logits[t])
                    buf.action[t].copy_(a)
            elif self.conti:
                sample, a, logp, value, d = self.policy.act(*inputs, explore=explore)
                buf.action[t].copy_(sample); buf.logp[t].copy_(logp); buf.value[t].copy_(value); buf.dist[t].copy_(d)
            else:
                a, logp, value, logits = self.policy.act(*inputs, explore=explore)
                buf.action[t].copy_(a); buf.logp[t].copy_(logp); buf.value[t].copy_(value); buf.logits[t].copy_(logits)
            obs, reward, done, info = env.step(a)      # clip_actions: the env gets clip(a, -1, 1), the buffer keeps a
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
        """trainer.compute_actions (modelfree_train.py:454): one batch of observations in the env's format (arrays or
        tensors), or RLlib's {env_id: observation} dict -> the actions: i32 [n] of the mask policy, clipped f32 [n, D] of the
        Gaussian policy (a dict keyed like the input for the RLlib form)."""
        import numpy as np
        if isinstance(obs, dict) and not {"obs", "action_mask"} & obs.keys():      # RLlib's {env_id: observation} form
            keys = list(obs.keys())
            rows = [obs[k] for k in keys]
            if isinstance(rows[0], dict):
                a = self.compute_actions({f: np.stack([np.asarray(r[f]) for r in rows]) for f in rows[0]}, explore)
            else:
                a = self.compute_actions(np.stack([np.asarray(r) for r in rows]), explore)
            return dict(zip(keys, a.tolist() if a.ndim == 1 else list(a)))
        if isinstance(obs, dict):
            obs = {k: torch.as_tensor(v, device=self.device) for k, v in obs.items()}
        o, *mask = self.policy.inputs(obs)
        o = torch.as_tensor(o, dtype=torch.float32, device=self.device).contiguous()
        mask = [m.to(torch.uint8).contiguous() for m in mask]
        n = o.shape[0]
        e = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.device)
        if not self.use_kernels:
            a = self.policy.act(o, *mask, explore=explore)[1 if self.conti else 0]
        elif self.conti:
            a = e(n, self.D)
            self.ops.act(self.policy.flat, o, explore, self._seed, e(n, self.D), a, e(n), e(n), None)
        else:
            a = torch.empty(n, dtype=torch.int32, device=self.device)
            self.ops.act(self.policy.flat, o, *mask, explore, self._seed, a, e(n), e(n), None)
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

    def loss(self, *args):
        """RLlib 1.5 ppo_surrogate_loss: loss(*inputs, action, old_logp, old_dist, old_value, adv, target), where inputs are
        the policy's forward() inputs and old_dist its stored dist inputs."""
        *inputs, action, old_logp, old_dist, old_value, adv, target = args
        c = self.config
        d, value = self.policy.forward(*inputs)
        logp, kl, entropy = self.policy.terms(d, action, old_dist)
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
        adv, target = adv.reshape(n), target.reshape(n)
        # StandardizeFields(["advantages"]) over the whole (global) train batch
        mean, sq = adv.mean(), (adv ** 2).mean()
        if _world() > 1:
            ms = torch.stack([mean, sq]); dist.all_reduce(ms); ms /= _world(); mean, sq = ms[0], ms[1]
        adv = (adv - mean) / torch.clamp((sq - mean ** 2).clamp_min(0).sqrt(), min=1e-4)
        # RLlib: sgd_minibatch_size is the TOTAL over devices; every rank contributes sgd_minibatch_size / world samples
        # of its own shard to each SGD step (multi-GPU tower semantics) and the loss is the mean over all of them
        mb = min(max(c["sgd_minibatch_size"] // _world(), 1), n)
        data = buf.columns() + (adv, target)
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

    def loss(self, *args):
        """RLlib 1.5 A3CLoss, summed terms: loss(*inputs, action, adv, target)."""
        *inputs, action, adv, target = args
        c = self.config
        d, value = self.policy.forward(*inputs)
        logp, _, entropy = self.policy.terms(d, action)
        pi_loss = -(logp * adv).sum()
        vf_loss = 0.5 * ((value - target) ** 2).sum()
        entropy = entropy.sum()
        total = pi_loss + c["vf_loss_coeff"] * vf_loss - c["entropy_coeff"] * entropy
        return total, {"policy_loss": pi_loss, "vf_loss": vf_loss, "entropy": entropy}

    def learn(self, buf):
        c = self.config
        target, adv = self._gae(buf)
        n = buf.T * buf.B
        adv, target = adv.reshape(n).contiguous(), target.reshape(n).contiguous()
        w = _world()
        if self.use_kernels:
            ops = self.ops
            data = buf.a2c_columns() + (adv, target)
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
        total, st = self.loss(*buf.columns()[:-3], adv, target)       # the policy inputs and the action
        total.backward()
        self._allreduce_grad(average=False)          # summed loss over the global batch
        gn = torch.nn.utils.clip_grad_norm_([self.policy.flat], c["grad_clip"]) if c["grad_clip"] else torch.zeros(())
        self.opt.step()
        out = {k: self._global_mean(v) * w for k, v in st.items()}
        out.update({"total_loss": self._global_mean(total) * w, "grad_gnorm": float(gn), "sgd_steps": 1})
        return out


class GaussPPOTrainer(PPOTrainer):
    """PPO_conti: PPOTrainer over the DiagGaussian policy of the continuous-action env."""
    algo = "PPO_conti"
    conti = True


class GaussA2CTrainer(A2CTrainer):
    """A2C_conti: A2CTrainer over the DiagGaussian policy of the continuous-action env."""
    algo = "A2C_conti"
    conti = True


# ---- DDPG / TD3 ------------------------------------------------------------------------------------------------------
# RLlib 1.5 ddpg / td3 defaults as modelfree_train.py leaves them (INTEGRATION.md section 3).  train_batch_size None =
# min(B * max_steps, 1024) over the global batch; exploration_config None = the actor output itself (the DDPG quirk,
# INTEGRATION.md section 4), or {"type": "OrnsteinUhlenbeckNoise", ...} over OU_DEFAULTS.
DDPG_DEFAULTS = {"gamma": 1.0, "actor_lr": 1e-3, "critic_lr": 1e-3, "tau": 0.002, "l2_reg": 1e-6, "twin_q": False,
                 "policy_delay": 1, "smooth_target_policy": False, "target_noise": 0.2, "target_noise_clip": 0.5,
                 "prioritized_replay": True, "prioritized_replay_alpha": 0.6, "prioritized_replay_beta": 0.4,
                 "prioritized_replay_eps": 1e-6, "buffer_size": 50000, "learning_starts": 1500,
                 "timesteps_per_iteration": 1000, "train_batch_size": None, "exploration_config": None}
TD3_DEFAULTS = dict(DDPG_DEFAULTS, tau=0.005, l2_reg=0.0, twin_q=True, policy_delay=2, smooth_target_policy=True,
                    prioritized_replay=False, buffer_size=1000000, learning_starts=10000,
                    exploration_config={"type": "OrnsteinUhlenbeckNoise", "random_timesteps": 10000})
OU_DEFAULTS = {"ou_theta": 0.15, "ou_sigma": 0.2, "ou_base_scale": 0.1, "initial_scale": 1.0, "final_scale": 0.02,
               "scale_timesteps": 10000, "random_timesteps": 1000}


class ReplayBuffer(object):
    """RLlib's ReplayBuffer (uniform) / PrioritizedReplayBuffer (proportional) as a device ring: obs f32[C,256], action
    f32[C,D], reward f32[C], new_obs f32[C,256], done u8[C] and, prioritized, prio f32[C] = p^alpha with max_prio f32[1]
    (the running max of |td| + eps).  With `ops` (DDPGKernelOps) the csrc/r4_ddpg.cuh kernels do the work; without, this
    torch code (the CPU path, and the reference of the tests).  The draws are the caller's: u in [0, 1) per sample.
    With n_step (RAINBOW; D is then unused) the actions are i32 [C] and every stored episode gets RLlib's n-step fold
    (_adjust_nstep with `gamma`); `ops` is then RainbowKernelOps."""

    def __init__(self, capacity, D, device, prioritized, alpha=0.6, ops=None, n_step=None, gamma=1.0):
        e = lambda *s, dt=torch.float32: torch.empty(*s, dtype=dt, device=device)   # untouched slots are never read
        self.C, self.D, self.device, self.alpha, self.ops = int(capacity), D, device, alpha, ops
        self.n_step, self.gamma = n_step, gamma
        self.obs, self.reward = e(self.C, 256), e(self.C)
        self.action = e(self.C, D) if n_step is None else e(self.C, dt=torch.int32)
        self.new_obs, self.done = e(self.C, 256), e(self.C, dt=torch.uint8)
        self.prio = e(self.C) if prioritized else None
        self.max_prio = torch.ones(1, dtype=torch.float32, device=device)
        self.added = 0                      # transitions stored since construction

    @property
    def size(self):
        return min(self.added, self.C)

    def store(self, obs, final_obs, action, reward, done):
        """A [T, B] rollout: row t*B + b -> slot (added + t*B + b) % C, new_obs = the next step's obs, or final_obs."""
        T, B = reward.shape
        n = T * B
        if self.ops is not None:
            self.ops.replay_store(self, obs, final_obs, action, reward, done)
        else:
            if self.n_step is None:
                nxt = torch.cat([obs[1:].reshape(-1, 256), final_obs.reshape(B, 256)])
            else:
                nxt, reward, done = self._nstep(obs, final_obs, reward, done)
            first = max(0, n - self.C)
            rows = torch.arange(first, n, device=self.device)
            slots = (self.added + rows) % self.C
            for dst, src in ((self.obs, obs.reshape(n, 256)), (self.new_obs, nxt), (self.action, action.reshape(n, *self.action.shape[1:])),
                             (self.reward, reward.reshape(n)), (self.done, done.reshape(n))):
                dst[slots] = src[rows].to(dst.dtype)
            if self.prio is not None:
                self.prio[slots] = self.max_prio.pow(self.alpha)
        self.added += n

    def _nstep(self, obs, final_obs, reward, done):
        """RLlib _adjust_nstep over every env row of a [T, B] episode -> (new_obs [T*B, 256], reward [T, B], done [T, B]):
        reward_t + sum_{0 < j < n, t + j < T} gamma^j reward_{t+j} (added in j order, float32, as k_replay_store_nstep),
        new_obs and done of step min(t + n - 1, T - 1)."""
        import numpy as np
        T, B = reward.shape
        nxt = torch.cat([obs[1:], final_obs.reshape(1, B, 256)])
        src = torch.clamp(torch.arange(T, device=reward.device) + self.n_step - 1, max=T - 1)
        rew = reward.to(torch.float32)
        R, gj = rew.clone(), np.float32(1.0)
        for j in range(1, min(self.n_step, T)):
            gj = np.float32(gj * np.float32(self.gamma))
            R[:T - j] = R[:T - j] + torch.tensor(gj, device=R.device) * rew[j:]
        return nxt[src].reshape(-1, 256), R, done[src]

    def sample(self, u, beta):
        """-> (idx i64 [n], importance weights f32 [n]) from the uniforms u [n]."""
        N = self.size
        if self.ops is not None:
            return self.ops.replay_sample(self, u, beta)
        if self.prio is None:
            return (u.double() * N).long().clamp(max=N - 1), torch.ones_like(u)
        p = self.prio[:N].double()
        cum = torch.cumsum(p, 0)
        total = cum[-1]
        idx = torch.searchsorted(cum, u.double() * total, right=True).clamp(max=N - 1)
        maxw = (p.min() / total * N) ** -beta
        return idx, ((p[idx] / total * N) ** -beta / maxw).to(torch.float32)

    def update_priorities(self, idx, td, eps):
        """prio[idx] = (|td| + eps)^alpha, the later position winning for a repeated index."""
        if self.ops is not None:
            return self.ops.replay_priorities(self, idx, td, eps)
        import numpy as np
        p = td.abs() + eps
        ix = idx.cpu().numpy()
        _, rev = np.unique(ix[::-1], return_index=True)
        keep = torch.as_tensor(len(ix) - 1 - rev, device=self.device)
        self.prio[idx[keep]] = p[keep].pow(self.alpha)
        self.max_prio.copy_(torch.maximum(self.max_prio, p.max().reshape(1)))

    def gather(self, idx):
        return self.obs[idx], self.action[idx], self.reward[idx], self.new_obs[idx], self.done[idx]


class DDPGKernelOps(object):
    """ctypes front of the DDPG / TD3 kernels (include/rl4rs_b200.h: r4_ddpg_* / r4_replay_*): the moments m, v of both
    Adams (one buffer, split by region), the learner scratch for n samples per step, the loss statistics."""

    def __init__(self, D, twin, device, n_params, n):
        from . import _capi
        self.capi, self.lib = _capi, _capi.load_library()
        self.D, self.twin, self.device, self.n, self.np = D, int(bool(twin)), device, n, n_params
        assert self.lib.r4_ddpg_num_params(D, self.twin) == n_params
        z = lambda k: torch.zeros(k, dtype=torch.float32, device=device)
        self.m, self.v, self.stats = z(n_params), z(n_params), z(3)
        self.grad, self.td = z(n_params), z(n)
        self.scratch = z(self.lib.r4_ddpg_scratch_size(D, self.twin, n))
        self.launches = 0

    _stream = KernelOps._stream
    _check = KernelOps._check

    def act(self, flat, obs, mode, seed, counter, ou_in, ou_out, theta, sigma, ns, action):
        rc = self.lib.r4_ddpg_act(_p(flat), _p(obs), obs.shape[0], self.D, mode, seed, counter, _p(ou_in), _p(ou_out), theta,
                                  sigma, ns, _p(action), self._stream())
        self._check(rc, "r4_ddpg_act")
        self.launches += 1

    def _replay(self, rb):
        return _p(rb.obs), _p(rb.action), _p(rb.reward), _p(rb.new_obs), _p(rb.done)

    def replay_store(self, rb, obs, final_obs, action, reward, done):
        T, B = reward.shape
        rc = self.lib.r4_replay_store(*self._replay(rb), _p(rb.prio), _p(rb.max_prio), rb.C, self.D, rb.added, rb.alpha,
                                      _p(obs), _p(final_obs), _p(action), _p(reward), _p(done), T, B, self._stream())
        self._check(rc, "r4_replay_store")
        self.launches += 1

    def replay_sample(self, rb, u, beta):
        n = u.shape[0]
        idx = torch.empty(n, dtype=torch.int64, device=self.device)
        w = torch.empty(n, dtype=torch.float32, device=self.device)
        rc = self.lib.r4_replay_sample(_p(rb.prio), rb.size, n, beta, _p(u), _p(idx), _p(w), self._stream())
        self._check(rc, "r4_replay_sample")
        self.launches += 1
        return idx, w

    def replay_priorities(self, rb, idx, td, eps):
        rc = self.lib.r4_replay_update_priorities(_p(rb.prio), _p(rb.max_prio), _p(idx), _p(td), idx.shape[0], rb.alpha, eps,
                                                  self._stream())
        self._check(rc, "r4_replay_update_priorities")
        self.launches += 1

    def grad_(self, pol, rb, idx, weights, noise, hp, inv_n):
        """self.grad, self.td, self.stats = r4_ddpg_grad over replay rows idx."""
        rc = self.lib.r4_ddpg_grad(_p(pol.flat), _p(pol.target), self.D, self.twin, *self._replay(rb), _p(idx), _p(weights),
                                   _p(noise), idx.shape[0], hp["gamma"], hp["target_noise"], hp["noise_clip"], inv_n,
                                   _p(self.scratch), _p(self.grad), _p(self.td), _p(self.stats), self._stream())
        self._check(rc, "r4_ddpg_grad")
        self.launches += 2

    def apply(self, pol, actor_step, critic_step, hp, grad_scale=1.0):
        rc = self.lib.r4_ddpg_apply(_p(pol.flat), _p(pol.target), _p(self.grad), _p(self.m), _p(self.v), self.D, self.twin,
                                    actor_step, critic_step, hp["actor_lr"], hp["critic_lr"], hp["l2_reg"], hp["tau"],
                                    grad_scale, self._stream())
        self._check(rc, "r4_ddpg_apply")
        self.launches += 1

    def train_step(self, comm, pol, rb, u, noise, actor_step, critic_step, hp):
        """One whole SGD step in one library call (sample, gradient, exchange over peer memory, Adams + soft update,
        priorities)."""
        rc = self.lib.r4_ddpg_train_step(comm.h if comm is not None else None, _p(pol.flat), _p(pol.target), _p(self.m),
                                         _p(self.v), self.D, self.twin, *self._replay(rb), _p(rb.prio), _p(rb.max_prio),
                                         rb.size, u.shape[0], _p(u), _p(noise), hp["beta"], rb.alpha, hp["eps"], hp["gamma"],
                                         hp["target_noise"], hp["noise_clip"], actor_step, critic_step, hp["actor_lr"],
                                         hp["critic_lr"], hp["l2_reg"], hp["tau"], _p(self.scratch), _p(self.stats),
                                         self._stream())
        self._check(rc, "r4_ddpg_train_step")
        self.launches += 5 if rb.prio is not None else 4
        self.launches += 1 if comm is not None else 0


class DDPGTrainer(_TrainerBase):
    """DDPG (RLlib 1.5 DDPGTrainer as modelfree_train.py configures it) over the deterministic actor-critic of the
    continuous-action env: rollout -> store in the replay -> one SGD step per stored vector episode once `learning_starts`
    transitions were stored (RLlib's 1:1 round robin); an iteration rolls episodes until it sampled
    `timesteps_per_iteration`.  On CUDA: the act kernel, the replay kernels and r4_ddpg_train_step (no host round trip per
    step); on CPU the torch twin.  Data parallel: every rank keeps its own replay and OU state and samples
    train_batch_size / world per step; the gradient is summed over the ranks (peer memory, or NCCL / gloo all-reduce).
    The replay is not checkpointed (RLlib 1.5's default): after restore, learning waits for `learning_starts` again."""
    algo = "DDPG"
    DEFAULTS = DDPG_DEFAULTS
    STATS = ("critic_loss", "actor_loss", "mean_q")     # the names of sgd_step's three statistics in train()'s result

    def __init__(self, config, env, device=None, seed=0):
        cfg = config or {}
        self.config = c = dict(self.DEFAULTS, **{k: v for k, v in cfg.items() if k in self.DEFAULTS})
        self.env = env
        self.T, self.B = env.config["max_steps"], env.config["batch_size"]
        self.D = env.config.get("action_emb_size", 32)
        self.device = torch.device(device) if device is not None else env.sim.engine.device
        world = _world()
        rank = dist.get_rank() if world > 1 else 0
        ex = dict(self.DEFAULTS["exploration_config"] or {}, **(cfg.get("exploration_config") or {}))
        self.ou = dict(OU_DEFAULTS, **{k: v for k, v in ex.items() if k != "type"}) \
            if ex.get("type") == "OrnsteinUhlenbeckNoise" else None
        self.policy = DeterministicActorCritic(self.D, self.device, seed=seed, twin=c["twin_q"])
        tb = c["train_batch_size"] or min(self.B * world * self.T, 1024)
        self.n_local = max(1, tb // world)
        self.use_kernels = self.device.type == "cuda" and cfg.get("use_kernels", True)
        self.ops = DDPGKernelOps(self.D, c["twin_q"], self.device, self.policy.n_params, self.n_local) if self.use_kernels else None
        self.comm = PeerComm(self.policy.n_params, self.device) if self.use_kernels else None
        self.replay = ReplayBuffer(c["buffer_size"], self.D, self.device, c["prioritized_replay"],
                                   c["prioritized_replay_alpha"], self.ops)
        na = self.policy.n_actor
        self._pa = torch.nn.Parameter(self.policy.flat.data[:na])     # the two optimisers update the flat buffer in place
        self._pc = torch.nn.Parameter(self.policy.flat.data[na:])
        self.opt_actor = torch.optim.Adam([self._pa], lr=c["actor_lr"])
        self.opt_critic = torch.optim.Adam([self._pc], lr=c["critic_lr"])
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=self.device)
        self.buf_obs, self.buf_action, self.buf_reward = z(self.T, self.B, 256), z(self.T, self.B, self.D), z(self.T, self.B)
        self.buf_done, self.final_obs = z(self.T, self.B, dt=torch.uint8), z(self.B, 256)
        self.ou_state = z(2, self.D)        # the OU state and its next value: the act kernel reads one, writes the other
        self._ou_slot = 0
        # exploration draws are per rank; the sampling / smoothing draws come from a per-rank generator on the device
        self._seed = (seed * 1000003 + rank) & 0x7fffffffffffffff
        self.gen = torch.Generator(device=self.device).manual_seed(seed * 1000003 + rank + 1)
        self.counter = 0                    # draw counter of the act kernel
        self.policy_ts = 0                  # global exploring timesteps: the OU scale / random-phase schedule
        self.actor_steps = self.critic_steps = 0
        self.iteration = self.timesteps_total = 0

    # ---- acting -------------------------------------------------------------------------------------------------
    def _ou_scale(self):
        o = self.ou
        f = min(max((self.policy_ts - o["random_timesteps"]) / max(o["scale_timesteps"], 1), 0.0), 1.0)
        return o["initial_scale"] + (o["final_scale"] - o["initial_scale"]) * f

    @torch.no_grad()
    def _act(self, obs, explore, out):
        """out [n, D] = the action of obs [n, 256]: the actor output, or OU / random-phase exploration when configured."""
        n, D = obs.shape[0], self.D
        mode = 0
        if explore and self.ou is not None:
            mode = 2 if self.policy_ts <= self.ou["random_timesteps"] else 1
        theta, sigma = (self.ou["ou_theta"], self.ou["ou_sigma"]) if self.ou else (0.0, 0.0)
        ns = self._ou_scale() * self.ou["ou_base_scale"] * 2.0 if mode == 1 else 0.0      # (high - low) = 2
        x_in, x_out = self.ou_state[self._ou_slot], self.ou_state[1 - self._ou_slot]
        if self.use_kernels:
            self.ops.act(self.policy.flat, obs, mode, self._seed, self.counter, x_in, x_out, theta, sigma, ns, out)
        elif mode == 2:
            out.copy_(torch.as_tensor(counter_draws(self._seed, self.counter, n, D)[0], dtype=torch.float32))
        else:
            a = self.policy.actor(obs)
            if mode == 1:
                z = torch.as_tensor(counter_draws(self._seed, self.counter, 1, D)[1][0], dtype=torch.float32, device=obs.device)
                x_out.copy_(x_in + (theta * -x_in + sigma * z))
                a = (a + ns * x_out).clamp(-1.0, 1.0)
            out.copy_(a)
        if mode == 1:
            self._ou_slot ^= 1
        self.counter += n
        if explore:
            self.policy_ts += n * _world()
        return out

    @torch.no_grad()
    def rollout(self, explore=True):
        env = self.env
        obs = env.reset()
        for t in range(self.T):
            self.buf_obs[t].copy_(self.policy.inputs(obs)[0])
            a = self._act(self.buf_obs[t], explore, self.buf_action[t])
            obs, reward, done, info = env.step(a)
            self.buf_reward[t].copy_(reward)
            self.buf_done[t].copy_(torch.as_tensor(done))
        self.final_obs.copy_(self.policy.inputs(obs)[0])
        self.reward = self.buf_reward
        return self

    @torch.no_grad()
    def compute_actions(self, obs, explore=False):
        if isinstance(obs, dict) and "obs" not in obs:                 # RLlib's {env_id: observation} form
            return super().compute_actions(obs, explore)
        o = torch.as_tensor(self.policy.inputs(obs)[0], dtype=torch.float32, device=self.device).contiguous()
        out = torch.empty(o.shape[0], self.D, dtype=torch.float32, device=self.device)
        return self._act(o, explore, out).cpu().numpy()

    # ---- learning -----------------------------------------------------------------------------------------------
    def _hp(self):
        c = self.config
        return {"gamma": c["gamma"], "target_noise": c["target_noise"], "noise_clip": c["target_noise_clip"],
                "actor_lr": c["actor_lr"], "critic_lr": c["critic_lr"], "l2_reg": c["l2_reg"], "tau": c["tau"],
                "beta": c["prioritized_replay_beta"], "eps": c["prioritized_replay_eps"]}

    def draws(self):
        """The caller-side draws of one SGD step: sampling uniforms [n], smoothing normals [n, D] (TD3) or None."""
        u = torch.rand(self.n_local, generator=self.gen, device=self.device)
        noise = (torch.randn(self.n_local, self.D, generator=self.gen, device=self.device)
                 if self.config["smooth_target_policy"] else None)
        return u, noise

    def sgd_step(self, u, noise):
        """One SGD step on this rank's replay with the given draws -> the statistics tensor [3] (critic loss, actor loss,
        mean Q1(s, pi(s)))."""
        c, hp, rb, w = self.config, self._hp(), self.replay, _world()
        update_actor = self.critic_steps % c["policy_delay"] == 0
        self.critic_steps += 1
        self.actor_steps += int(update_actor)
        a_step = self.actor_steps if update_actor else 0
        if self.use_kernels and (w == 1 or self.comm.ok):
            self.ops.train_step(self.comm if w > 1 else None, self.policy, rb, u, noise, a_step, self.critic_steps, hp)
            return self.ops.stats
        idx, wt = rb.sample(u, hp["beta"])
        weights = wt if rb.prio is not None else None
        if self.use_kernels:                # NCCL between the gradient and the optimiser
            self.ops.grad_(self.policy, rb, idx, weights, noise, hp, 1.0 / (self.n_local * w))
            dist.all_reduce(self.ops.grad, op=dist.ReduceOp.SUM)
            self.ops.apply(self.policy, a_step, self.critic_steps, hp)
            td, stats = self.ops.td, self.ops.stats
        else:
            td, stats = self.twin_step(*rb.gather(idx), weights, noise, update_actor)
        if rb.prio is not None:
            rb.update_priorities(idx, td, hp["eps"])
        return stats

    def twin_step(self, obs, action, reward, new_obs, done, weights, noise, update_actor):
        """The torch twin's step over an explicit batch: losses (mean over the global batch), gradient summed over the ranks,
        l2 terms, torch.optim.Adam for the critic(s) and, unless delayed, the actor, then the soft target update."""
        c, pol, w = self.config, self.policy, _world()
        if pol.flat.grad is not None:
            pol.flat.grad.zero_()
        cl, al, td = pol.losses(obs, action, reward, new_obs, done, weights, noise, c["gamma"], c["target_noise"],
                                c["target_noise_clip"], 1.0 / (obs.shape[0] * w))
        (cl + al).backward()
        self._allreduce_grad(average=False)
        g = pol.flat.grad
        if c["l2_reg"]:
            g.add_(c["l2_reg"] * pol.flat.detach() * pol.kernel_mask)
        na = pol.n_actor
        self._pa.grad, self._pc.grad = g[:na], g[na:]
        if update_actor:
            self.opt_actor.step()
        self.opt_critic.step()
        pol.soft_update(c["tau"])
        return td, torch.stack([cl.detach(), al.detach(), -al.detach()])

    def train(self):
        c, w = self.config, _world()
        sampled = steps = 0
        rew, stats = [], torch.zeros(3, dtype=torch.float64, device=self.device)
        while sampled < c["timesteps_per_iteration"]:
            self.rollout(explore=True)
            self.replay.store(self.buf_obs, self.final_obs, self.buf_action, self.buf_reward, self.buf_done)
            sampled += self.T * self.B * w
            rew.append(self.buf_reward.sum(0).mean())
            if self.replay.added * w >= c["learning_starts"]:
                stats += self.sgd_step(*self.draws()).double()
                steps += 1
        self.iteration += 1
        self.timesteps_total += sampled
        g = self._global_means(dict({"_r": torch.stack(rew).mean()}, **{s: stats[i] for i, s in enumerate(self.STATS)}))
        k = max(steps, 1) / w              # each rank's statistics are its share of the global mean
        out = {"episode_reward_mean": g["_r"], "training_iteration": self.iteration, "timesteps_this_iter": sampled,
               "timesteps_total": self.timesteps_total, "episodes_this_iter": len(rew) * self.B * w, "sgd_steps": steps,
               "num_steps_trained": self.critic_steps * self.n_local * w, "replay_size": self.replay.size}
        out.update({s: g[s] / k if steps else float("nan") for s in self.STATS})
        return out

    # ---- checkpoint ---------------------------------------------------------------------------------------------
    def save(self, checkpoint_dir):
        os.makedirs(checkpoint_dir, exist_ok=True)
        path = os.path.join(checkpoint_dir, "checkpoint_%06d.pt" % self.iteration)
        kst = {"m": self.ops.m.cpu(), "v": self.ops.v.cpu()} if self.use_kernels else None
        torch.save({"algo": self.algo, "flat": self.policy.flat.detach().cpu(), "target": self.policy.target.cpu(),
                    "opt_actor": self.opt_actor.state_dict(), "opt_critic": self.opt_critic.state_dict(), "kernel_adam": kst,
                    "ou_state": self.ou_state.cpu(), "ou_slot": self._ou_slot, "counter": self.counter,
                    "policy_ts": self.policy_ts, "actor_steps": self.actor_steps, "critic_steps": self.critic_steps,
                    "gen": self.gen.get_state(), "iteration": self.iteration, "timesteps_total": self.timesteps_total}, path)
        return path

    def restore(self, path):
        st = torch.load(path, map_location="cpu")
        assert st["algo"] == self.algo
        with torch.no_grad():
            self.policy.flat.copy_(st["flat"].to(self.device))
            self.policy.target.copy_(st["target"].to(self.device))
            self.ou_state.copy_(st["ou_state"].to(self.device))
        self.opt_actor.load_state_dict(st["opt_actor"])
        self.opt_critic.load_state_dict(st["opt_critic"])
        if self.use_kernels and st.get("kernel_adam"):
            self.ops.m.copy_(st["kernel_adam"]["m"]); self.ops.v.copy_(st["kernel_adam"]["v"])
        self.gen.set_state(st["gen"])
        for k in ("counter", "policy_ts", "actor_steps", "critic_steps", "iteration", "timesteps_total"):
            setattr(self, k, st[k])
        self._ou_slot = st["ou_slot"]


class TD3Trainer(DDPGTrainer):
    """TD3: DDPGTrainer with RLlib 1.5's TD3 defaults (twin critics with the min target, policy_delay 2, target policy
    smoothing, uniform replay of 10^6, OU exploration after 10 000 random timesteps)."""
    algo = "TD3"
    DEFAULTS = TD3_DEFAULTS


# ---- RAINBOW ---------------------------------------------------------------------------------------------------------
# RLlib 1.5 dqn defaults with modelfree_train.py's RAINBOW overrides (INTEGRATION.md section 3).  train_batch_size None =
# min(B * max_steps, 1024) over the global batch; the target is hard-copied every target_network_update_freq sampled
# timesteps.
RAINBOW_DEFAULTS = {"gamma": 1.0, "lr": 5e-4, "adam_epsilon": 1e-8, "grad_clip": 40.0, "num_atoms": 8, "v_min": 0.0,
                    "v_max": 1000.0, "n_step": 3, "prioritized_replay": True, "prioritized_replay_alpha": 0.6,
                    "prioritized_replay_beta": 0.4, "prioritized_replay_eps": 1e-6, "buffer_size": 100000,
                    "learning_starts": 1000, "target_network_update_freq": 500, "timesteps_per_iteration": 1000,
                    "train_batch_size": None}


class RainbowKernelOps(object):
    """ctypes front of the RAINBOW kernels (include/rl4rs_b200.h: r4_rainbow_* / r4_replay_store_nstep, and the sampling
    and priority kernels of the DDPG replay): the Adam moments m, v, the learner scratch for n samples per step, the loss
    statistics."""

    def __init__(self, A, atoms, device, n_params, n):
        from . import _capi
        self.capi, self.lib = _capi, _capi.load_library()
        self.A, self.atoms, self.device, self.n, self.np = A, atoms, device, n, n_params
        assert self.lib.r4_rainbow_num_params(A, atoms) == n_params
        z = lambda k: torch.zeros(k, dtype=torch.float32, device=device)
        self.m, self.v, self.stats = z(n_params), z(n_params), z(3)
        self.grad, self.td = z(n_params), z(n)
        self.scratch = z(self.lib.r4_rainbow_scratch_size(A, atoms, n))
        self.launches = 0

    _stream = KernelOps._stream
    _check = KernelOps._check
    _replay = DDPGKernelOps._replay
    replay_sample = DDPGKernelOps.replay_sample
    replay_priorities = DDPGKernelOps.replay_priorities

    def act(self, pol, obs, explore, seed, counter, action, q=None):
        rc = self.lib.r4_rainbow_act(_p(pol.flat), _p(obs), obs.shape[0], self.A, self.atoms, pol.v_min, pol.v_max,
                                     int(bool(explore)), seed, counter, _p(action), _p(q), self._stream())
        self._check(rc, "r4_rainbow_act")
        self.launches += 1

    def replay_store(self, rb, obs, final_obs, action, reward, done):
        T, B = reward.shape
        rc = self.lib.r4_replay_store_nstep(*self._replay(rb), _p(rb.prio), _p(rb.max_prio), rb.C, rb.added, rb.alpha,
                                            rb.n_step, rb.gamma, _p(obs), _p(final_obs), _p(action), _p(reward), _p(done),
                                            T, B, self._stream())
        self._check(rc, "r4_replay_store_nstep")
        self.launches += 1

    def grad_(self, pol, rb, idx, weights, gamma_n, inv_n):
        """self.grad, self.td, self.stats = r4_rainbow_grad over replay rows idx."""
        rc = self.lib.r4_rainbow_grad(_p(pol.flat), _p(pol.target), self.A, self.atoms, pol.v_min, pol.v_max,
                                      *self._replay(rb), _p(idx), _p(weights), idx.shape[0], gamma_n, inv_n,
                                      _p(self.scratch), _p(self.grad), _p(self.td), _p(self.stats), self._stream())
        self._check(rc, "r4_rainbow_grad")
        self.launches += 2

    def apply(self, pol, step, hp, copy_target):
        rc = self.lib.r4_rainbow_apply(_p(pol.flat), _p(pol.target), _p(self.grad), _p(self.m), _p(self.v), self.A,
                                       self.atoms, step, hp["lr"], hp["adam_eps"], hp["grad_clip"], int(copy_target),
                                       self._stream())
        self._check(rc, "r4_rainbow_apply")
        self.launches += 1

    def train_step(self, comm, pol, rb, u, step, copy_target, hp):
        """One whole SGD step in one library call (sample, gradient, exchange over peer memory, clip + Adam + target copy,
        priorities)."""
        rc = self.lib.r4_rainbow_train_step(comm.h if comm is not None else None, _p(pol.flat), _p(pol.target), _p(self.m),
                                            _p(self.v), self.A, self.atoms, pol.v_min, pol.v_max, *self._replay(rb),
                                            _p(rb.prio), _p(rb.max_prio), rb.size, u.shape[0], _p(u), hp["beta"], rb.alpha,
                                            hp["eps"], hp["gamma_n"], step, hp["lr"], hp["adam_eps"], hp["grad_clip"],
                                            int(copy_target), _p(self.scratch), _p(self.stats), self._stream())
        self._check(rc, "r4_rainbow_train_step")
        self.launches += 5 if rb.prio is not None else 4
        self.launches += 1 if comm is not None else 0


class RainbowTrainer(DDPGTrainer):
    """RAINBOW (RLlib 1.5 DQNTrainer as modelfree_train.py configures it: distributional, dueling, double Q, n-step 3,
    prioritized replay, noisy off) over the plain observation of the discrete env, acting in Discrete(A) with SoftQ(T = 1)
    exploration and argmax evaluation.  DDPGTrainer's schedule: rollout -> n-step store -> one SGD step per stored vector
    episode once `learning_starts` transitions were stored; an iteration rolls episodes until it sampled
    `timesteps_per_iteration`.  The target net is hard-copied after the SGD step at which target_network_update_freq
    timesteps were sampled since the last copy (RLlib's UpdateTargetNetwork; the first step copies).  On CUDA: the act
    kernel, the replay kernels and r4_rainbow_train_step; on CPU the torch twin.  Data parallel as DDPGTrainer: per-rank
    replay, train_batch_size / world samples per rank, the gradient summed over the ranks before the per-tensor clip.
    The replay is not checkpointed."""
    algo = "RAINBOW"
    DEFAULTS = RAINBOW_DEFAULTS
    STATS = ("loss", "mean_td_error", "mean_q")

    def __init__(self, config, env, device=None, seed=0):
        cfg = config or {}
        self.config = c = dict(self.DEFAULTS, **{k: v for k, v in cfg.items() if k in self.DEFAULTS})
        self.env = env
        self.T, self.B, self.A = env.config["max_steps"], env.config["batch_size"], env.config["action_size"]
        self.device = torch.device(device) if device is not None else env.sim.engine.device
        world = _world()
        rank = dist.get_rank() if world > 1 else 0
        self.policy = DistributionalQNetwork(self.A, self.device, seed=seed, num_atoms=c["num_atoms"], v_min=c["v_min"],
                                             v_max=c["v_max"])
        tb = c["train_batch_size"] or min(self.B * world * self.T, 1024)
        self.n_local = max(1, tb // world)
        self.use_kernels = self.device.type == "cuda" and cfg.get("use_kernels", True)
        self.ops = (RainbowKernelOps(self.A, c["num_atoms"], self.device, self.policy.n_params, self.n_local)
                    if self.use_kernels else None)
        self.comm = PeerComm(self.policy.n_params, self.device) if self.use_kernels else None
        self.replay = ReplayBuffer(c["buffer_size"], None, self.device, c["prioritized_replay"], c["prioritized_replay_alpha"],
                                   self.ops, n_step=c["n_step"], gamma=c["gamma"])
        self.opt = torch.optim.Adam([self.policy.flat], lr=c["lr"], eps=c["adam_epsilon"])
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=self.device)
        self.buf_obs, self.buf_action, self.buf_reward = z(self.T, self.B, 256), z(self.T, self.B, dt=torch.int32), z(self.T, self.B)
        self.buf_done, self.final_obs = z(self.T, self.B, dt=torch.uint8), z(self.B, 256)
        self._seed = (seed * 1000003 + rank) & 0x7fffffffffffffff
        self.gen = torch.Generator(device=self.device).manual_seed(seed * 1000003 + rank + 1)
        self.counter = 0                    # draw counter of the act kernel
        self.policy_ts = 0                  # global exploring timesteps: RLlib's sampled-steps counter
        self.last_target_update = 0         # policy_ts at the last hard target copy
        self.critic_steps = 0               # SGD steps taken (the Adam step count)
        self.iteration = self.timesteps_total = 0

    @torch.no_grad()
    def _act(self, obs, explore, out):
        """out i32 [n] = the action of obs [n, 256]: SoftQ sampling when exploring, else argmax Q."""
        n = obs.shape[0]
        if self.use_kernels:
            self.ops.act(self.policy, obs, explore, self._seed, self.counter, out)
        else:
            out.copy_(self.policy.act(obs, explore, self._seed, self.counter)[0])
        self.counter += n
        if explore:
            self.policy_ts += n * _world()
        return out

    @torch.no_grad()
    def compute_actions(self, obs, explore=False):
        if isinstance(obs, dict) and "obs" not in obs:                 # RLlib's {env_id: observation} form
            return _TrainerBase.compute_actions(self, obs, explore)
        o = torch.as_tensor(self.policy.inputs(obs)[0], dtype=torch.float32, device=self.device).contiguous()
        out = torch.empty(o.shape[0], dtype=torch.int32, device=self.device)
        return self._act(o, explore, out).cpu().numpy()

    def _hp(self):
        c = self.config
        return {"gamma_n": c["gamma"] ** c["n_step"], "lr": c["lr"], "adam_eps": c["adam_epsilon"],
                "grad_clip": float(c["grad_clip"] or 0.0), "beta": c["prioritized_replay_beta"],
                "eps": c["prioritized_replay_eps"]}

    def draws(self):
        """The caller-side draws of one SGD step: the sampling uniforms [n]."""
        return (torch.rand(self.n_local, generator=self.gen, device=self.device),)

    def sgd_step(self, u):
        """One SGD step on this rank's replay with the uniforms u -> the statistics tensor [3] (loss, mean td, mean Q(s, a));
        then the hard target copy when due."""
        c, hp, rb, w = self.config, self._hp(), self.replay, _world()
        self.critic_steps += 1
        copy = self.policy_ts - self.last_target_update >= c["target_network_update_freq"]
        if copy:
            self.last_target_update = self.policy_ts
        if self.use_kernels and (w == 1 or self.comm.ok):
            self.ops.train_step(self.comm if w > 1 else None, self.policy, rb, u, self.critic_steps, copy, hp)
            return self.ops.stats
        idx, wt = rb.sample(u, hp["beta"])
        weights = wt if rb.prio is not None else None
        if self.use_kernels:                # NCCL between the gradient and the optimiser
            self.ops.grad_(self.policy, rb, idx, weights, hp["gamma_n"], 1.0 / (self.n_local * w))
            dist.all_reduce(self.ops.grad, op=dist.ReduceOp.SUM)
            self.ops.apply(self.policy, self.critic_steps, hp, copy)
            td, stats = self.ops.td, self.ops.stats
        else:
            td, stats = self.twin_step(*rb.gather(idx), weights, copy)
        if rb.prio is not None:
            rb.update_priorities(idx, td, hp["eps"])
        return stats

    def twin_step(self, obs, action, reward, new_obs, done, weights, copy_target):
        """The torch twin's step over an explicit batch: the loss (mean over the global batch), gradient summed over the
        ranks, the per-tensor clip, torch.optim.Adam, then the hard target copy when asked -> (td, statistics [3])."""
        c, pol, w = self.config, self.policy, _world()
        if pol.flat.grad is not None:
            pol.flat.grad.zero_()
        inv_n = 1.0 / (obs.shape[0] * w)
        loss, td = pol.loss(obs, action, reward, new_obs, done, weights, self._hp()["gamma_n"], inv_n)
        loss.backward()
        self._allreduce_grad(average=False)
        pol.clip_per_tensor(pol.flat.grad, c["grad_clip"])
        with torch.no_grad():
            q = pol.forward(obs)[1].gather(1, action.long().unsqueeze(1)).sum() * inv_n
        self.opt.step()
        if copy_target:
            with torch.no_grad():
                pol.target.copy_(pol.flat.detach())
        return td, torch.stack([loss.detach(), td.sum() * inv_n, q])

    def save(self, checkpoint_dir):
        os.makedirs(checkpoint_dir, exist_ok=True)
        path = os.path.join(checkpoint_dir, "checkpoint_%06d.pt" % self.iteration)
        kst = {"m": self.ops.m.cpu(), "v": self.ops.v.cpu()} if self.use_kernels else None
        torch.save({"algo": self.algo, "flat": self.policy.flat.detach().cpu(), "target": self.policy.target.cpu(),
                    "opt": self.opt.state_dict(), "kernel_adam": kst, "counter": self.counter, "policy_ts": self.policy_ts,
                    "last_target_update": self.last_target_update, "sgd_steps": self.critic_steps,
                    "gen": self.gen.get_state(), "iteration": self.iteration, "timesteps_total": self.timesteps_total}, path)
        return path

    def restore(self, path):
        st = torch.load(path, map_location="cpu")
        assert st["algo"] == self.algo
        with torch.no_grad():
            self.policy.flat.copy_(st["flat"].to(self.device))
            self.policy.target.copy_(st["target"].to(self.device))
        self.opt.load_state_dict(st["opt"])
        if self.use_kernels and st.get("kernel_adam"):
            self.ops.m.copy_(st["kernel_adam"]["m"]); self.ops.v.copy_(st["kernel_adam"]["v"])
        self.gen.set_state(st["gen"])
        for k in ("counter", "policy_ts", "last_target_update", "iteration", "timesteps_total"):
            setattr(self, k, st[k])
        self.critic_steps = st["sgd_steps"]


def get_rl_model(algo, rllib_config, env=None, **kw):
    """script/modelfree_trainer.py:11-36.  Only the algorithms of the BASELINE configs are built.  On an env built with
    support_conti_env, PPO / A2C (and PPO_conti / A2C_conti, modelfree_train.py:46-48) train the Gaussian policy, and
    DDPG / TD3 (modelfree_trainer.py:25-28) the deterministic actor-critic."""
    conti = env is not None and bool(env.config.get("support_conti_env", False))
    if algo.replace("_rawstate", "") in ("DDPG", "TD3"):
        if algo.endswith("_rawstate") or (env is not None and env.config.get("rawstate_as_obs", False)):
            raise NotImplementedError("%s on a rawstate_as_obs env (model_rawstate) is not built" % algo)
        if not conti:
            raise ValueError("%s needs an env built with support_conti_env=True (modelfree_train.py:46-48)" % algo)
        if env.config.get("support_rllib_mask", False):
            raise ValueError("%s takes the plain observation: build the env with support_rllib_mask=False "
                             "(the reference turns the mask off for DDPG / TD3, modelfree_train.py:46-48)" % algo)
        return (DDPGTrainer if algo == "DDPG" else TD3Trainer)(rllib_config, env, **kw)
    if algo in ("RAINBOW", "RAINBOW_rawstate"):          # exact names: the reference's substring tests are INTEGRATION.md's quirk
        if algo.endswith("_rawstate") or (env is not None and env.config.get("rawstate_as_obs", False)):
            raise NotImplementedError("%s on a rawstate_as_obs env (model_rawstate) is not built" % algo)
        if conti:
            raise ValueError("RAINBOW acts in Discrete(action_size): build the env without support_conti_env")
        if env is not None and env.config.get("support_rllib_mask", False):
            raise ValueError("RAINBOW takes the plain observation: build the env with support_rllib_mask=False "
                             "(the reference turns the mask off for RAINBOW, modelfree_train.py:50-51)")
        return RainbowTrainer(rllib_config, env, **kw)
    if algo.endswith("_conti") or (conti and algo in ("PPO", "A2C")):
        base = algo[:-len("_conti")] if algo.endswith("_conti") else algo
        if base not in ("PPO", "A2C"):
            raise NotImplementedError("%s is outside the hot-path scope (SURVEY.md section 2, row 11)" % algo)
        if not conti:
            raise ValueError("%s needs an env built with support_conti_env=True" % algo)
        if env.config.get("rawstate_as_obs", False):
            raise NotImplementedError("%s on a rawstate_as_obs env (model_rawstate) is not built" % algo)
        if env.config.get("support_rllib_mask", False):
            raise ValueError("%s takes the plain observation: build the env with support_rllib_mask=False "
                             "(the reference turns the mask off for *_conti, modelfree_train.py:46-48)" % algo)
        return (GaussPPOTrainer if base == "PPO" else GaussA2CTrainer)(rllib_config, env, **kw)
    if algo in ("PPO", "PPO_rawstate"):        # '*_rawstate' = the same trainer on an env built with rawstate_as_obs (modelfree_train.py:55-56)
        return PPOTrainer(rllib_config, env, **kw)
    if algo in ("A2C", "A2C_rawstate"):
        return A2CTrainer(rllib_config, env, **kw)
    algo = algo.replace("_rawstate", "")
    assert algo in ("PPO", "DQN", "A2C", "A3C", "PG", "IMPALA", "TD3", "RAINBOW", "SLATEQ", "DDPG")
    raise NotImplementedError("%s is outside the hot-path scope (SURVEY.md section 2, row 11)" % algo)
