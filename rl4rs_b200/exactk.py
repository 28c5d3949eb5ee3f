"""Exact-K (nets/exact_k/model.py, script/exact_k_train.py): the transformer-encoder / pointer-network slate generator and
its reward critic, trained on SlateRecEnv-v0 the way the script trains them.

On CUDA every forward, backward and Adam step is a kernel of csrc/r4_exactk.cuh behind the r4_exactk_* C-ABI, and the loop
keeps observations, paths and rewards on the device (the env runs with output_format='torch').  On the CPU the same
networks run as a torch twin (autograd), with the same counter-based draws, so a seed gives the same dropout masks and
the same sampled slates on both.

    python -m rl4rs_b200.exactk train "{'epoch': 1000, 'trial_name': 'a'}"
    python -m rl4rs_b200.exactk eval "{'trial_name': 'a'}"
"""
import ast
import glob
import math
import os
import sys

import numpy as np
import torch

from rl4rs_b200 import _capi

D, HU, UIN, NH, DH, FF, VOCAB, RES, NBLK = 128, 64, 256, 4, 32, 256, 500, 9, 2
SAMPLE, GREEDY, TRAIN = 0, 1, 2
MODES = {"SAMPLE": SAMPLE, "GREEDY": GREEDY, "TRAIN": TRAIN}
GENERATOR, CRITIC = 0, 1
NEG = -2.0 ** 32 + 1
ADAM = dict(beta1=0.9, beta2=0.98, eps=1e-8)
ST_INPUT, ST_ATT0, ST_ATT1, ST_SAMPLE = 0, 1, 2, 3
MAXN, MAX_NTT = 4096, 4096 * 284 * 284    # rows, and rows x candidates^2 (r4_exactk.cuh: MAXN, MAXNTT)

CONFIG = {"epoch": 10000, "maxlen": 64, "batch_size": 256, "action_size": 284, "class_num": 2, "dense_feature_num": 432,
          "category_feature_num": 21, "category_hash_size": 100000, "seq_num": 2, "emb_size": 128, "page_items": 9,
          "hidden_units": 128, "max_steps": 9, "sample_file": '../dataset/rl4rs_dataset_b3_shuf.csv',
          "iteminfo_file": '../item_info.csv', "model_file": "../output/simulator_b2_dien/model", "support_rllib_mask": False,
          "is_eval": False, 'env': "SlateRecEnv-v0"}


def generator_shapes():
    """The flat generator layout of include/rl4rs_b200.h, in order: [(name, shape)]."""
    s = [("u_w", (UIN, HU)), ("u_b", (HU,)), ("emb", (VOCAB, HU))]
    for l in range(NBLK):
        s += [("b%d_%s" % (l, k), sh) for k, sh in (("qkv_w", (D, 3 * D)), ("qkv_b", (3 * D,)), ("ln1_b", (D,)),
                                                   ("ln1_g", (D,)), ("f1_w", (D, FF)), ("f1_b", (FF,)), ("f2_w", (FF, D)),
                                                   ("f2_b", (D,)), ("ln2_b", (D,)), ("ln2_g", (D,)))]
    s += [("lstm_w", (2 * D, 4 * D)), ("lstm_b", (4 * D,)), ("c0", (D,)), ("x0", (D,)), ("h0", (D,)),
          ("w_b", (D, D)), ("v_dec", (D,)), ("w_bef", (D, D)), ("bias_dec", (D,))]
    for a in ("g", "p"):
        s += [(a + "_" + k, sh) for k, sh in (("w_q", (D, D)), ("w_dec", (D, D)), ("v", (D,)), ("bias", (D,)),
                                             ("w_ref", (D, D)))]
    return s


def critic_shapes():
    return [("w1", (UIN, 128)), ("b1", (128,)), ("w2", (128, 128)), ("b2", (128,)), ("w3", (128, 128)), ("b3", (128,)),
            ("w4", (128, 1)), ("b4", (1,))]


def unflatten(flat, shapes):
    out, o = {}, 0
    for name, sh in shapes:
        k = int(np.prod(sh))
        out[name] = flat[o:o + k].view(sh)
        o += k
    return out


def _glorot(g, shape, fan_in, fan_out):
    lim = math.sqrt(6.0 / (fan_in + fan_out))
    return (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) * lim


def init_generator(seed=0):
    """TF1 initialisers of the graph: glorot-uniform kernels (dense, conv1d k=1, LSTMCell, the xavier W_* and v), zero
    biases and initial states, LayerNorm gamma 1 / beta 0, the item embedding uniform(+-0.08)."""
    g = torch.Generator().manual_seed(seed)
    parts = []
    for name, sh in generator_shapes():
        base = name.split("_", 1)[1] if name[:2] in ("b0", "b1", "g_", "p_") else name
        if base in ("emb",):
            t = (torch.rand(sh, generator=g, dtype=torch.float64) * 2 - 1) * 0.08
        elif base in ("ln1_g", "ln2_g"):
            t = torch.ones(sh, dtype=torch.float64)
        elif len(sh) == 2:
            t = _glorot(g, sh, sh[0], sh[1])
        elif base in ("v", "v_dec"):
            t = _glorot(g, sh, sh[0], sh[0])
        else:
            t = torch.zeros(sh, dtype=torch.float64)
        parts.append(t.reshape(-1))
    return torch.cat(parts).float()


def init_critic(seed=0):
    g = torch.Generator().manual_seed(seed)
    parts = [(_glorot(g, sh, sh[0], sh[1]) if len(sh) == 2 else torch.zeros(sh, dtype=torch.float64)).reshape(-1)
             for _, sh in critic_shapes()]
    return torch.cat(parts).float()


# ---- draws: the hash of csrc/r4_exactk.cuh (draw24) over int64 tensors with wrapping arithmetic --------------------------
_M64 = (1 << 64) - 1


def _s64(c):
    return c - (1 << 64) if c >= 1 << 63 else c


def _shr(x, k):
    return (x >> k) & ((1 << (64 - k)) - 1)


def _mix64(x):
    x = x + _s64(0x9E3779B97F4A7C15)
    x = (x ^ _shr(x, 30)) * _s64(0xBF58476D1CE4E5B9)
    x = (x ^ _shr(x, 27)) * _s64(0x94D049BB133111EB)
    return x ^ _shr(x, 31)


def _mix64_int(x):
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def draw24(seed, call, stream, elem):
    """(seed, call, stream, elem int64 tensor) -> the top 24 bits of the device hash, int64 tensor."""
    k = _mix64_int((call * 8 + stream) & _M64)
    return _shr(_mix64(torch.bitwise_xor(_mix64(elem + _s64(k)), _s64(seed & _M64))), 40)


def keep_scale(seed, call, stream, shape, rate, device, dtype):
    """The inverted-dropout factor of every element of a row-major tensor of shape: 0 or 1 / (1 - rate)."""
    if rate <= 0:
        return torch.ones(shape, device=device, dtype=dtype)
    n = int(np.prod(shape))
    out = torch.empty(n, device=device, dtype=dtype)
    step = 1 << 24
    for o in range(0, n, step):
        e = torch.arange(o, min(n, o + step), device=device, dtype=torch.int64)
        u = draw24(seed, call, stream, e).to(torch.float32) * (1.0 / 16777216.0)
        out[o:o + len(e)] = (u >= rate).to(dtype) * (1.0 / (1.0 - np.float32(rate)))
    return out.view(shape)


def point_masks(masks, path, t):
    """The point mask of step t [n, T] (bool) from masks [4, T] and the earlier choices path[:, :t]."""
    n, T = path.shape[0], masks.shape[1]
    m = masks[t // 3].bool().unsqueeze(0).expand(n, T).clone()
    if t == 0:
        return m
    sel = torch.zeros(n, T, dtype=torch.bool, device=path.device)
    sel.scatter_(1, path[:, :t].long(), True)
    special = masks[3].bool()
    any_sp = (sel & special).any(1, keepdim=True)
    return m & ~sel & ~(any_sp & special)


def twin_forward(w, user, masks, mode, seed, call, rate, temperature=1.0, target=None):
    """The generator's forward as torch ops over the dict of parameter views w (any dtype / device; autograd-capable):
    -> (logits [n, 9, T], path [n, 9] int64).  mode TRAIN follows target."""
    n, T = user.shape[0], masks.shape[1]
    dt, dev = w["u_w"].dtype, w["u_w"].device
    uenc = torch.relu(user @ w["u_w"] + w["u_b"])
    x = torch.cat([uenc.unsqueeze(1).expand(n, T, HU), w["emb"][:T].unsqueeze(0).expand(n, T, HU) * 8.0], 2)
    x = x * keep_scale(seed, call, ST_INPUT, (n, T, D), rate, dev, dt)
    for l in range(NBLK):
        p = "b%d_" % l
        m = (x.sum(-1) != 0).to(dt)                                             # [n, T] key / query mask
        qkv = torch.relu(x @ w[p + "qkv_w"] + w[p + "qkv_b"]).view(n, T, 3, NH, DH)
        q, k, v = (qkv[:, :, i].transpose(1, 2) for i in range(3))              # [n, 4, T, 32]
        s = q @ k.transpose(-1, -2) / math.sqrt(DH)
        s = torch.where(m[:, None, None, :] != 0, s, torch.full_like(s, NEG))
        a = torch.softmax(s, -1) * m[:, None, :, None]
        a = a * keep_scale(seed, call, ST_ATT0 + l, (n, NH, T, T), rate, dev, dt)
        o = (a @ v).transpose(1, 2).reshape(n, T, D)
        y1 = _ln(o + x, w[p + "ln1_b"], w[p + "ln1_g"])
        f = torch.relu(y1 @ w[p + "f1_w"] + w[p + "f1_b"]) @ w[p + "f2_w"] + w[p + "f2_b"]
        x = _ln(f + y1, w[p + "ln2_b"], w[p + "ln2_g"])
    enc = x
    eref = [enc @ w["g_w_ref"], enc @ w["p_w_ref"]]
    c = w["c0"].expand(n, D)
    h = w["h0"].expand(n, D)
    inp = w["x0"].expand(n, D)
    outs, hbs, logits, path = [], [], [], torch.zeros(n, RES, dtype=torch.int64, device=dev)
    rows = torch.arange(n, device=dev)
    for t in range(RES):
        gates = torch.cat([inp, h], 1) @ w["lstm_w"] + w["lstm_b"]
        gi, gj, gf, go = gates.split(D, 1)
        c = torch.sigmoid(gf + 1.0) * c + torch.sigmoid(gi) * torch.tanh(gj)
        h = torch.sigmoid(go) * torch.tanh(c)
        if t == 0:
            intra = torch.zeros(n, D, dtype=dt, device=dev)
        elif t == 1:
            intra = outs[0]
        else:
            bef = torch.stack(outs, 1)                                          # [n, t, D]
            sc = (w["v_dec"] * torch.tanh(torch.stack(hbs, 1) + (h @ w["w_b"]).unsqueeze(1) + w["bias_dec"])).sum(-1)
            intra = (torch.softmax(sc, 1).unsqueeze(2) * bef).sum(1)
        outs.append(h)
        hbs.append(h @ w["w_bef"])
        a1 = h @ w["g_w_q"] + intra @ w["g_w_dec"] + w["g_bias"]
        p1 = torch.softmax((w["g_v"] * torch.tanh(eref[0] + a1.unsqueeze(1))).sum(-1), 1)
        gl = (p1.unsqueeze(2) * enc).sum(1)
        a2 = gl @ w["p_w_q"] + intra @ w["p_w_dec"] + w["p_bias"]
        lg = (w["p_v"] * torch.tanh(eref[1] + a2.unsqueeze(1))).sum(-1)
        lg = torch.where(point_masks(masks, path, t), lg, torch.full_like(lg, NEG))
        logits.append(lg)
        if mode == TRAIN:
            pick = target[:, t].long()
        elif mode == GREEDY:
            pick = lg.detach().argmax(1)
        else:
            pick = sample_index(lg.detach(), seed, call, t, temperature)
        path[:, t] = pick
        inp = enc[rows, pick]
    return torch.stack(logits, 1), path


def _ln(z, beta, gamma):
    mean = z.mean(-1, keepdim=True)
    var = ((z - mean) ** 2).mean(-1, keepdim=True)
    return gamma * (z - mean) / (var + 1e-8) ** 0.5 + beta


def sample_index(lg, seed, call, t, temperature):
    """The SAMPLE choice of step t: inverse CDF of softmax(lg / temperature) on the row's draw (b, t); float32 running sum
    in candidate order as the kernel sums."""
    n, T = lg.shape
    x = (lg.float() / np.float32(temperature))
    e = torch.exp(x - x.max(1, keepdim=True).values)
    bits = draw24(seed, call, ST_SAMPLE, torch.arange(n, device=lg.device, dtype=torch.int64) * RES + t)
    run = torch.cumsum(e, 1)
    u = (bits.float() + 0.5) * (1.0 / 16777216.0) * run[:, -1]
    hit = (run >= u.unsqueeze(1)) & (e > 0)
    last = T - 1 - torch.flip(e > 0, [1]).int().argmax(1)
    return torch.where(hit.any(1), hit.int().argmax(1), last)


def policy_loss(logits, target, reward):
    """mean_b(sum_t CE(logits[b, t], target[b, t]) reward[b])."""
    ce = torch.nn.functional.cross_entropy(logits.reshape(-1, logits.shape[-1]), target.reshape(-1).long(),
                                           reduction="none").view(target.shape)
    return (ce.sum(1) * reward).mean()


def critic_forward(w, user):
    x = torch.relu(user @ w["w1"] + w["b1"])
    x = torch.relu(x @ w["w2"] + w["b2"])
    x = torch.relu(x @ w["w3"] + w["b3"])
    return (x @ w["w4"] + w["b4"])[:, 0]


class _Adam(object):
    """TF1 AdamOptimizer over one flat parameter vector: the kernel (r4_exactk_adam) on CUDA, the same update on the CPU."""

    def __init__(self, net, flat, lr):
        self.net, self.flat, self.lr = net, flat, lr
        self.m, self.v = torch.zeros_like(flat), torch.zeros_like(flat)
        self.step = 0

    def apply(self, grad):
        self.step += 1
        b1, b2, eps = ADAM["beta1"], ADAM["beta2"], ADAM["eps"]
        if self.flat.is_cuda:
            lib = _capi.load_library()
            _capi.check(lib, None, lib.r4_exactk_adam(self.net, _capi.ptr(self.flat), _capi.ptr(grad), _capi.ptr(self.m),
                                                      _capi.ptr(self.v), self.step, self.lr, b1, b2, eps,
                                                      _capi.stream(self.flat.device)), "r4_exactk_adam")
            return
        alpha = self.lr * math.sqrt(1 - b2 ** self.step) / (1 - b1 ** self.step)
        self.m += (grad - self.m) * (1 - b1)
        self.v += (grad * grad - self.v) * (1 - b2)
        self.flat -= alpha * self.m / (self.v.sqrt() + eps)


def check_shape(n, T):
    """Raise ValueError unless the generator runs n rows over T candidates: n in 1..4096 and n T^2 <= 4096 * 284^2 (the
    generator's scratch holds five [n, 4, T, T] planes: 47.4 GB at that bound)."""
    if not 1 <= n <= MAXN or n * T * T > MAX_NTT:
        raise ValueError("Exact-K runs 1..%d rows with rows x seq_length^2 <= %d (4096 rows at 284 candidates, %d at %d); "
                         "got %d rows at seq_length %d" % (MAXN, MAX_NTT, min(MAXN, MAX_NTT // (T * T)), T, n, T))


def _not_built(**opts):
    for name, (value, ok) in opts.items():
        if not ok:
            raise NotImplementedError("Exact-K option %s=%r is not built (the script uses the default)" % (name, value))


class Generator(object):
    """model.py's Generator: the constructor arguments of the reference.  draw(user, mode) -> (path, logits);
    grad(user, target, reward) -> (grad, loss); train(user, target, reward) takes one Adam step."""

    def __init__(self, l1_mask, l2_mask, l3_mask, l0_ssr_mask, is_training=True, lr=0.001, temperature=1,
                 train_sample='random', predict_sample='random', seq_length=500, res_length=9, hidden_units=64,
                 dropout_rate=0.1, num_heads=4, num_layers=1, num_glimpse=1, num_blocks=2, use_mha=True, beam_size=3,
                 device="cuda", seed=0):
        _not_built(use_mha=(use_mha, bool(use_mha)), num_layers=(num_layers, num_layers == 1),
                   num_glimpse=(num_glimpse, num_glimpse == 1), hidden_units=(hidden_units, hidden_units == HU),
                   num_heads=(num_heads, num_heads == NH), num_blocks=(num_blocks, num_blocks == NBLK),
                   res_length=(res_length, res_length == RES))
        if not 9 <= seq_length <= VOCAB:
            raise ValueError("seq_length must be in 9..500 (the item embedding has 500 rows), got %d" % seq_length)
        self.device = torch.device(device)
        self.T, self.lr, self.temperature = int(seq_length), lr, float(temperature)
        self.rate = float(dropout_rate) if is_training else 0.0
        self.masks = torch.tensor(np.stack([np.asarray(m, dtype=np.float64)[:seq_length] for m in
                                            (l1_mask, l2_mask, l3_mask, l0_ssr_mask)]) != 0, dtype=torch.uint8,
                                  device=self.device)
        self.flat = init_generator(seed).to(self.device)
        self.opt = _Adam(GENERATOR, self.flat, lr)
        self.seed, self.call = int(seed), 0
        self._scratch = {}

    def params(self, flat=None):
        return unflatten(self.flat if flat is None else flat, generator_shapes())

    def _next_call(self):
        self.call += 1
        return self.call

    def _scr(self, n):
        if n not in self._scratch:
            lib = _capi.load_library()
            self._scratch = {n: torch.empty(lib.r4_exactk_scratch_size(GENERATOR, n, self.T), dtype=torch.uint8,
                                            device=self.device)}
        return self._scratch[n]

    def draw(self, user, mode=SAMPLE):
        """One decode (SAMPLE or GREEDY) of the rows of user [n, 256] -> (path [n, 9] int64, logits [n, 9, T])."""
        mode = MODES.get(mode, mode)
        if mode in ("BEAMSEARCH", "CUSTOM"):
            raise NotImplementedError("Exact-K decode mode %s is not built (the script samples and decodes greedily)" % mode)
        if mode not in (SAMPLE, GREEDY):
            raise ValueError("draw mode must be SAMPLE or GREEDY, got %r" % (mode,))
        check_shape(user.shape[0], self.T)
        call = self._next_call()
        user = user.to(self.device, torch.float32).contiguous()
        n = user.shape[0]
        if self.device.type != "cuda":
            with torch.no_grad():
                lg, path = twin_forward(self.params(), user, self.masks, mode, self.seed, call, self.rate, self.temperature)
            return path, lg
        lib = _capi.load_library()
        path = torch.empty(n, RES, dtype=torch.int32, device=self.device)
        lg = torch.empty(n, RES, self.T, dtype=torch.float32, device=self.device)
        _capi.check(lib, None, lib.r4_exactk_decode(_capi.ptr(self.flat), _capi.ptr(user), n, self.T, _capi.ptr(self.masks),
                                                    mode, self.temperature, self.seed, call, self.rate, _capi.ptr(path),
                                                    _capi.ptr(lg), _capi.ptr(self._scr(n)), _capi.stream(self.device)),
                    "r4_exactk_decode")
        return path.long(), lg

    def grad(self, user, target, reward):
        """The gradient of the policy loss on the teacher path target [n, 9] -> (grad [num_params], loss [1])."""
        check_shape(user.shape[0], self.T)
        call = self._next_call()
        user = user.to(self.device, torch.float32).contiguous()
        reward = reward.to(self.device, torch.float32).contiguous()
        n = user.shape[0]
        if self.device.type != "cuda":
            flat = self.flat.detach().clone().requires_grad_(True)
            lg, _ = twin_forward(self.params(flat), user, self.masks, TRAIN, self.seed, call, self.rate, target=target)
            loss = policy_loss(lg, target, reward)
            loss.backward()
            return flat.grad, loss.detach().view(1)
        lib = _capi.load_library()
        tgt = target.to(self.device, torch.int32).contiguous()
        grad = torch.empty_like(self.flat)
        loss = torch.empty(1, dtype=torch.float32, device=self.device)
        _capi.check(lib, None, lib.r4_exactk_grad(_capi.ptr(self.flat), _capi.ptr(user), n, self.T, _capi.ptr(self.masks),
                                                  _capi.ptr(tgt), _capi.ptr(reward), self.seed, call, self.rate,
                                                  _capi.ptr(grad), _capi.ptr(loss), _capi.ptr(self._scr(n)),
                                                  _capi.stream(self.device)), "r4_exactk_grad")
        return grad, loss

    def train(self, user, target, reward):
        grad, loss = self.grad(user, target, reward)
        self.opt.apply(grad)
        return loss


class Discriminator(object):
    """model.py's Discriminator: an MLP 256 -> 128 -> 128 -> 128 -> 1 on the user features, trained on the summed squared
    error to the rollout reward."""

    def __init__(self, lr=0.005, seq_length=500, device="cuda", seed=1):
        self.device = torch.device(device)
        self.lr = lr
        self.flat = init_critic(seed).to(self.device)
        self.opt = _Adam(CRITIC, self.flat, lr)
        self._scratch = {}

    def _run(self, user, target):
        user = user.to(self.device, torch.float32).contiguous()
        n = user.shape[0]
        if self.device.type != "cuda":
            flat = self.flat.detach().clone().requires_grad_(target is not None)
            pred = critic_forward(unflatten(flat, critic_shapes()), user)
            if target is None:
                return pred.detach(), None, None
            loss = ((target.to(pred.dtype) - pred) ** 2).sum()
            loss.backward()
            return pred.detach(), flat.grad, loss.detach().view(1)
        lib = _capi.load_library()
        if n not in self._scratch:
            self._scratch = {n: torch.empty(lib.r4_exactk_scratch_size(CRITIC, n, 0), dtype=torch.uint8, device=self.device)}
        pred = torch.empty(n, dtype=torch.float32, device=self.device)
        grad = torch.empty_like(self.flat) if target is not None else None
        loss = torch.empty(1, dtype=torch.float32, device=self.device) if target is not None else None
        tgt = target.to(self.device, torch.float32).contiguous() if target is not None else None
        _capi.check(lib, None, lib.r4_exactk_critic(_capi.ptr(self.flat), _capi.ptr(user), n, _capi.ptr(tgt), _capi.ptr(pred),
                                                    _capi.ptr(grad), _capi.ptr(loss), _capi.ptr(self._scratch[n]),
                                                    _capi.stream(self.device)), "r4_exactk_critic")
        return pred, grad, loss

    def predict(self, user):
        return self._run(user, None)[0]

    def train(self, user, target):
        _, grad, loss = self._run(user, target)
        self.opt.apply(grad)
        return loss


# ---- the script's two stages -----------------------------------------------------------------------------------------------
def model_dir(config, output_dir=None):
    """'<rl4rs_output_dir>/exactk_<env>_<trial_name>/', the script's directory naming."""
    output_dir = output_dir or os.environ.get("rl4rs_output_dir", ".")
    return '%s/%s/' % (output_dir, 'exactk_' + config.get('env', CONFIG['env']) + '_' + str(config.get('trial_name', '')))


def save(path, gen, critic, episode):
    torch.save({"episode": episode, "generator": gen.flat.cpu(), "critic": critic.flat.cpu(),
                "gen_adam": (gen.opt.m.cpu(), gen.opt.v.cpu(), gen.opt.step),
                "critic_adam": (critic.opt.m.cpu(), critic.opt.v.cpu(), critic.opt.step), "call": gen.call}, path)
    return path


def newest_checkpoint(directory):
    """The newest exact_k.ckpt.<episode> under directory (the script's find_newest_files), or None."""
    files = glob.glob(os.path.join(directory, 'exact_k.ckpt.*'))
    return max(files, key=lambda f: (os.path.getmtime(f), int(f.rsplit('.', 1)[1]))) if files else None


def restore(path, gen, critic):
    st = torch.load(path, map_location="cpu")
    gen.flat.copy_(st["generator"])
    critic.flat.copy_(st["critic"])
    for opt, (m, v, step) in ((gen.opt, st["gen_adam"]), (critic.opt, st["critic_adam"])):
        opt.m.copy_(m); opt.v.copy_(v); opt.step = step
    gen.call = st["call"]
    return st["episode"]


def _check_env(config):
    if config.get('env', 'SlateRecEnv-v0') == 'SeqSlateRecEnv-v0':
        raise ValueError("Exact-K decodes one 9-item slate per episode; SeqSlateRecEnv-v0 takes 36 steps per episode, "
                         "and the reference script fails stepping 36 columns of a 9-column path: use SlateRecEnv-v0")


def make_env(config):
    from rl4rs_b200 import gymshim
    from rl4rs_b200.env.slate import SlateRecEnv, SlateState
    sim = SlateRecEnv(dict(config, output_format='torch'), state_cls=SlateState)
    return gymshim.make('SlateRecEnv-v0', recsim=sim)


def build_nets(config, device, seed=0):
    from rl4rs_b200.env.slate import SlateState
    A = config["action_size"]
    check_shape(config.get("batch_size", CONFIG["batch_size"]), A)
    if "catalog" in config:
        location_mask = SlateState._location_mask(A)
        special_items = [int(x) for x in config["catalog"].special_items]
    else:
        location_mask, special_items = SlateState.get_mask_from_file(config['iteminfo_file'], A)
    l0_ssr_mask = np.zeros(A)
    l0_ssr_mask[special_items] = 1
    g = Generator(location_mask[0], location_mask[1], location_mask[2], l0_ssr_mask, is_training=True, seq_length=A,
                  device=device, seed=seed)
    d = Discriminator(seq_length=A, device=device, seed=seed + 1)
    return g, d


def _as_tensor(x):
    return x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x))


def train(config, env=None, device=None, output_dir=None, seed=0, log=print):
    """exact_k_train.py's train stage: per episode two sampled rollouts (three env resets), best-of-2 per row, one critic
    step, one generator step on the normalised advantage; checkpoints every 500 episodes and at the end.
    -> (generator, critic, per-episode stats list)."""
    config = dict(CONFIG, **config)
    _check_env(config)
    env = env if env is not None else make_env(config)
    device = torch.device(device or ("cuda" if torch.cuda.is_available() else "cpu"))
    gen, critic = build_nets(config, device, seed)
    directory = model_dir(config, output_dir)
    os.makedirs(directory, exist_ok=True)
    path = directory + 'exact_k.ckpt'
    stats = []
    episode = -1
    for episode in range(config["epoch"]):
        obs = _as_tensor(env.reset()).to(device, torch.float32)
        rollouts = []
        for _ in range(2):
            sampled, _ = gen.draw(obs, SAMPLE)
            for step in range(config['max_steps']):
                _, reward, _, _ = env.step(sampled[:, step] if device.type == "cuda" else sampled[:, step].numpy())
            env.reset()
            rollouts.append((sampled, _as_tensor(reward).to(device, torch.float32)))
        (p0, r0), (p1, r1) = rollouts
        second = r1 > r0                                           # stable sort, descending: ties keep the first rollout
        target = torch.where(second.unsqueeze(1), p1, p0)
        reward = torch.where(second, r1, r0)
        reward_ = critic.predict(obs)
        closs = critic.train(obs, reward)
        adv = reward - reward_
        std = adv.double().std(unbiased=False)                     # np.std
        if float(std) == 0.0:
            raise FloatingPointError("Exact-K episode %d: the advantage reward - critic(obs) has zero std; normalising it "
                                     "would write NaN into the generator" % episode)
        gloss = gen.train(obs, target, (adv / std.to(adv.dtype)))
        stats.append({"episode": episode, "reward": float(reward.mean()), "critic_loss": float(closs[0]),
                      "policy_loss": float(gloss[0])})
        if episode % 50 == 0 and log:
            log('episode: %d reward %.4f reward_target %.4f' % (episode, float(reward.mean()), float(reward_.mean())))
        if episode % 500 == 0:
            save(path + '.' + str(episode), gen, critic, episode)
    save(path + '.' + str(episode), gen, critic, episode)
    return gen, critic, stats


def evaluate(config, env=None, device=None, output_dir=None, batches=4, log=print):
    """exact_k_train.py's eval stage: restore the newest checkpoint, run `batches` greedy batches (dropout live, as the
    script's is_training=True graph) and return the running average reward per row."""
    config = dict(CONFIG, **config)
    _check_env(config)
    env = env if env is not None else make_env(config)
    device = torch.device(device or ("cuda" if torch.cuda.is_available() else "cpu"))
    gen, critic = build_nets(config, device)
    ckpt = newest_checkpoint(model_dir(config, output_dir))
    if ckpt is None:
        raise FileNotFoundError("no exact_k.ckpt.* under %s" % model_dir(config, output_dir))
    restore(ckpt, gen, critic)
    total, avg = 0.0, 0.0
    for i in range(batches):
        obs = _as_tensor(env.reset()).to(device, torch.float32)
        path, _ = gen.draw(obs, GREEDY)
        for step in range(config['max_steps']):
            _, reward, _, _ = env.step(path[:, step] if device.type == "cuda" else path[:, step].numpy())
            total += float(_as_tensor(reward).double().sum())
        avg = total / config['batch_size'] / (i + 1)
        if log:
            log('avg reward', avg)
    return avg


def main(argv=None):
    argv = sys.argv[1:] if argv is None else argv
    stage, extra = argv[0], ast.literal_eval(argv[1]) if len(argv) > 1 else {}
    config = dict(CONFIG, **extra)
    if stage == 'train':
        train(config)
    elif stage == 'eval':
        return evaluate(config)
    else:
        raise ValueError("stage must be 'train' or 'eval', got %r" % stage)


if __name__ == "__main__":
    main()
