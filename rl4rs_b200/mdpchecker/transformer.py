"""keras-transformer 0.40's `get_model`, restated: the encoder-decoder transformer the MDP checker trains
(script/mdpchecker/mdp_checker.py), with the Keras surface the script calls -- compile, summary, fit, predict,
save_weights and load_weights.

On CUDA the forward, backward, loss and Adam run as kernels of csrc/r4_seq2seq.cuh behind the r4_s2s_* C-ABI, and `fit`
chains each epoch's minibatches on the device (r4_s2s_epoch).  On the CPU the same model runs as a torch twin (autograd)
with the same counter-based dropout draws, so a seed gives the same masks on both.  INTEGRATION.md lists what is restated
from keras-transformer, keras-self-attention, keras-layer-normalization, keras-embed-sim, keras-pos-embd and keras 2.2.5.
"""
import math
import time

import numpy as np
import torch

from rl4rs_b200 import _capi
from rl4rs_b200.exactk import keep_scale

MASK = 10000.0
CLIP = np.float32(1e-7)
ADAM = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-7)        # keras 2.2.5 Adam defaults; epsilon = K.epsilon()
SCRATCH_BUDGET = 4 << 30                                     # bytes of scratch one chunk of rows may take


class Config(object):
    def __init__(self, src_tokens, tgt_tokens, embed_dim, head_num, hidden_dim, encoder_num, decoder_num, use_same_embed):
        self.Vs, self.Vt, self.E, self.H, self.F = src_tokens, tgt_tokens, embed_dim, head_num, hidden_dim
        self.Le, self.Ld, self.same = encoder_num, decoder_num, bool(use_same_embed)

    def c(self):
        return _capi.S2SConfig(self.Vs, self.Vt, self.E, self.H, self.F, self.Le, self.Ld, int(self.same))


def weight_names(cfg):
    """[(Keras weight name, shape)] in the flat order of include/rl4rs_b200.h."""
    E, F = cfg.E, cfg.F
    out = []
    if cfg.same:
        out.append(("Token-Embedding/embeddings:0", (cfg.Vs, E)))
    else:
        out += [("Encoder-Token-Embedding/embeddings:0", (cfg.Vs, E)), ("Decoder-Token-Embedding/embeddings:0", (cfg.Vt, E))]

    def att(name):
        return [("%s/%s_%s:0" % (name, name, k), (E, E) if k[0] == "W" else (E,))
                for k in ("Wq", "bq", "Wk", "bk", "Wv", "bv", "Wo", "bo")]

    def norm(name):
        return [("%s-Norm/gamma:0" % name, (E,)), ("%s-Norm/beta:0" % name, (E,))]

    def ff(name):
        return [("%s/%s_W1:0" % (name, name), (E, F)), ("%s/%s_b1:0" % (name, name), (F,)),
                ("%s/%s_W2:0" % (name, name), (F, E)), ("%s/%s_b2:0" % (name, name), (E,))]

    for l in range(cfg.Le):
        a, f = "Encoder-%d-MultiHeadSelfAttention" % (l + 1), "Encoder-%d-FeedForward" % (l + 1)
        out += att(a) + norm(a) + ff(f) + norm(f)
    for l in range(cfg.Ld):
        a, q, f = ("Decoder-%d-MultiHeadSelfAttention" % (l + 1), "Decoder-%d-MultiHeadQueryAttention" % (l + 1),
                   "Decoder-%d-FeedForward" % (l + 1))
        out += att(a) + norm(a) + att(q) + norm(q) + ff(f) + norm(f)
    out.append(("Output/bias:0", (cfg.Vt,)))
    return out


def _truncated_normal(g, shape, std):
    x = torch.randn(shape, generator=g, dtype=torch.float64)
    while True:
        bad = x.abs() > 2.0
        if not bad.any():
            return x * std
        x[bad] = torch.randn(int(bad.sum()), generator=g, dtype=torch.float64)


def init_params(cfg, seed=0):
    """keras 2.2.5 initialisers: embeddings U(-0.05, 0.05), glorot_normal kernels (a normal truncated at two standard
    deviations, stddev sqrt(2 / (fan_in + fan_out)) / 0.8796), zero biases, LayerNorm gamma 1 / beta 0; flat f32."""
    g = torch.Generator().manual_seed(seed)
    parts = []
    for name, sh in weight_names(cfg):
        leaf = name.split("/")[-1]
        if "embeddings" in leaf:
            t = (torch.rand(sh, generator=g, dtype=torch.float64) * 2 - 1) * 0.05
        elif len(sh) == 2:
            t = _truncated_normal(g, sh, math.sqrt(2.0 / (sh[0] + sh[1])) / 0.87962566103423978)
        elif leaf == "gamma:0":
            t = torch.ones(sh, dtype=torch.float64)
        else:
            t = torch.zeros(sh, dtype=torch.float64)
        parts.append(t.reshape(-1))
    return torch.cat(parts).float()


def unflatten(flat, cfg):
    out, o = {}, 0
    for name, sh in weight_names(cfg):
        k = int(np.prod(sh))
        out[name] = flat[o:o + k].view(sh)
        o += k
    return out


# ---- the torch twin -----------------------------------------------------------------------------------------------
def trig(T, E, dtype, device):
    """TrigPosEmbedding's table [T, E]: sin at even columns, cos at odd, angle position / 10000^(2k / E)."""
    p = torch.arange(T, dtype=torch.float32, device=device)[:, None]
    k2 = (torch.arange(E, device=device) // 2 * 2).to(torch.float32)
    ang = p * (1.0 / torch.pow(torch.tensor(10000.0, device=device), k2 / E))
    return torch.where(torch.arange(E, device=device) % 2 == 0, torch.sin(ang), torch.cos(ang)).to(dtype)


def _ln(z, g, b):
    mean = z.mean(-1, keepdim=True)
    var = ((z - mean) ** 2).mean(-1, keepdim=True)
    return (z - mean) / torch.sqrt(var + 1e-14) * g + b


def _mha(w, name, xq, xkv, kmask, causal, H):
    p = lambda k: w["%s/%s_%s:0" % (name, name, k)]
    q, k, v = xq @ p("Wq") + p("bq"), xkv @ p("Wk") + p("bk"), xkv @ p("Wv") + p("bv")
    n, Tq, E = q.shape
    Tk, dh = k.shape[1], E // H
    q, k, v = (t.reshape(n, -1, H, dh).transpose(1, 2) for t in (q, k, v))
    s = q @ k.transpose(-1, -2) / math.sqrt(dh)
    if causal:
        s = s - MASK * torch.triu(torch.ones(Tq, Tk, dtype=s.dtype, device=s.device), 1)
    s = s - MASK * (1.0 - kmask[:, None, None, :].to(s.dtype))
    a = torch.softmax(s, -1)
    o = (a @ v).transpose(1, 2).reshape(n, Tq, E)
    return o @ p("Wo") + p("bo")


def _ffn(w, name, x, keep=None):
    p = lambda k: w["%s/%s_%s:0" % (name, name, k)]
    h = x @ p("W1") + p("b1")
    return (torch.relu(h) if keep is None else h * keep) @ p("W2") + p("b2")


def forward(w, cfg, enc, dec, seed=0, call=0, rate=0.0, relu_keep=None):
    """Logits [n, Tt, Vt] of the twin on enc [n, Ts] and dec [n, Tt] (int64); dropout keyed as the kernels key it.
    relu_keep (optional): per FeedForward, encoder blocks first, the relu decisions to take (a 0 / 1 tensor shaped like
    its hidden layer) instead of deciding them here."""
    E, H = cfg.E, cfg.H
    dt, dev = w["Output/bias:0"].dtype, enc.device
    emb_e = w["Token-Embedding/embeddings:0" if cfg.same else "Encoder-Token-Embedding/embeddings:0"]
    emb_d = w["Token-Embedding/embeddings:0" if cfg.same else "Decoder-Token-Embedding/embeddings:0"]
    layer = [0]

    def wrap(x, y, name):
        k = keep_scale(seed, call * 32 + layer[0], 0, tuple(y.shape), rate, dev, dt)
        layer[0] += 1
        return _ln(x + y * k, w["%s-Norm/gamma:0" % name], w["%s-Norm/beta:0" % name])

    x = emb_e[enc.clamp(0, cfg.Vs - 1)] + trig(enc.shape[1], E, dt, dev)
    em = enc != 0
    for l in range(cfg.Le):
        a, f = "Encoder-%d-MultiHeadSelfAttention" % (l + 1), "Encoder-%d-FeedForward" % (l + 1)
        x = wrap(x, _mha(w, a, x, x, em, False, H), a)
        x = wrap(x, _ffn(w, f, x, relu_keep[l] if relu_keep else None), f)
    e_out = x
    x = emb_d[dec.clamp(0, cfg.Vt - 1)] + trig(dec.shape[1], E, dt, dev)
    dm = dec != 0
    for l in range(cfg.Ld):
        a, q, f = ("Decoder-%d-MultiHeadSelfAttention" % (l + 1), "Decoder-%d-MultiHeadQueryAttention" % (l + 1),
                   "Decoder-%d-FeedForward" % (l + 1))
        x = wrap(x, _mha(w, a, x, x, dm, True, H), a)
        x = wrap(x, _mha(w, q, x, e_out, em, False, H), q)
        x = wrap(x, _ffn(w, f, x, relu_keep[cfg.Le + l] if relu_keep else None), f)
    return x @ emb_d.t() + w["Output/bias:0"]


def loss_fn(logits, dec, target):
    """keras 2.2.5 sparse categorical cross-entropy on the softmax output: the probabilities clipped to [1e-7, 1 - 1e-7],
    their log renormalised by the sparse softmax cross-entropy, masked by dec != 0: sum(mask ce) / sum(mask)."""
    p = torch.softmax(logits, -1)
    q = p.clamp(float(CLIP), float(np.float32(1) - CLIP))
    ce = torch.log(q.sum(-1)) - torch.log(q.gather(-1, target.clamp(0, logits.shape[-1] - 1).unsqueeze(-1)).squeeze(-1))
    m = (dec != 0).to(ce.dtype)
    return (ce * m).sum() / m.sum()


# ---- the Keras surface ---------------------------------------------------------------------------------------------
class History(object):
    def __init__(self):
        self.history = {"loss": []}


class Model(object):
    def __init__(self, cfg, dropout_rate, seed=0, device=None):
        self.cfg, self.dropout_rate, self.seed = cfg, float(dropout_rate), seed
        self.device = torch.device(device if device is not None else ("cuda" if torch.cuda.is_available() else "cpu"))
        self.flat = init_params(cfg, seed).to(self.device)
        self.compiled = False
        self.m = self.v = None
        self.step = 0
        self.call = 0                     # dropout key: one per training step
        if self.device.type == "cuda":
            lib = _capi.load_library()
            assert lib.r4_s2s_num_params(_capi.C.byref(cfg.c())) == self.flat.numel()

    # -- Keras methods --
    def compile(self, optimizer, loss, **kwargs):
        if optimizer != "adam":
            raise NotImplementedError("optimizer %r is not built (the MDP checker compiles with 'adam')" % (optimizer,))
        if loss != "sparse_categorical_crossentropy":
            raise NotImplementedError("loss %r is not built (the MDP checker uses 'sparse_categorical_crossentropy')"
                                      % (loss,))
        if kwargs:
            raise NotImplementedError("compile options %s are not built" % sorted(kwargs))
        self.compiled = True
        self.m, self.v = torch.zeros_like(self.flat), torch.zeros_like(self.flat)

    def count_params(self):
        return int(self.flat.numel())

    def summary(self, print_fn=print):
        layers = []
        for name, sh in weight_names(self.cfg):
            layer = name.split("/")[0]
            if not layers or layers[-1][0] != layer:
                layers.append([layer, 0])
            layers[-1][1] += int(np.prod(sh))
        print_fn("_" * 80)
        print_fn("%-60s%s" % ("Layer (type)", "Param #"))
        print_fn("=" * 80)
        for layer, k in layers:
            print_fn("%-60s%d" % (layer, k))
        print_fn("=" * 80)
        print_fn("Total params: {:,}".format(self.count_params()))
        print_fn("Trainable params: {:,}".format(self.count_params()))
        print_fn("Non-trainable params: 0")
        print_fn("_" * 80)

    def weights(self):
        return {k: t.detach().cpu().numpy().copy() for k, t in unflatten(self.flat, self.cfg).items()}

    def save_weights(self, filepath):
        if str(filepath).endswith((".h5", ".hdf5")):
            raise ValueError("%s: Keras .h5 weight files need h5py, which this package does not use; save to a .npz "
                             "path (arrays keyed by the Keras weight names)" % filepath)
        with open(filepath, "wb") as f:
            np.savez(f, **self.weights())

    def load_weights(self, filepath):
        if str(filepath).endswith((".h5", ".hdf5")):
            raise ValueError("%s: Keras .h5 weight files need h5py, which this package does not use; load a .npz "
                             "written by save_weights" % filepath)
        z = np.load(filepath)
        views = unflatten(self.flat, self.cfg)
        missing = [k for k in views if k not in z.files]
        if missing:
            raise ValueError("%s lacks weights %s" % (filepath, missing[:3]))
        with torch.no_grad():
            for k, t in views.items():
                if tuple(z[k].shape) != tuple(t.shape):
                    raise ValueError("%s: %s has shape %s, the model %s" % (filepath, k, z[k].shape, tuple(t.shape)))
                t.copy_(torch.from_numpy(np.asarray(z[k], dtype=np.float32)))

    # -- helpers --
    def _tok(self, a):
        a = np.asarray(a)
        if a.ndim == 3:
            a = a[..., 0]
        return torch.as_tensor(a.astype(np.int64), device=self.device)

    def _chunk(self, mode, n, Ts, Tt, beam=1, k=0):
        """Rows per call so that one call's scratch stays within SCRATCH_BUDGET (and the grid limits hold)."""
        lib = _capi.load_library()
        c = self.cfg.c()
        m = min(n, max(1, 65535 // (beam * self.cfg.H)))
        while m > 1 and (lib.r4_s2s_scratch_size(_capi.C.byref(c), mode, m, Ts, Tt, beam, k) > SCRATCH_BUDGET):
            m = (m + 1) // 2
        size = lib.r4_s2s_scratch_size(_capi.C.byref(c), mode, m, Ts, Tt, beam, k)
        if size < 0:
            raise ValueError("shape out of the kernels' range: n=%d src_len=%d tgt_len=%d beam=%d k=%d" % (n, Ts, Tt, beam, k))
        return m, torch.empty(size // 4 + 1, dtype=torch.float32, device=self.device)

    def grad(self, enc, dec, target, call=0):
        """(loss, flat gradient) of one minibatch at the current weights, dropout keyed by call."""
        enc, dec, target = self._tok(enc), self._tok(dec), self._tok(target)
        n, Ts = enc.shape
        Tt = dec.shape[1]
        if self.device.type == "cuda":
            lib = _capi.load_library()
            c = self.cfg.c()
            size = lib.r4_s2s_scratch_size(_capi.C.byref(c), _capi.S2S_TRAIN, n, Ts, Tt, 1, 0)
            if size < 0:
                raise ValueError("shape out of the kernels' range: n=%d src_len=%d tgt_len=%d" % (n, Ts, Tt))
            scr = torch.empty(size // 4 + 1, dtype=torch.float32, device=self.device)
            g = torch.empty_like(self.flat)
            loss = torch.empty(1, dtype=torch.float32, device=self.device)
            e32, d32, y32 = (t.to(torch.int32).contiguous() for t in (enc, dec, target))
            _capi.check(lib, None, lib.r4_s2s_grad(_capi.C.byref(c), _capi.ptr(self.flat), _capi.ptr(e32), _capi.ptr(d32),
                                                   _capi.ptr(y32), n, Ts, Tt, self.seed, call, self.dropout_rate,
                                                   _capi.ptr(g), _capi.ptr(loss), _capi.ptr(scr),
                                                   _capi.stream(self.device)), "r4_s2s_grad")
            return float(loss.item()), g
        p = self.flat.detach().clone().requires_grad_(True)
        loss = loss_fn(forward(unflatten(p, self.cfg), self.cfg, enc, dec, self.seed, call, self.dropout_rate), dec, target)
        loss.backward()
        return float(loss.item()), p.grad.detach()

    def apply(self, g):
        """One keras 2.2.5 Adam step with gradient g."""
        self.step += 1
        a = ADAM
        if self.device.type == "cuda":
            lib = _capi.load_library()
            _capi.check(lib, None, lib.r4_s2s_apply(_capi.C.byref(self.cfg.c()), _capi.ptr(self.flat), _capi.ptr(g),
                                                    _capi.ptr(self.m), _capi.ptr(self.v), self.step, a["lr"], a["beta1"],
                                                    a["beta2"], a["eps"], _capi.stream(self.device)), "r4_s2s_apply")
            return
        alpha = a["lr"] * math.sqrt(1 - a["beta2"] ** self.step) / (1 - a["beta1"] ** self.step)
        self.m += (g - self.m) * (1 - a["beta1"])
        self.v += (g * g - self.v) * (1 - a["beta2"])
        self.flat -= alpha * self.m / (self.v.sqrt() + a["eps"])

    def fit(self, x=None, y=None, batch_size=32, epochs=1, verbose=1, shuffle=True, print_fn=print, **kwargs):
        """keras 2.2.5 fit_loop: per epoch one permutation of the rows by np.random.shuffle when shuffle, minibatches of
        batch_size with the last partial one kept, one Adam step each; the epoch's loss is the size-weighted mean."""
        if not self.compiled:
            raise RuntimeError("You must compile a model before training/testing. Use `model.compile(optimizer, loss)`.")
        if kwargs:
            raise NotImplementedError("fit options %s are not built" % sorted(kwargs))
        enc, dec, tgt = self._tok(x[0]), self._tok(x[1]), self._tok(y)
        N, Ts = enc.shape
        Tt = dec.shape[1]
        hist = History()
        steps = (N + batch_size - 1) // batch_size
        sizes = np.minimum(batch_size, N - np.arange(steps) * batch_size).astype(np.float64)
        if self.device.type == "cuda":
            lib = _capi.load_library()
            c = self.cfg.c()
            size = lib.r4_s2s_scratch_size(_capi.C.byref(c), _capi.S2S_TRAIN, batch_size, Ts, Tt, 1, 0)
            if size < 0:
                raise ValueError("shape out of the kernels' range: batch=%d src_len=%d tgt_len=%d" % (batch_size, Ts, Tt))
            scr = torch.empty(size // 4 + 1, dtype=torch.float32, device=self.device)
            g = torch.empty_like(self.flat)
            e32, d32, y32 = (t.to(torch.int32).contiguous() for t in (enc, dec, tgt))
        for ep in range(epochs):
            t0 = time.time()
            idx = np.arange(N)
            if shuffle:
                np.random.shuffle(idx)
            if self.device.type == "cuda":
                perm = torch.as_tensor(idx, dtype=torch.int64, device=self.device)
                losses = torch.empty(steps, dtype=torch.float32, device=self.device)
                a = ADAM
                _capi.check(lib, None, lib.r4_s2s_epoch(
                    _capi.C.byref(c), _capi.ptr(self.flat), _capi.ptr(g), _capi.ptr(self.m), _capi.ptr(self.v),
                    _capi.ptr(e32), _capi.ptr(d32), _capi.ptr(y32), N, Ts, Tt, _capi.ptr(perm), N, batch_size, self.step,
                    self.seed, self.call, self.dropout_rate, a["lr"], a["beta1"], a["beta2"], a["eps"], _capi.ptr(losses),
                    _capi.ptr(scr), _capi.stream(self.device)), "r4_s2s_epoch")
                self.step += steps
                self.call += steps
                ls = losses.double().cpu().numpy()
            else:
                ls = np.empty(steps)
                for k in range(steps):
                    b = torch.as_tensor(idx[k * batch_size:(k + 1) * batch_size], device=self.device)
                    ls[k], gk = self.grad(enc[b], dec[b], tgt[b], call=self.call)
                    self.call += 1
                    self.apply(gk)
            loss = float((ls * sizes).sum() / N)
            hist.history["loss"].append(loss)
            if verbose == 2:
                print_fn("Epoch %d/%d" % (ep + 1, epochs))
                print_fn(" - %ds - loss: %.4f" % (round(time.time() - t0), loss))
            elif verbose:
                print_fn("Epoch %d/%d - loss: %.4f" % (ep + 1, epochs, loss))
        return hist

    def predict_tensor(self, enc, dec):
        """Softmax probabilities [n, Tt, Vt] as a float32 tensor on the model's device."""
        enc, dec = self._tok(enc), self._tok(dec)
        n, Ts = enc.shape
        Tt = dec.shape[1]
        if self.device.type != "cuda":
            with torch.no_grad():
                return torch.softmax(forward(unflatten(self.flat, self.cfg), self.cfg, enc, dec), -1)
        lib = _capi.load_library()
        c = self.cfg.c()
        out = torch.empty(n, Tt, self.cfg.Vt, dtype=torch.float32, device=self.device)
        m, scr = self._chunk(_capi.S2S_PREDICT, n, Ts, Tt)
        e32, d32 = enc.to(torch.int32).contiguous(), dec.to(torch.int32).contiguous()
        for r0 in range(0, n, m):
            k = min(m, n - r0)
            _capi.check(lib, None, lib.r4_s2s_predict(_capi.C.byref(c), _capi.ptr(self.flat), _capi.ptr(e32[r0:r0 + k]),
                                                      _capi.ptr(d32[r0:r0 + k]), k, Ts, Tt, _capi.ptr(out[r0:r0 + k]),
                                                      _capi.ptr(scr), _capi.stream(self.device)), "r4_s2s_predict")
        return out

    def predict(self, x, batch_size=None, verbose=0):
        return self.predict_tensor(x[0], x[1]).cpu().numpy()


def get_model(token_num, embed_dim, encoder_num, decoder_num, head_num, hidden_dim, attention_activation=None,
              feed_forward_activation='relu', dropout_rate=0.0, use_same_embed=True, embed_weights=None,
              embed_trainable=None, trainable=True, use_adapter=False, adapter_units=None, adapter_activation='relu',
              seed=0, device=None):
    """keras-transformer 0.40's get_model.  token_num: one count, or [encoder, decoder] counts when use_same_embed is
    False.  seed and device choose the initialisation draws and where the model runs (CUDA when available)."""
    unbuilt = [("attention_activation", attention_activation, attention_activation is None),
               ("feed_forward_activation", feed_forward_activation, feed_forward_activation == "relu"),
               ("use_adapter", use_adapter, not use_adapter), ("embed_weights", embed_weights, embed_weights is None),
               ("embed_trainable", embed_trainable, embed_trainable in (None, True)),
               ("trainable", trainable, trainable is True)]
    for name, value, ok in unbuilt:
        if not ok:
            raise NotImplementedError("get_model option %s=%r is not built (the MDP checker uses the default)" % (name, value))
    if not isinstance(token_num, (list, tuple)):
        token_num = [token_num, token_num]
    src, tgt = int(token_num[0]), int(token_num[1])
    if use_same_embed:
        tgt = src                     # one table of the encoder's size (keras-transformer sizes the shared table so)
    checks = [(4 <= src <= 65536 and 4 <= tgt <= 65536, "token_num in 4..65536"),
              (embed_dim % 32 == 0 and 32 <= embed_dim <= 512, "embed_dim a multiple of 32 up to 512"),
              (head_num >= 1 and embed_dim % head_num == 0, "head_num dividing embed_dim"),
              (hidden_dim % 32 == 0 and 32 <= hidden_dim <= 1024, "hidden_dim a multiple of 32 up to 1024"),
              (1 <= encoder_num <= 6 and 1 <= decoder_num <= 6, "encoder_num / decoder_num in 1..6"),
              (0.0 <= dropout_rate < 1.0, "dropout_rate in [0, 1)")]
    for ok, what in checks:
        if not ok:
            raise ValueError("get_model: %s is required" % what)
    cfg = Config(src, tgt, embed_dim, head_num, hidden_dim, encoder_num, decoder_num, use_same_embed)
    return Model(cfg, dropout_rate, seed=seed, device=device)
