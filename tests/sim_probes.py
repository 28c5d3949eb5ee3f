"""Probe weights that route one stage of a simulator's forward to its observation, and float64 references of each stage.

The simulators' observation is a dense head over a long feature vector (dien: ELU(allf . obs_w + obs_b), 3456 inputs per
output), so an error inside a recurrence reaches the observation diluted by the head.  A probe replaces the head by a
pass-through of one 128-column block x of the feature vector:

    obs_w[off + j, j] = +1,  obs_w[off + j, 128 + j] = -1,  obs_b = 0   =>   obs[:, j] = ELU(x_j),  obs[:, 128 + j] = ELU(-x_j)

and `decode` recovers x_j from whichever of the two is positive (ELU is the identity there, and a product with an exact
1.0 adds no rounding in any split of the operand).  A probe changes only the tensors it lists; the reference of a stage is
the oracle's own stage computation in float64 on the probe weights, so a probe makes a stage visible without changing what
the reference computes.

Probes (name -> tensors changed):
  dien   augru{i}{a,b}  obs_w/obs_b: +-I on column half a (0..127) / b (128..255) of AUGRU i's output
         gru1_last{i}   AUGRU i reduced to tanh(last GRU-1 state): u gate off (weights 0, bias -20), candidate = x on
                        columns 0..127 (x-rows I, h-rows 0, bias 0); head as augru{i}a
         scores{i}      AUGRU i reduced to h_t = (1 - a_t) h_(t-1) + a_t c_t with the DIN scores a_t as its only
                        gate: u gate on (weights 0, bias +20), candidate c_t = tanh(k_j H_t,j) (x-rows diag(k) on columns
                        0..127, k log-spaced 1 .. 100 so some columns stay off the tanh plateau in every regime; h-rows
                        0, bias 0); head as augru{i}a.  h_63 = sum_t a_t prod_(s>t) (1 - a_s) c_t is linear in the last
                        ~20 scores (a_t ~ 0.55), each weighted by c_t - h_(t-1).  Bounded scores only.
         dense, catattn +-I on the dense tower / the pooled category self-attention
         flatten{s}     +-I on category slot s of the head's gathered half (slots 0, 10, 20)
  lstm   sgru0, sgru1, dense, cgru   +-I on each block of the head's materialised half
  dnn    catpool, dense   fc_w = +-I on the category mean-pool / the dense tower, fc_b = 0, obs_w = I, obs_b = 0
  widedeep  pool0, pool1  fc_w = +-I on one sequence's mean-pool, fc_b = 0

Every probe also names a perturbation of the stage it exposes (`perturb`: a small change to a weight the stage reads);
tests/test_sim_probes_cpu.py requires the decoded block to move past the probe's bar under it, so a probe that exposes
nothing cannot pass for coverage.
"""
import re

import numpy as np

from oracle.dien_np import DienOracle
from oracle.dnn_np import DnnOracle
from oracle.lstm_np import LstmOracle, keras_gru_last
from oracle.widedeep_np import WideDeepOracle

E = 128
NCAT = 21
FLATTEN_SLOTS = (0, 10, 20)

# --- regimes ------------------------------------------------------------------------------------------------------------
DIEN_REGIMES = ("default", "bounded", "synthetic")
LSTM_REGIMES = ("default", "clipping")
BOUNDED = ("bounded", "synthetic")              # the regimes whose DIN scores stay in (0, 1)


def sim_cfg(algo="dien", hash_size=100000, B=8, **flags):
    cfg = {"maxlen": 64, "batch_size": B, "action_size": 284, "class_num": 2, "dense_feature_num": 432,
           "category_feature_num": NCAT, "category_hash_size": hash_size, "seq_num": 2, "emb_size": E,
           "hidden_units": 128, "max_steps": 9, "page_items": 9, "action_emb_size": 32, "is_eval": True,
           "cache_size": B, "algo": algo}
    cfg.update(flags)
    return cfg


def regime_weights(algo, regime, **flags):
    """(cfg, W-table) of one weight regime:
    dien      default   = bench.py's glorot weights (hash 100 000, raw unbounded DIN scores)
              bounded   = bias_noise 0.1, bounded scores (hash 100 000)
              synthetic = stress 2, bias_noise 0.1, bounded scores (hash 5 000; test_gpu_parity._synthetic)
    lstm      default   = Keras initialisers; clipping = gru_stress 2.5, gru_bias_noise 1.5 (~25 % of the gates clip)
    dnn, widedeep: default = stress 1, bias_noise 0.1."""
    from rl4rs_b200 import synth
    hs = 5000 if regime == "synthetic" else 100000
    cfg = sim_cfg(algo, hs, **flags)
    if algo == "dien":
        kw = {"default": {}, "bounded": {"bias_noise": 0.1, "bounded_scores": True},
              "synthetic": {"stress": 2.0, "bias_noise": 0.1, "bounded_scores": True}}[regime]
        return cfg, synth.make_weights(cfg, **kw)
    if algo == "lstm":
        kw = {"default": {}, "clipping": {"gru_stress": 2.5, "gru_bias_noise": 1.5}}[regime]
        return cfg, synth.make_lstm_weights(cfg, **kw)
    assert regime == "default", regime
    if algo == "dnn":
        return cfg, synth.make_dnn_weights(cfg, stress=1.0, bias_noise=0.1)
    return cfg, synth.make_widedeep_weights(cfg, stress=1.0, bias_noise=0.1)


# --- feature rows -------------------------------------------------------------------------------------------------------
EDGE_LENGTHS = (0, 1, 2, 63, 64)


def feature_rows(R, seed, hash_size):
    """R feature rows (seq i32 [R,2,64], dense f32 [R,432], cat i32 [R,21]) with the edges in the first rows:
    sequence lengths 0, 1, 2, 63, 64 (both sequences) in rows 0..4, ids 0 and hash - 1 in sequences and categories,
    dense rows with log-uniform magnitudes 1e-6 .. 1e4, random signs and exact zeros (rows 5..9) and one row with every
    dense input at 1e4 (row 10)."""
    rs = np.random.RandomState(seed)
    seq = np.zeros((R, 2, 64), np.int32)
    n = rs.randint(0, 65, (R, 2))
    k = min(R, len(EDGE_LENGTHS))
    n[:k] = np.asarray(EDGE_LENGTHS[:k])[:, None]
    ids = rs.randint(1, 284, (R, 2, 64))
    edge = rs.rand(R, 2, 64) < 0.05
    ids[edge] = hash_size - 1
    keep = np.arange(64)[None, None, :] >= (64 - n)[:, :, None]
    seq[keep] = ids[keep]
    dense = rs.normal(0, 2, (R, 432)).astype(np.float32)
    wide = range(5, min(R, 10))
    for r in wide:
        mag = 10.0 ** rs.uniform(-6, 4, 432)
        d = mag * rs.choice([-1.0, 1.0], 432)
        d[rs.rand(432) < 0.1] = 0.0
        dense[r] = d.astype(np.float32)
    if R > 10:
        dense[10] = 1e4
    cat = rs.randint(0, hash_size, (R, NCAT)).astype(np.int32)
    cat[rs.rand(R, NCAT) < 0.05] = 0
    cat[rs.rand(R, NCAT) < 0.05] = hash_size - 1
    return seq, dense, cat


def sample_rows(R, cta=64, extra=()):
    """Every row up to 129; above that the first, a middle and the last row of every `cta`-row CTA (+ `extra`)."""
    if R <= 129:
        return np.arange(R)
    s = np.arange(0, R, cta)
    idx = np.concatenate([s, np.minimum(s + cta // 2, R - 1), np.minimum(s + cta - 1, R - 1), np.asarray(extra, np.int64)])
    return np.unique(idx[(idx >= 0) & (idx < R)])


# --- the head pass-through and its recovery ---------------------------------------------------------------------------
def pm_identity(K, off, n_out=256):
    """[K, n_out] head: +I on rows off..off+127 -> outputs 0..127, -I -> outputs 128..255."""
    w = np.zeros((K, n_out), np.float32)
    j = np.arange(E)
    w[off + j, j] = 1.0
    w[off + j, E + j] = -1.0
    return w


def decode(obs):
    """obs [R, >=256] of a +-I head -> the 128-column block it passes through."""
    obs = np.asarray(obs)
    p, m = obs[:, :E], obs[:, E:2 * E]
    return np.where(p > 0, p, -m)


# --- probes -------------------------------------------------------------------------------------------------------------
class Probe(object):
    """name, simulator, the tensors it changes, build(w) -> probe W-table, stage(oracle, seq, dense, cat) -> the block
    the observation carries, `kind`: 'recur' (bar against max(|ref|, rms(row))), 'gemm' (bar against the magnitude
    pass `mag(oracle, ...)`) or 'exact' (bit-exact)."""

    def __init__(self, sim, name, changed, build, stage, kind, perturb, mag=None, bounded_only=False):
        self.sim, self.name, self.changed, self.build_fn = sim, name, tuple(changed), build
        self.stage, self.kind, self.mag, self.bounded_only = stage, kind, mag, bounded_only
        self.perturb_fn = perturb

    def perturb(self, w):
        """The base W-table with the probe's perturbation applied (to tensors the probe does not replace)."""
        out = dict(w)
        ch = self.perturb_fn(w)
        assert not set(ch) & set(self.changed), (self.name, sorted(ch))
        out.update(ch)
        return out

    def build(self, w):
        out = dict(w)
        out.update(self.build_fn(w))
        assert set(self.build_fn(w)) == set(self.changed), (self.name, sorted(self.build_fn(w)))
        return out

    def __repr__(self):
        return "%s/%s" % (self.sim, self.name)


def _abs_dense_mag(o, dense):
    """Magnitude pass of the dense tower: the same two layers over |x|, |W|, |b| (ELU is 1-Lipschitz)."""
    w = o.w
    m = np.abs(np.asarray(dense, np.float64)) @ np.abs(w["dense_w1"].astype(np.float64)) + np.abs(w["dense_b1"].astype(np.float64))
    return m @ np.abs(w["dense_w2"].astype(np.float64)) + np.abs(w["dense_b2"].astype(np.float64))


def _dense_stage(o, dense):
    w = o.w
    el = lambda x: np.where(x > 0, x, np.expm1(np.minimum(x, 0)))
    x = el(np.asarray(dense).astype(o.dt) @ w["dense_w1"] + w["dense_b1"])
    return el(x @ w["dense_w2"] + w["dense_b2"]).astype(o.dt)


# dien ---------------------------------------------------------------------------------------------------------------------
DIEN_K = 2 * 256 + 128 + 128 + NCAT * E          # 3456
DIEN_OFF = {"augru0a": 0, "augru0b": 128, "augru1a": 256, "augru1b": 384, "dense": 512, "catattn": 640}


def dien_augru_stage(o, i, seq, cat):
    """AUGRU i's output h_63 [R, 256] (GRU-1 -> DIN scores -> AUGRU) through the oracle's own stage methods."""
    seq = np.asarray(seq).astype(np.int64)
    es = o.w["emb_seq"]
    q = es[np.asarray(cat).astype(np.int64)[:, -10:]].mean(axis=1).astype(o.dt)
    H = o.gru(i, es[seq[:, i, :]])
    return o.augru(i, H, o.att_scores(i, q, H))


def dien_augru_stage_torch(w, i, seq, cat, device="cpu"):
    """`dien_augru_stage` of DienOracle(w, float64), ported to torch float64 so that it runs on the device at the env
    path's row counts.  Held to the NumPy oracle within 1e-12 by tests/test_sim_probes_cpu.py."""
    import torch
    T = lambda a: torch.as_tensor(np.asarray(a, np.float64), device=device)
    seq = np.asarray(seq).astype(np.int64)
    es = w["emb_seq"]
    q = T(es[np.asarray(cat).astype(np.int64)[:, -10:]]).mean(dim=1)
    x = T(es[seq[:, i, :]])
    B, L, _ = x.shape
    sig = lambda z: 1.0 / (1.0 + torch.exp(-z))

    def cell(xt, h, wg, bg, wc, bc, a=None):
        U = wc.shape[1]
        g = sig(torch.cat([xt, h], 1) @ wg + bg)
        r, u = g[:, :U], g[:, U:]
        c = torch.tanh(torch.cat([xt, r * h], 1) @ wc + bc)
        if a is not None:
            u = (1.0 - a[:, None]) * u
        return u * h + (1 - u) * c

    g = [T(w["gru%d_%s" % (i, k)]) for k in ("wg", "bg", "wc", "bc")]
    h = torch.zeros((B, E), dtype=torch.float64, device=device)
    H = []
    for t in range(L):
        h = cell(x[:, t], h, *g)
        H.append(h)
    H = torch.stack(H, 1)
    qq = q[:, None, :].expand_as(H)
    a = torch.cat([qq, H, qq - H, qq * H], -1)
    a = sig(a @ T(w["att%d_w1" % i]) + T(w["att%d_b1" % i]))
    a = sig(a @ T(w["att%d_w2" % i]) + T(w["att%d_b2" % i]))
    s = (a @ T(w["att%d_k" % i]) + T(w["att%d_b" % i]))[..., 0]
    ag = [T(w["augru%d_%s" % (i, k)]) for k in ("wg", "bg", "wc", "bc")]
    h = torch.zeros((B, ag[2].shape[1]), dtype=torch.float64, device=device)
    for t in range(L):
        h = cell(H[:, t], h, *ag, a=s[:, t])
    return h.cpu().numpy()


def _head(off):
    return lambda w: {"obs_w": pm_identity(DIEN_K, off), "obs_b": np.zeros(256, np.float32)}


def _gru1_last(i):
    def build(w):
        wg, bg = w["augru%d_wg" % i].copy(), w["augru%d_bg" % i].copy()
        wg[:, 256:] = 0.0
        bg[256:] = -20.0
        wc = np.zeros_like(w["augru%d_wc" % i])
        wc[np.arange(E), np.arange(E)] = 1.0                   # x-rows: I on columns 0..127; h-rows 0
        out = {"augru%d_wg" % i: wg, "augru%d_bg" % i: bg, "augru%d_wc" % i: wc,
               "augru%d_bc" % i: np.zeros_like(w["augru%d_bc" % i])}
        out.update(_head(256 * i)(w))
        return out
    return build


SCORES_GAIN = np.geomspace(1.0, 8.0, E).astype(np.float32)


def _scores(i):
    def build(w):
        wg, bg = w["augru%d_wg" % i].copy(), w["augru%d_bg" % i].copy()
        wg[:, 256:] = 0.0
        bg[256:] = 20.0
        wc = np.zeros_like(w["augru%d_wc" % i])
        wc[np.arange(E), np.arange(E)] = SCORES_GAIN           # x-rows: diag(k) on columns 0..127; h-rows 0
        out = {"augru%d_wg" % i: wg, "augru%d_bg" % i: bg, "augru%d_wc" % i: wc,
               "augru%d_bc" % i: np.zeros_like(w["augru%d_bc" % i])}
        out.update(_head(256 * i)(w))
        return out
    return build


def _catattn_mag(o, seq, dense, cat):
    """Magnitude pass of the pooled self-attention: mean over slots of P |E| (P = the float64 attention weights)."""
    emb = o.w["emb_cat"][np.asarray(cat).astype(np.int64)].astype(np.float64)
    s = np.matmul(emb, emb.transpose(0, 2, 1))
    p = np.exp(s - s.max(axis=-1, keepdims=True))
    p /= p.sum(axis=-1, keepdims=True)
    return np.matmul(p, np.abs(emb)).mean(axis=1)


HEAD = ("obs_w", "obs_b")
CHUNK = 64                                        # the recurrences' and GEMMs' column chunk


def _scale(name, eps, cols=None):
    """Perturbation: tensor `name` times (1 + eps), on columns `cols` only when given."""
    def f(w):
        t = np.array(w[name], np.float64)
        if cols is None:
            t *= 1.0 + eps
        else:
            t[..., cols] *= 1.0 + eps
        return {name: t.astype(np.float32)}
    return f


def _ulp_up(name):
    return lambda w: {name: np.nextafter(np.asarray(w[name], np.float32), np.float32(np.inf))}


def dien_probes():
    P = []
    for i in range(2):
        for half in "ab":
            c0 = 128 * (half == "b")
            P.append(Probe("dien", "augru%d%s" % (i, half), HEAD, _head(DIEN_OFF["augru%d%s" % (i, half)]),
                           (lambda i, h: lambda o, s, d, c: dien_augru_stage(o, i, s, c)[:, h * E:(h + 1) * E])(i, half == "b"),
                           "recur", _scale("augru%d_wc" % i, 1e-3, slice(c0, c0 + CHUNK))))
    for i in range(2):
        names = ("augru%d_wg" % i, "augru%d_bg" % i, "augru%d_wc" % i, "augru%d_bc" % i) + HEAD
        P.append(Probe("dien", "gru1_last%d" % i, names, _gru1_last(i),
                       (lambda i: lambda o, s, d, c: dien_augru_stage(o, i, s, c)[:, :E])(i), "recur",
                       _scale("gru%d_wc" % i, 1e-3, slice(0, CHUNK))))
        P.append(Probe("dien", "scores%d" % i, names, _scores(i),
                       (lambda i: lambda o, s, d, c: dien_augru_stage(o, i, s, c)[:, :E])(i), "recur",
                       _scale("att%d_k" % i, 1e-2), bounded_only=True))
    P.append(Probe("dien", "dense", HEAD, _head(DIEN_OFF["dense"]), lambda o, s, d, c: o.dense_feature(d), "gemm",
                   _scale("dense_w2", 1e-4, slice(0, CHUNK)), mag=lambda o, s, d, c: _abs_dense_mag(o, d)))
    P.append(Probe("dien", "catattn", HEAD, _head(DIEN_OFF["catattn"]),
                   lambda o, s, d, c: o.category_feature(np.asarray(c).astype(np.int64))[:, :E], "gemm",
                   _scale("emb_cat", 1e-5), mag=_catattn_mag))
    for slot in FLATTEN_SLOTS:
        P.append(Probe("dien", "flatten%d" % slot, HEAD, _head(768 + E * slot),
                       (lambda slot: lambda o, s, d, c: o.w["emb_cat"][np.asarray(c).astype(np.int64)[:, slot]])(slot), "exact",
                       _ulp_up("emb_cat")))
    return P


# lstm ---------------------------------------------------------------------------------------------------------------------
LSTM_K = 4 * E + NCAT * E
LSTM_OFF = {"sgru0": 0, "sgru1": 128, "dense": 256, "cgru": 384}


def lstm_stage(o, name, seq, dense, cat):
    w, dt = o.w, o.dt
    if name == "dense":
        return _dense_stage(o, dense)
    if name == "cgru":
        return keras_gru_last(w["emb_cat"][np.asarray(cat).astype(np.int64)], w["cgru_k"], w["cgru_rk"], w["cgru_b"], dt)
    i = int(name[-1])
    x = w["emb_seq"][np.asarray(seq).astype(np.int64)[:, i, :]]
    return keras_gru_last(x, w["sgru%d_k" % i], w["sgru%d_rk" % i], w["sgru%d_b" % i], dt)


def lstm_probes():
    P = []
    for name, off in LSTM_OFF.items():
        build = (lambda off: lambda w: {"obs_w": pm_identity(LSTM_K, off), "obs_b": np.zeros(256, np.float32)})(off)
        stage = (lambda name: lambda o, s, d, c: lstm_stage(o, name, s, d, c))(name)
        if name == "dense":
            P.append(Probe("lstm", name, HEAD, build, stage, "gemm", _scale("dense_w2", 1e-4, slice(0, CHUNK)),
                           mag=lambda o, s, d, c: _abs_dense_mag(o, d)))
        else:
            kx = name + "_k"
            P.append(Probe("lstm", name, HEAD, build, stage, "recur", _scale(kx, 1e-2, slice(0, CHUNK))))
    return P


# dnn / widedeep ---------------------------------------------------------------------------------------------------------
def _pool_mag(table):
    return lambda o, ids: np.abs(o.w[table][ids].astype(np.float64)).mean(axis=1)


def dnn_probes():
    def build(off):
        return lambda w: {"fc_w": pm_identity(2 * E, off), "fc_b": np.zeros(256, np.float32),
                          "obs_w": np.eye(256, dtype=np.float32), "obs_b": np.zeros(256, np.float32)}
    changed = ("fc_w", "fc_b", "obs_w", "obs_b")
    pool = lambda o, s, d, c: o.w["emb_cat"][np.asarray(c).astype(np.int64)].mean(axis=1).astype(o.dt)
    return [Probe("dnn", "catpool", changed, build(0), pool, "gemm", _scale("emb_cat", 1e-5),
                  mag=lambda o, s, d, c: _pool_mag("emb_cat")(o, np.asarray(c).astype(np.int64))),
            Probe("dnn", "dense", changed, build(E), lambda o, s, d, c: _dense_stage(o, d), "gemm",
                  _scale("dense_w2", 1e-4, slice(0, CHUNK)), mag=lambda o, s, d, c: _abs_dense_mag(o, d))]


def widedeep_probes():
    P = []
    for i in range(2):
        build = (lambda i: lambda w: {"fc_w": pm_identity(2 * E, E * i), "fc_b": np.zeros(256, np.float32)})(i)
        pool = (lambda i: lambda o, s, d, c: o.w["emb_seq"][np.asarray(s).astype(np.int64)[:, i, :]].mean(axis=1).astype(o.dt))(i)
        mag = (lambda i: lambda o, s, d, c: _pool_mag("emb_seq")(o, np.asarray(s).astype(np.int64)[:, i, :]))(i)
        P.append(Probe("widedeep", "pool%d" % i, ("fc_w", "fc_b"), build, pool, "gemm", _scale("emb_seq", 1e-5), mag=mag))
    return P


ORACLES = {"dien": DienOracle, "lstm": LstmOracle, "dnn": DnnOracle, "widedeep": WideDeepOracle}


def all_probes():
    return dien_probes() + lstm_probes() + dnn_probes() + widedeep_probes()


def regimes_of(probe):
    if probe.sim == "dien":
        return BOUNDED if probe.bounded_only else DIEN_REGIMES
    if probe.sim == "lstm":
        return LSTM_REGIMES
    return ("default",)


def oracle(probe_or_sim, w, dtype):
    sim = getattr(probe_or_sim, "sim", probe_or_sim)
    return ORACLES[sim](w, dtype)


# --- bars ---------------------------------------------------------------------------------------------------------------
# Per stage family (and regime where it matters), about 3x the worst error measured on an H100 80GB HBM3 and never above
# the 1e-4 the observations are held to (one exception, below) (DESIGN.md section 2): relative to max(|ref|, rms(row)) for the recurrences,
# relative to the float64 magnitude pass for the GEMM-only stages.  Flatten is bit-exact.
TOL = {
    "augru": 7e-5, ("augru", "synthetic"): 1e-4,            # worst 2.3e-5 default, 1.6e-5 bounded, 6.7e-5 synthetic
    "gru1_last": 7e-5, ("gru1_last", "synthetic"): 1e-4,    # 2.2e-5 default, 0.8e-5 bounded, 3.5e-5 synthetic
    # the scores probe's candidate tanh(k H_t) (k up to 8) also carries GRU-1's error (3.5e-5 of rms at stress 2) into
    # its block, so stress 2 is held to 3x its measured worst, above the 1e-4 of the other stages
    "scores": 4e-5, ("scores", "synthetic"): 3e-4,          # 1.3e-5 bounded, 1.04e-4 synthetic
    "sgru": 6e-5, "cgru": 6e-5,                             # 1.8e-5, 1.7e-5 (clipping regime)
    "dense": 6e-7, "catattn": 8e-7, "catpool": 6e-7,        # 1.9e-7, 2.5e-7, 1.8e-7 of the magnitude pass
    "pool": 3e-6,                                           # 9.4e-7
}


def family(probe):
    return re.sub(r"\d+[ab]?$", "", probe.name)


def tol(probe, regime):
    f = family(probe)
    return TOL.get((f, regime), TOL[f])


def rel_bound(ref):
    """max(|ref|, rms(ref row)) per element: the bar of the recurrences and the scores."""
    ref = np.asarray(ref, np.float64)
    return np.maximum(np.abs(ref), np.sqrt((ref ** 2).mean(axis=-1, keepdims=True)))


def bound(probe, regime, ref, mag):
    """Per-element bound of |got - ref| (0 for the bit-exact probes)."""
    if probe.kind == "exact":
        return np.zeros(np.shape(ref))
    return tol(probe, regime) * (rel_bound(ref) if probe.kind == "recur" else mag)
