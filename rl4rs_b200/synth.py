"""Synthetic catalog / log / simulator weights of the RL4RS dataset's shape (SURVEY.md section 8d).

No dataset or checkpoint ships with the reference (README.md:22-24,89-138) and there is no
network, so every measurement and most parity cases run on data generated here:

* ``make_catalog``  -- a 283-item catalog in the ``item_info.csv`` layout (slate.py:28-65):
  40-d item vector, price, location in {1,2,3} by id range (1..39 / 40..147 / 148..283),
  special flag in {0,1,2} (164 / 6 / 113 items).
* ``make_log``      -- N log rows as structure-of-arrays (the GPU loader's layout) with the
  statistics of dataset A / b3 (tutorial.ipynb:68-73); ``render_records`` turns rows into the
  '@'-separated text format (datautil.py:20-32, data_preprocess.py:64-85) so the reference's
  own parser can read the very same rows.
* ``make_weights``  -- the DIEN W-table with Keras/TF1 default initialisers (section 8a/8d).
"""
import numpy as np

LOG_SEED = 1234
WEIGHT_SEED = 4321
CATALOG_SEED = 283


class Catalog(object):
    """Item table.  Row 0 is the implicit padding item (slate.py:42-46): zero vector, price 0."""

    def __init__(self, item_vec, price, location, special):
        self.item_vec = item_vec      # f64 [A, 40]  (row 0 zeros)
        self.price = price            # f64 [A]
        self.location = location      # i8  [A]   file column (1..3), row 0 = 0
        self.special = special        # i8  [A]   file column (0..2), row 0 = 0
        self.action_size = item_vec.shape[0]

    @property
    def special_items(self):
        """ids whose special column == 2 (slate.py:59)."""
        return np.nonzero(self.special == 2)[0].astype(np.int64)

    def action_emb(self, emb_size=32):
        """slate.py:47-52: last ``emb_size`` dims, L2-normalised, f64; row 0 zeros."""
        emb = np.zeros((self.action_size, emb_size))
        v = self.item_vec[1:, -emb_size:]
        emb[1:] = np.einsum("ij,i->ij", v, 1.0 / np.linalg.norm(v, axis=1))
        return emb

    def to_text(self):
        lines = ["item_id item_vec price location special_item"]
        for i in range(1, self.action_size):
            vec = ",".join(repr(float(x)) for x in self.item_vec[i])
            lines.append("%d %s %s %d %d" % (i, vec, repr(float(self.price[i])),
                                             int(self.location[i]), int(self.special[i])))
        return "\n".join(lines)   # no trailing newline (slate.py:30,40 would break on one)

    @staticmethod
    def from_text(text):
        rows = [x.split(" ") for x in text.split("\n")[1:] if x]
        A = len(rows) + 1
        item_vec = np.zeros((A, len(rows[0][1].split(","))))
        price = np.zeros(A)
        location = np.zeros(A, np.int8)
        special = np.zeros(A, np.int8)
        for (iid, vec, p, loc, sp) in rows:
            i = int(iid)
            item_vec[i] = [float(x) for x in vec.split(",")]
            price[i] = float(p)
            location[i] = int(loc)
            special[i] = int(sp)
        return Catalog(item_vec, price, location, special)

    @staticmethod
    def from_file(path):
        with open(path, "r") as f:
            return Catalog.from_text(f.read())


def make_catalog(n_items=283, vec_dim=40, seed=CATALOG_SEED):
    rs = np.random.RandomState(seed)
    A = n_items + 1
    item_vec = np.zeros((A, vec_dim))
    item_vec[1:] = np.round(rs.normal(0.0, 1.0, (n_items, vec_dim)), 4)
    price = np.zeros(A)
    price[1:] = np.round(rs.uniform(1.0, 60.0, n_items), 1)
    location = np.zeros(A, np.int8)
    ids = np.arange(A)
    location[(ids >= 1) & (ids < 40)] = 1
    location[(ids >= 40) & (ids < 148)] = 2
    location[ids >= 148] = 3
    special = np.zeros(A, np.int8)
    perm = rs.permutation(np.arange(1, A))
    n2 = int(round(113 * n_items / 283.0))
    n1 = int(round(6 * n_items / 283.0))
    special[perm[:n2]] = 2
    special[perm[n2:n2 + n1]] = 1
    return Catalog(item_vec, price, location, special)


class LogSoA(object):
    """Structure-of-arrays log (the GPU-resident layout, DESIGN.md section 3)."""

    FIELDS = ("timestamp", "session_id", "sequence_id", "user_cat", "user_dense", "user_seq",
              "seq_len", "items", "feedback")

    def __init__(self, **kw):
        for k in self.FIELDS:
            setattr(self, k, kw[k])
        self.hist = kw.get("hist")     # optional list of full-length histories (text rendering)

    @property
    def n(self):
        return self.user_cat.shape[0]

    def save(self, path):
        np.savez(path, **{k: getattr(self, k) for k in self.FIELDS})

    @staticmethod
    def load(path):
        z = np.load(path)
        return LogSoA(**{k: z[k] for k in LogSoA.FIELDS})


def _page_items(rs, n, catalog):
    """One logged page: 3 distinct ids per layer [1,39], [40,147], [148,283] (valid per
    slate.py:61-63) holding at most ONE special item (valid per slate.py:144-146)."""
    out = np.empty((n, 9), np.int32)
    A = catalog.action_size
    is_sp = catalog.special == 2
    bounds = ((1, min(39, A - 1)), (40, min(147, A - 1)), (148, A - 1))
    for k, (lo, hi) in enumerate(bounds):
        keys = rs.random_sample((n, hi - lo + 1))
        keys[:, is_sp[lo:hi + 1]] += 2.0                     # non-special ids sort first
        pick = np.argsort(keys, axis=1)[:, :3]
        out[:, 3 * k:3 * k + 3] = pick[:, np.arange(3) % pick.shape[1]] + lo    # a layer of 1-2 ids repeats them
    # half of the pages carry exactly one special item, in a random slot of the matching layer
    with_sp = rs.random_sample(n) < 0.5
    slot = rs.randint(0, 9, n)
    u = rs.random_sample(n)
    for k, (lo, hi) in enumerate(bounds):
        pool = np.nonzero(is_sp[lo:hi + 1])[0] + lo
        if not len(pool):
            continue
        sel = with_sp & (slot // 3 == k)
        out[sel, slot[sel]] = pool[(u[sel] * len(pool)).astype(np.int64)]
    return out


def make_log(n, pages=1, catalog=None, seed=LOG_SEED, hash_size=100000, maxlen=64,
             corrupt_frac=0.05, keep_hist=False):
    """N synthetic log rows.  ``pages``=1 -> dataset A rows (9 items), 4 -> b3 trajectories (36)."""
    rs = np.random.RandomState(seed)
    catalog = catalog or make_catalog()
    S = 9 * pages
    items = np.concatenate([_page_items(rs, n, catalog) for _ in range(pages)], axis=1)
    # deliberate corruption to exercise get_violation (slate.py:133-147) and Q6-Q9
    n_bad = int(n * corrupt_frac)
    bad = rs.choice(n, n_bad, replace=False) if n_bad else np.zeros(0, np.int64)
    kind = rs.randint(0, 3, n_bad)
    special_ids = catalog.special_items
    for r, k in zip(bad, kind):
        p = rs.randint(0, pages) * 9
        if k == 0:      # duplicate adjacent (or distance-2) id
            j = rs.randint(0, 7)
            items[r, p + j + 1 + rs.randint(0, 2)] = items[r, p + j]
        elif k == 1:    # wrong layer
            j = rs.randint(0, 9)
            items[r, p + j] = rs.randint(1, 284 if catalog.action_size >= 284 else catalog.action_size)
        else:           # two distinct special ids in the page
            js = rs.choice(9, 2, replace=False)
            sp = rs.choice(special_ids, 2, replace=False)
            items[r, p + js[0]] = sp[0]
            items[r, p + js[1]] = sp[1]
    feedback = (rs.random_sample((n, S)) < 0.35).astype(np.uint8)
    # history: length ~ Gamma(1.6, 22.7) clipped to [1,140] (mean ~36.3; ~14.5% exceed 64)
    L = np.clip(np.round(rs.gamma(1.6, 22.7, n)), 1, 140).astype(np.int32)
    full = rs.randint(1, catalog.action_size, (n, 140)).astype(np.int32)
    # pre-pad with 0 / keep the LAST maxlen ids (datautil.py:43-46)
    user_seq = np.zeros((n, maxlen), np.int32)
    cols = np.arange(maxlen)[None, :]
    eff = np.minimum(L, maxlen)[:, None]
    src = (L[:, None] - eff) + (cols - (maxlen - eff))           # index into full[:, :L]
    valid = cols >= (maxlen - eff)
    user_seq[valid] = np.take_along_axis(full, np.clip(src, 0, 139), axis=1)[valid]
    user_cat = rs.randint(0, hash_size, (n, 10)).astype(np.int32)
    dense = np.round(np.maximum(0.0, rs.normal(6.0, 6.0, (n, 32))), 3)
    dense[rs.random_sample((n, 32)) < 0.25] = 0.0
    user_dense = dense.astype(np.float32)
    log = LogSoA(
        timestamp=np.arange(n, dtype=np.int64), session_id=np.arange(1, n + 1, dtype=np.int64),
        sequence_id=np.ones(n, np.int32), user_cat=user_cat, user_dense=user_dense,
        user_seq=user_seq, seq_len=L, items=items.astype(np.int32), feedback=feedback,
        hist=[full[i, :L[i]].copy() for i in range(n)] if keep_hist else None)
    log._dense64 = dense if keep_hist else None
    return log


def render_records(log, catalog, rows=None):
    """Rows of the log as '@'-separated text records (no header; Appendix A of SURVEY.md)."""
    assert log.hist is not None, "make_log(..., keep_hist=True) is needed to render text"
    rows = range(log.n) if rows is None else rows
    out = []
    for i in rows:
        items = log.items[i]
        portrait = [str(int(x)) for x in log.user_cat[i]] + [repr(float(x)) for x in log._dense64[i]]
        pages = []
        for p in range(0, len(items), 9):
            pages.append(";".join(",".join(repr(float(x)) for x in catalog.item_vec[it])
                                  for it in items[p:p + 9]))
        out.append("@".join([
            str(int(log.timestamp[i])), str(int(log.session_id[i])), str(int(log.sequence_id[i])),
            ",".join(str(int(x)) for x in items),
            ",".join(str(int(x)) for x in log.feedback[i]),
            ",".join(str(int(x)) for x in log.hist[i]),
            ",".join(portrait), ";".join(pages), "1"]))
    return out


def _glorot_uniform(rs, shape):
    lim = np.sqrt(6.0 / (shape[0] + shape[1]))
    return rs.uniform(-lim, lim, shape).astype(np.float32)


def _glorot_normal(rs, shape):
    # keras glorot_normal: truncated normal, stddev = sqrt(2/(fan_in+fan_out)) / .8796
    std = np.sqrt(2.0 / (shape[0] + shape[1]))
    x = rs.normal(0.0, 1.0, shape)
    bad = np.abs(x) > 2.0
    while bad.any():
        x[bad] = rs.normal(0.0, 1.0, int(bad.sum()))
        bad = np.abs(x) > 2.0
    return (x * std / 0.87962566103423978).astype(np.float32)


def weight_shapes(cfg=None):
    cfg = cfg or {}
    H = cfg.get("category_hash_size", 100000)
    E = cfg.get("emb_size", 128)
    U = cfg.get("hidden_units", 128)
    D = cfg.get("dense_feature_num", 432)
    C = cfg.get("category_feature_num", 21)
    seq_num = cfg.get("seq_num", 2)
    shapes = [("emb_cat", (H, E)), ("dense_w1", (D, U)), ("dense_b1", (U,)),
              ("dense_w2", (U, U)), ("dense_b2", (U,)), ("emb_seq", (H, E))]
    for i in range(seq_num):
        shapes += [("gru%d_wg" % i, (2 * E, 2 * E)), ("gru%d_bg" % i, (2 * E,)),
                   ("gru%d_wc" % i, (2 * E, E)), ("gru%d_bc" % i, (E,)),
                   ("att%d_w1" % i, (4 * E, 64)), ("att%d_b1" % i, (64,)),
                   ("att%d_w2" % i, (64, 16)), ("att%d_b2" % i, (16,)),
                   ("att%d_k" % i, (16, 1)), ("att%d_b" % i, (1,)),
                   ("augru%d_wg" % i, (3 * E, 4 * E)), ("augru%d_bg" % i, (4 * E,)),
                   ("augru%d_wc" % i, (3 * E, 2 * E)), ("augru%d_bc" % i, (2 * E,))]
    shapes += [("obs_w", (2 * E * seq_num + U + E + C * E, 256)), ("obs_b", (256,)),
               ("rew_w", (256, 2)), ("rew_b", (2,))]
    return shapes


def dnn_weight_shapes(cfg=None):
    """W-table of the `dnn` simulator (rl4rs/nets/dnn.py:8-45): the graph's second Embedding feeds nothing and is
    not part of the table."""
    cfg = cfg or {}
    H, E, U = cfg.get("category_hash_size", 100000), cfg.get("emb_size", 128), cfg.get("hidden_units", 128)
    D = cfg.get("dense_feature_num", 432)
    return [("emb_cat", (H, E)), ("dense_w1", (D, U)), ("dense_b1", (U,)), ("dense_w2", (U, U)), ("dense_b2", (U,)),
            ("fc_w", (E + U, 256)), ("fc_b", (256,)), ("obs_w", (256, 256)), ("obs_b", (256,)),
            ("rew_w", (256, cfg.get("class_num", 2))), ("rew_b", (cfg.get("class_num", 2),))]


def make_dnn_weights(cfg=None, seed=WEIGHT_SEED, stress=1.0, bias_noise=0.0):
    """Keras default initialisers for the `dnn` simulator (embeddings U(-0.05, 0.05), Dense glorot-uniform, bias 0)."""
    rs = np.random.RandomState(seed)
    w = {}
    for name, shape in dnn_weight_shapes(cfg):
        if name.startswith("emb_"):
            w[name] = rs.uniform(-0.05, 0.05, shape).astype(np.float32)
        elif len(shape) == 1:
            w[name] = np.zeros(shape, np.float32)
            if bias_noise:
                w[name] += rs.normal(0.0, bias_noise, shape).astype(np.float32)
        else:
            w[name] = _glorot_uniform(rs, shape) * np.float32(stress)
    return w


def widedeep_weight_shapes(cfg=None):
    """W-table of the `widedeep` simulator (rl4rs/nets/widedeep.py:8-45); 'simulator_obs' is a Concatenate (no weights)."""
    cfg = cfg or {}
    H, E, U = cfg.get("category_hash_size", 100000), cfg.get("emb_size", 128), cfg.get("hidden_units", 128)
    D, C, S = cfg.get("dense_feature_num", 432), cfg.get("category_feature_num", 21), cfg.get("seq_num", 2)
    return [("emb_cat", (H, E)), ("dense_w1", (D, U)), ("dense_b1", (U,)), ("dense_w2", (U, U)), ("dense_b2", (U,)),
            ("emb_seq", (H, E)), ("fc_w", (S * E, 256)), ("fc_b", (256,)),
            ("rew_w", (256 + U + C * E, cfg.get("class_num", 2))), ("rew_b", (cfg.get("class_num", 2),))]


def _make_plain(shapes, seed, stress, bias_noise):
    rs = np.random.RandomState(seed)
    w = {}
    for name, shape in shapes:
        if name.startswith("emb_"):
            w[name] = rs.uniform(-0.05, 0.05, shape).astype(np.float32)
        elif len(shape) == 1:
            w[name] = np.zeros(shape, np.float32)
            if bias_noise:
                w[name] += rs.normal(0.0, bias_noise, shape).astype(np.float32)
        else:
            w[name] = _glorot_uniform(rs, shape) * np.float32(stress)
    return w


def make_widedeep_weights(cfg=None, seed=WEIGHT_SEED, stress=1.0, bias_noise=0.0):
    """Keras default initialisers for the `widedeep` simulator."""
    return _make_plain(widedeep_weight_shapes(cfg), seed, stress, bias_noise)


def lstm_weight_shapes(cfg=None):
    """W-table of the `lstm` simulator (rl4rs/nets/lstm.py:8-45, nets/utils.py:28-36,78-97): Keras GRU layers -- kernel
    [in, 3U], recurrent kernel [U, 3U], ONE bias [3U] (reset_after = False), gate order [z | r | h]."""
    cfg = cfg or {}
    H, E, U = cfg.get("category_hash_size", 100000), cfg.get("emb_size", 128), cfg.get("hidden_units", 128)
    D, C, S = cfg.get("dense_feature_num", 432), cfg.get("category_feature_num", 21), cfg.get("seq_num", 2)
    shapes = [("emb_cat", (H, E)), ("cgru_k", (E, 3 * U)), ("cgru_rk", (U, 3 * U)), ("cgru_b", (3 * U,)),
              ("dense_w1", (D, U)), ("dense_b1", (U,)), ("dense_w2", (U, U)), ("dense_b2", (U,)), ("emb_seq", (H, E))]
    for i in range(S):
        shapes += [("sgru%d_k" % i, (E, 3 * U)), ("sgru%d_rk" % i, (U, 3 * U)), ("sgru%d_b" % i, (3 * U,))]
    return shapes + [("obs_w", (S * U + U + U + C * E, 256)), ("obs_b", (256,)),
                     ("rew_w", (256, cfg.get("class_num", 2))), ("rew_b", (cfg.get("class_num", 2),))]


def make_lstm_weights(cfg=None, seed=WEIGHT_SEED, stress=1.0, bias_noise=0.0, gru_stress=1.0, gru_bias_noise=None):
    """Keras default initialisers for the `lstm` simulator (the recurrent kernels get glorot instead of orthogonal: same
    scale, and nothing downstream depends on orthogonality).  ``gru_stress`` scales the GRU kernels only and
    ``gru_bias_noise`` replaces the GRU biases by N(0, gru_bias_noise): with default initialisers the gate pre-activations
    stay inside (-2.5, 2.5) and the hard sigmoid never clips; (2.5, 1.5) clips ~25 % of the gates and is still
    well-conditioned (f32 and f64 oracles agree to 2e-6), larger kernels make the recurrence chaotic."""
    w = _make_plain(lstm_weight_shapes(cfg), seed, stress, bias_noise)
    rs = np.random.RandomState(seed + 17)
    for k in sorted(w):
        if "gru" in k and not k.endswith("_b") and gru_stress != 1.0:
            w[k] = (w[k] * np.float32(gru_stress)).astype(np.float32)
        if "gru" in k and k.endswith("_b") and gru_bias_noise is not None:
            w[k] = rs.normal(0.0, gru_bias_noise, w[k].shape).astype(np.float32)
    return w


def make_weights(cfg=None, seed=WEIGHT_SEED, stress=1.0, bias_noise=0.0, bounded_scores=False):
    """W-table with TF1/Keras default initialisers; ``stress`` scales all non-embedding kernels,
    ``bias_noise`` adds N(0, bias_noise) to every bias (so parity tests see non-trivial biases).
    ``bounded_scores`` makes the attention read-out ``att*_k`` positive with unit sum and its bias
    ~0, so DIN scores stay in (0,1) like a trained model's and the AUGRU update gate
    (1-score)*u stays a convex weight; with raw glorot read-outs the scores are unbounded
    (nets/utils.py:121-122 uses weight_normalization=False) and large weights make the
    recurrence grow geometrically, which tests nothing but overflow."""
    rs = np.random.RandomState(seed)
    w = {}
    for name, shape in weight_shapes(cfg):
        if name.startswith("emb_"):
            w[name] = rs.uniform(-0.05, 0.05, shape).astype(np.float32)
        elif len(shape) == 1:
            gate_bias = name.endswith("_bg")               # GRUCell gate bias init 1
            w[name] = np.full(shape, 1.0 if gate_bias else 0.0, np.float32)
            if bias_noise:
                noise = rs.normal(0.0, bias_noise, shape).astype(np.float32)
                if bounded_scores and name.startswith("att") and name.endswith("_b"):
                    noise = np.abs(noise) * np.float32(0.1)
                w[name] += noise
        elif name.startswith("att"):
            w[name] = _glorot_normal(rs, shape) * np.float32(stress)
            if bounded_scores and name.endswith("_k"):
                k = np.abs(w[name]) + np.float32(1e-3)
                w[name] = (k / k.sum()).astype(np.float32)
        else:
            w[name] = _glorot_uniform(rs, shape) * np.float32(stress)
    return w
