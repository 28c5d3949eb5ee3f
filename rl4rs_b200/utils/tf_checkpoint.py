"""TF1 ``tf.train.Saver`` checkpoints (tensor-bundle V2) without TensorFlow: reader, writer, and the
variable-name map of the DIEN simulator graph -> the W-table the CUDA library loads.

The reference restores its simulator with ``tf.train.Saver().restore(sess, model_file)``
(rl4rs/env/base.py:119-131,148-151; files ``model.index`` + ``model.data-00000-of-00001``, README.md:124-137).
TensorFlow is not installable here, so the two files are decoded directly:

* ``<prefix>.index`` is a LevelDB-format sorted string table (blocks of prefix-compressed key/value entries with a
  restart array, a 5-byte trailer per block = compression type + masked crc32c, an index block, a 48-byte footer with
  magic 0xdb4775248b80fb57).  Key "" -> ``BundleHeaderProto``; every other key is a variable name -> ``BundleEntryProto``
  {dtype, shape, shard_id, offset, size, crc32c}.
* ``<prefix>.data-XXXXX-of-YYYYY`` holds the raw little-endian tensor bytes at those offsets.

``TensorBundleWriter`` writes the same format (used by the round-trip tests, and to export a W-table as a Saver-style
checkpoint).  ``load_dien_checkpoint`` maps the graph of rl4rs/nets/dien.py:8-45 + rl4rs/nets/utils.py:16-25,48-54,
100-129 onto the flat W-table names of SURVEY.md section 8a.  The reference ships no checkpoint, so the inner variable
names of the deepctr 0.9.0 layers are NOT verified against a real file; the resolver therefore keys on what is certain --
the Keras auto-names of the TOP-LEVEL layers in creation order and the variable SHAPES, which are unique inside every
such layer -- and accepts an explicit ``name_map`` for anything that differs.
"""
import os
import re
import struct

import numpy as np

TABLE_MAGIC = 0xdb4775248b80fb57
# tensorflow/core/framework/types.proto
DTYPES = {1: np.float32, 2: np.float64, 3: np.int32, 4: np.uint8, 5: np.int16, 6: np.int8, 9: np.int64, 10: np.bool_,
          17: np.uint16, 19: np.float16, 22: np.uint32, 23: np.uint64}
DTYPE_IDS = {np.dtype(v): k for k, v in DTYPES.items()}


# ---- crc32c (Castagnoli), masked as in leveldb / tensorflow ------------------------------------------
def _make_crc_table():
    tbl = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ 0x82F63B78 if c & 1 else c >> 1
        tbl.append(c)
    return tbl


_CRC_TABLE = _make_crc_table()


def crc32c(data, crc=0):
    crc ^= 0xFFFFFFFF
    tbl = _CRC_TABLE
    for b in bytes(data):
        crc = tbl[(crc ^ b) & 0xFF] ^ (crc >> 8)
    return crc ^ 0xFFFFFFFF


def mask_crc(crc):
    return (((crc >> 15) | (crc << 17)) + 0xa282ead8) & 0xFFFFFFFF


# ---- varints / minimal protobuf ---------------------------------------------------------------------
def _read_varint(buf, pos):
    out, shift = 0, 0
    while True:
        b = buf[pos]
        pos += 1
        out |= (b & 0x7F) << shift
        if not b & 0x80:
            return out, pos
        shift += 7


def _write_varint(v):
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _pb_fields(buf):
    """Yield (field_number, wire_type, value) of one serialized message."""
    pos, n = 0, len(buf)
    while pos < n:
        tag, pos = _read_varint(buf, pos)
        f, wt = tag >> 3, tag & 7
        if wt == 0:
            v, pos = _read_varint(buf, pos)
        elif wt == 1:
            v = buf[pos:pos + 8]
            pos += 8
        elif wt == 2:
            ln, pos = _read_varint(buf, pos)
            v = buf[pos:pos + ln]
            pos += ln
        elif wt == 5:
            v = buf[pos:pos + 4]
            pos += 4
        else:
            raise ValueError("unsupported protobuf wire type %d" % wt)
        yield f, wt, v


def _pb_field(f, wt, payload):
    tag = _write_varint((f << 3) | wt)
    if wt == 0:
        return tag + _write_varint(payload)
    if wt == 2:
        return tag + _write_varint(len(payload)) + payload
    return tag + payload


def _parse_shape(buf):
    dims = []
    for f, _, v in _pb_fields(buf):
        if f == 2:                                    # TensorShapeProto.dim
            size = 0
            for g, _, w in _pb_fields(v):
                if g == 1:
                    size = w if w < (1 << 63) else w - (1 << 64)
            dims.append(size)
    return tuple(dims)


def _parse_entry(buf):
    e = {"dtype": 0, "shape": (), "shard_id": 0, "offset": 0, "size": 0, "crc32c": None, "sliced": False}
    for f, wt, v in _pb_fields(buf):
        if f == 1:
            e["dtype"] = v
        elif f == 2:
            e["shape"] = _parse_shape(v)
        elif f == 3:
            e["shard_id"] = v
        elif f == 4:
            e["offset"] = v
        elif f == 5:
            e["size"] = v
        elif f == 6:
            e["crc32c"] = struct.unpack("<I", v)[0]
        elif f == 7:
            e["sliced"] = True
    return e


# ---- snappy (index blocks are normally stored uncompressed; decoded if they are not) -------------------
def _snappy_uncompress(buf):
    n, pos = _read_varint(buf, 0)
    out = bytearray()
    while pos < len(buf):
        tag = buf[pos]
        pos += 1
        kind = tag & 3
        if kind == 0:
            ln = tag >> 2
            if ln >= 60:
                nb = ln - 59
                ln = int.from_bytes(buf[pos:pos + nb], "little")
                pos += nb
            ln += 1
            out += buf[pos:pos + ln]
            pos += ln
            continue
        if kind == 1:
            ln = ((tag >> 2) & 7) + 4
            off = ((tag >> 5) << 8) | buf[pos]
            pos += 1
        elif kind == 2:
            ln = (tag >> 2) + 1
            off = buf[pos] | (buf[pos + 1] << 8)
            pos += 2
        else:
            ln = (tag >> 2) + 1
            off = int.from_bytes(buf[pos:pos + 4], "little")
            pos += 4
        if off == 0 or off > len(out):
            raise ValueError("corrupt snappy stream")
        for _ in range(ln):                            # overlapping copies are legal
            out.append(out[-off])
    if len(out) != n:
        raise ValueError("snappy length mismatch")
    return bytes(out)


# ---- table reader -----------------------------------------------------------------------------------
def _read_block(data, offset, size, verify=True):
    raw = data[offset:offset + size]
    ctype = data[offset + size]
    if verify:
        stored = struct.unpack("<I", data[offset + size + 1:offset + size + 5])[0]
        if mask_crc(crc32c(data[offset:offset + size + 1])) != stored:
            raise ValueError("checkpoint index: block checksum mismatch at offset %d" % offset)
    if ctype == 1:
        raw = _snappy_uncompress(raw)
    elif ctype != 0:
        raise ValueError("checkpoint index: unknown block compression %d" % ctype)
    return raw


def _block_entries(block):
    nrestart = struct.unpack("<I", block[-4:])[0]
    end = len(block) - 4 - 4 * nrestart
    pos, key = 0, b""
    while pos < end:
        shared, pos = _read_varint(block, pos)
        non_shared, pos = _read_varint(block, pos)
        vlen, pos = _read_varint(block, pos)
        key = key[:shared] + block[pos:pos + non_shared]
        pos += non_shared
        yield key, block[pos:pos + vlen]
        pos += vlen


def _read_handle(buf, pos=0):
    off, pos = _read_varint(buf, pos)
    size, pos = _read_varint(buf, pos)
    return off, size, pos


class TensorBundleReader(object):
    """``tf.train.load_checkpoint(prefix)`` without TensorFlow: ``variables()`` and ``get_tensor(name)``."""

    def __init__(self, prefix, verify_index=True):
        self.prefix = str(prefix)
        path = self.prefix + ".index"
        if not os.path.exists(path):
            raise FileNotFoundError("%s: not a Saver checkpoint prefix (no .index file)" % prefix)
        with open(path, "rb") as f:
            data = f.read()
        if len(data) < 48 or struct.unpack("<Q", data[-8:])[0] != TABLE_MAGIC:
            raise ValueError("%s is not a tensor-bundle index (bad table magic)" % path)
        footer = data[-48:]
        _, _, p = _read_handle(footer, 0)                               # metaindex handle (unused)
        ioff, isize, _ = _read_handle(footer, p)
        self.entries, self.header = {}, None
        for _, handle in _block_entries(_read_block(data, ioff, isize, verify_index)):
            boff, bsize, _ = _read_handle(handle)
            for key, val in _block_entries(_read_block(data, boff, bsize, verify_index)):
                if key == b"":
                    self.header = self._parse_header(val)
                else:
                    self.entries[key.decode()] = _parse_entry(val)
        if self.header is None:
            raise ValueError("%s: no bundle header" % path)
        if self.header["endianness"] != 0:
            raise ValueError("big-endian tensor bundles are not supported")
        self._shards = {}

    @staticmethod
    def _parse_header(buf):
        h = {"num_shards": 1, "endianness": 0}
        for f, _, v in _pb_fields(buf):
            if f == 1:
                h["num_shards"] = v
            elif f == 2:
                h["endianness"] = v
        return h

    def variables(self):
        """name -> (numpy dtype, shape)"""
        return {k: (DTYPES.get(e["dtype"]), e["shape"]) for k, e in self.entries.items()}

    def _shard(self, i):
        if i not in self._shards:
            path = "%s.data-%05d-of-%05d" % (self.prefix, i, self.header["num_shards"])
            self._shards[i] = np.memmap(path, dtype=np.uint8, mode="r")
        return self._shards[i]

    def get_tensor(self, name, verify=None):
        e = self.entries[name]
        if e["sliced"]:
            raise ValueError("%s: partitioned (sliced) variables are not supported" % name)
        dt = DTYPES.get(e["dtype"])
        if dt is None:
            raise ValueError("%s: unsupported dtype id %d" % (name, e["dtype"]))
        raw = self._shard(e["shard_id"])[e["offset"]:e["offset"] + e["size"]]
        want = int(np.prod(e["shape"], dtype=np.int64)) * np.dtype(dt).itemsize
        if want != e["size"]:
            raise ValueError("%s: %d bytes stored, shape %s needs %d" % (name, e["size"], e["shape"], want))
        if verify is None:
            verify = e["size"] <= (1 << 20)             # pure-Python crc: small tensors only by default
        if verify and e["crc32c"] is not None and mask_crc(crc32c(raw.tobytes())) != e["crc32c"]:
            raise ValueError("%s: tensor checksum mismatch" % name)
        return np.frombuffer(raw.tobytes(), dtype=dt).reshape(e["shape"])


# ---- writer -----------------------------------------------------------------------------------------
def _block(entries):
    """One table block with a restart point at every entry (legal: shared = 0 throughout)."""
    out, restarts = bytearray(), []
    for k, v in entries:
        restarts.append(len(out))
        out += _write_varint(0) + _write_varint(len(k)) + _write_varint(len(v)) + k + v
    for r in restarts or [0]:
        out += struct.pack("<I", r)
    out += struct.pack("<I", max(len(restarts), 1))
    return bytes(out)


def _append_block(buf, block):
    off = len(buf)
    buf += block + b"\x00"
    buf += struct.pack("<I", mask_crc(crc32c(block + b"\x00")))
    return _write_varint(off) + _write_varint(len(block))


def write_bundle(prefix, tensors, entries_per_block=16, with_crc=True):
    """Write ``{name: array}`` as a V2 checkpoint (``prefix.index`` + ``prefix.data-00000-of-00001``)."""
    names = sorted(tensors, key=lambda s: s.encode())
    data, items = bytearray(), []
    header = _pb_field(1, 0, 1) + _pb_field(3, 2, _pb_field(1, 0, 1))      # num_shards = 1, version.producer = 1
    items.append((b"", header))
    for nm in names:
        a = np.asarray(tensors[nm], order="C")
        if a.dtype not in DTYPE_IDS:
            raise ValueError("%s: dtype %s cannot be stored" % (nm, a.dtype))
        raw = a.tobytes()
        shape = b"".join(_pb_field(2, 2, _pb_field(1, 0, int(d))) for d in a.shape)
        ent = _pb_field(1, 0, DTYPE_IDS[a.dtype]) + _pb_field(2, 2, shape)
        if len(data):
            ent += _pb_field(4, 0, len(data))
        ent += _pb_field(5, 0, len(raw))
        if with_crc and len(raw) <= (1 << 20):
            ent += _pb_field(6, 5, struct.pack("<I", mask_crc(crc32c(raw))))
        items.append((nm.encode(), ent))
        data += raw
    buf, index = bytearray(), []
    for i in range(0, len(items), entries_per_block):
        chunk = items[i:i + entries_per_block]
        index.append((chunk[-1][0], _append_block(buf, _block(chunk))))
    meta = _append_block(buf, _block([]))
    idx = _append_block(buf, _block(index))
    footer = meta + idx
    buf += footer + b"\x00" * (40 - len(footer)) + struct.pack("<Q", TABLE_MAGIC)
    os.makedirs(os.path.dirname(os.path.abspath(prefix)) or ".", exist_ok=True)
    with open(str(prefix) + ".index", "wb") as f:
        f.write(buf)
    with open(str(prefix) + ".data-00000-of-00001", "wb") as f:
        f.write(data)
    return prefix


# ---- DIEN graph -> W-table ----------------------------------------------------------------------------
def dien_layer_plan(config=None):
    """[(W-table name, top-level Keras layer scope, variable shape)] for the graph of nets/dien.py:8-45.

    Scopes are the Keras auto-names in creation order inside a fresh graph (base.py:119-121 builds one per simulator):
    id_input_processing_attn -> Embedding #0; dense_input_processing -> Dense #0, #1; sequence_input_attn -> Embedding #1,
    then per sequence DynamicGRU (GRU), AttentionSequencePoolingLayer, DynamicGRU (AUGRU); then the two named Dense heads."""
    cfg = config or {}
    H, E, U = cfg.get("category_hash_size", 100000), cfg.get("emb_size", 128), cfg.get("hidden_units", 128)
    D, C, S = cfg.get("dense_feature_num", 432), cfg.get("category_feature_num", 21), cfg.get("seq_num", 2)
    cls = cfg.get("class_num", 2)
    suf = lambda base, k: base if k == 0 else "%s_%d" % (base, k)
    plan = [("emb_cat", "embedding", (H, E)),
            ("dense_w1", "dense", (D, U)), ("dense_b1", "dense", (U,)),
            ("dense_w2", "dense_1", (U, U)), ("dense_b2", "dense_1", (U,)),
            ("emb_seq", "embedding_1", (H, E))]
    for i in range(S):
        g, a, u = suf("dynamic_gru", 2 * i), suf("attention_sequence_pooling_layer", i), suf("dynamic_gru", 2 * i + 1)
        plan += [("gru%d_wg" % i, g, (2 * E, 2 * E)), ("gru%d_bg" % i, g, (2 * E,)),
                 ("gru%d_wc" % i, g, (2 * E, E)), ("gru%d_bc" % i, g, (E,)),
                 ("att%d_w1" % i, a, (4 * E, 64)), ("att%d_b1" % i, a, (64,)),
                 ("att%d_w2" % i, a, (64, 16)), ("att%d_b2" % i, a, (16,)),
                 ("att%d_k" % i, a, (16, 1)), ("att%d_b" % i, a, (1,)),
                 ("augru%d_wg" % i, u, (3 * E, 4 * E)), ("augru%d_bg" % i, u, (4 * E,)),
                 ("augru%d_wc" % i, u, (3 * E, 2 * E)), ("augru%d_bc" % i, u, (2 * E,))]
    plan += [("obs_w", "simulator_obs", (2 * E * S + U + E + C * E, 256)), ("obs_b", "simulator_obs", (256,)),
             ("rew_w", "simulator_reward", (256, cls)), ("rew_b", "simulator_reward", (cls,))]
    return plan


# best-knowledge full TF1 variable names (deepctr 0.9.0 / TF 1.15 sources as published; unverified, documentation only:
# the resolver below does not depend on the inner names)
_INNER = {"emb_cat": "embeddings", "emb_seq": "embeddings", "dense_w1": "kernel", "dense_b1": "bias", "dense_w2": "kernel",
          "dense_b2": "bias", "obs_w": "kernel", "obs_b": "bias", "rew_w": "kernel", "rew_b": "bias",
          "gru_wg": "gru_cell/gates/kernel", "gru_bg": "gru_cell/gates/bias", "gru_wc": "gru_cell/candidate/kernel",
          "gru_bc": "gru_cell/candidate/bias", "augru_wg": "vec_att_gru_cell/gates/kernel",
          "augru_bg": "vec_att_gru_cell/gates/bias", "augru_wc": "vec_att_gru_cell/candidate/kernel",
          "augru_bc": "vec_att_gru_cell/candidate/bias", "att_w1": "local_activation_unit/dnn/kernel0",
          "att_b1": "local_activation_unit/dnn/bias0", "att_w2": "local_activation_unit/dnn/kernel1",
          "att_b2": "local_activation_unit/dnn/bias1", "att_k": "local_activation_unit/kernel",
          "att_b": "local_activation_unit/bias"}


def dien_variable_names(config=None):
    """W-table name -> expected TF1 variable name (documentation / writer side of the tests)."""
    out = {}
    for name, scope, _ in dien_layer_plan(config):
        out[name] = scope + "/" + _INNER[re.sub(r"^(gru|att|augru)\d+_", r"\1_", name)]
    return out


_SLOT = re.compile(r"(/Adam(_\d+)?$|/Momentum$|/RMSProp(_\d+)?$|^training/|^beta\d_power$|^Adam/|/optimizer/|^metrics/|^total|^count|^true_positives|^false_|^true_neg)")


def load_dien_checkpoint(prefix, config=None, name_map=None):
    """Saver prefix -> W-table ``{name: float32 array}`` (what ``r4_load_weight`` takes).

    Resolution per W-table entry: (1) ``name_map[name]`` if given; (2) the expected full name if present; (3) the one
    variable under the expected top-level scope whose shape matches (optimizer slots and metric counters ignored).
    Anything missing or ambiguous raises with the candidates listed."""
    return _load_by_plan(prefix, dien_layer_plan(config), dien_variable_names(config), name_map)


def dnn_layer_plan(config=None):
    """[(W-table name, top-level Keras layer scope, shape)] for the graph of nets/dnn.py:8-45 in creation order:
    id_input_processing -> Embedding #0; dense_input_processing -> Dense #0, #1; sequence_input_concat -> Embedding #1
    (feeds nothing, not loaded); Dense(256) -> Dense #2; then the two named heads."""
    cfg = config or {}
    H, E, U = cfg.get("category_hash_size", 100000), cfg.get("emb_size", 128), cfg.get("hidden_units", 128)
    D, cls = cfg.get("dense_feature_num", 432), cfg.get("class_num", 2)
    return [("emb_cat", "embedding", (H, E)), ("dense_w1", "dense", (D, U)), ("dense_b1", "dense", (U,)),
            ("dense_w2", "dense_1", (U, U)), ("dense_b2", "dense_1", (U,)),
            ("fc_w", "dense_2", (E + U, 256)), ("fc_b", "dense_2", (256,)),
            ("obs_w", "simulator_obs", (256, 256)), ("obs_b", "simulator_obs", (256,)),
            ("rew_w", "simulator_reward", (256, cls)), ("rew_b", "simulator_reward", (cls,))]


def dnn_variable_names(config=None):
    inner = {"emb_cat": "embeddings"}
    return {name: scope + "/" + inner.get(name, "kernel" if name.endswith(("_w", "_w1", "_w2")) else "bias")
            for name, scope, _ in dnn_layer_plan(config)}


def _load_by_plan(prefix, plan, expect, name_map):
    rd = TensorBundleReader(prefix)
    allv = rd.variables()
    live = {k: v for k, v in allv.items() if not _SLOT.search(k)}
    name_map = name_map or {}
    out, used = {}, set()
    for name, scope, shape in plan:
        if name in name_map:
            cand = name_map[name]
            if cand not in allv:
                raise KeyError("name_map[%s] = %s is not in the checkpoint" % (name, cand))
        elif expect[name] in live and tuple(live[expect[name]][1]) == tuple(shape):
            cand = expect[name]
        else:
            hits = [k for k, (dt, sh) in live.items()
                    if k.split("/")[0] == scope and tuple(sh) == tuple(shape) and k not in used]
            if len(hits) != 1:
                near = sorted(k for k in live if k.split("/")[0] == scope)
                raise KeyError("cannot resolve %s (scope %r, shape %s): %d candidates %s; variables under that scope: %s; "
                               "pass name_map={%r: <variable name>}" % (name, scope, shape, len(hits), hits, near, name))
            cand = hits[0]
        used.add(cand)
        arr = rd.get_tensor(cand)
        if tuple(arr.shape) != tuple(shape):
            raise ValueError("%s <- %s has shape %s, expected %s" % (name, cand, arr.shape, shape))
        out[name] = np.ascontiguousarray(arr, dtype=np.float32)
    return out


def load_dnn_checkpoint(prefix, config=None, name_map=None):
    """Saver prefix of a `dnn` simulator (nets/dnn.py) -> its W-table; same resolution rules as load_dien_checkpoint."""
    return _load_by_plan(prefix, dnn_layer_plan(config), dnn_variable_names(config), name_map)


def widedeep_layer_plan(config=None):
    """nets/widedeep.py:8-45 in creation order: id_input_processing_concat -> Embedding #0; dense tower -> Dense #0, #1;
    sequence_input_concat -> Embedding #1; Dense(256) on the pooled sequences -> Dense #2; simulator_obs is a Concatenate;
    simulator_reward."""
    cfg = config or {}
    H, E, U = cfg.get("category_hash_size", 100000), cfg.get("emb_size", 128), cfg.get("hidden_units", 128)
    D, C, S, cls = cfg.get("dense_feature_num", 432), cfg.get("category_feature_num", 21), cfg.get("seq_num", 2), cfg.get("class_num", 2)
    return [("emb_cat", "embedding", (H, E)), ("dense_w1", "dense", (D, U)), ("dense_b1", "dense", (U,)),
            ("dense_w2", "dense_1", (U, U)), ("dense_b2", "dense_1", (U,)), ("emb_seq", "embedding_1", (H, E)),
            ("fc_w", "dense_2", (S * E, 256)), ("fc_b", "dense_2", (256,)),
            ("rew_w", "simulator_reward", (256 + U + C * E, cls)), ("rew_b", "simulator_reward", (cls,))]


def widedeep_variable_names(config=None):
    inner = {"emb_cat": "embeddings", "emb_seq": "embeddings"}
    return {name: scope + "/" + inner.get(name, "kernel" if name.endswith(("_w", "_w1", "_w2")) else "bias")
            for name, scope, _ in widedeep_layer_plan(config)}


def load_widedeep_checkpoint(prefix, config=None, name_map=None):
    return _load_by_plan(prefix, widedeep_layer_plan(config), widedeep_variable_names(config), name_map)


def save_widedeep_checkpoint(prefix, weights, config=None):
    names = widedeep_variable_names(config)
    return write_bundle(prefix, {names[k]: np.asarray(v, dtype=np.float32) for k, v in weights.items() if k in names})


def lstm_layer_plan(config=None):
    """nets/lstm.py:8-45 in creation order: id_input_processing_lstm -> Embedding #0, GRU #0; dense tower -> Dense #0, #1;
    sequence_input_LSTM -> Embedding #1, GRU #1, #2 (one per sequence); simulator_obs; simulator_reward.  A Keras (v1,
    reset_after = False) GRU layer owns kernel [in, 3U], recurrent_kernel [U, 3U], bias [3U]."""
    cfg = config or {}
    H, E, U = cfg.get("category_hash_size", 100000), cfg.get("emb_size", 128), cfg.get("hidden_units", 128)
    D, C, S, cls = cfg.get("dense_feature_num", 432), cfg.get("category_feature_num", 21), cfg.get("seq_num", 2), cfg.get("class_num", 2)
    plan = [("emb_cat", "embedding", (H, E)), ("cgru_k", "gru", (E, 3 * U)), ("cgru_rk", "gru", (U, 3 * U)), ("cgru_b", "gru", (3 * U,)),
            ("dense_w1", "dense", (D, U)), ("dense_b1", "dense", (U,)), ("dense_w2", "dense_1", (U, U)), ("dense_b2", "dense_1", (U,)),
            ("emb_seq", "embedding_1", (H, E))]
    for i in range(S):
        sc = "gru_%d" % (i + 1)
        plan += [("sgru%d_k" % i, sc, (E, 3 * U)), ("sgru%d_rk" % i, sc, (U, 3 * U)), ("sgru%d_b" % i, sc, (3 * U,))]
    return plan + [("obs_w", "simulator_obs", (S * U + U + U + C * E, 256)), ("obs_b", "simulator_obs", (256,)),
                   ("rew_w", "simulator_reward", (256, cls)), ("rew_b", "simulator_reward", (cls,))]


def lstm_variable_names(config=None):
    def inner(name):
        if name.startswith("emb_"):
            return "embeddings"
        if name.endswith("_rk"):
            return "recurrent_kernel"
        return "kernel" if name.endswith(("_k", "_w", "_w1", "_w2")) else "bias"
    return {name: scope + "/" + inner(name) for name, scope, _ in lstm_layer_plan(config)}


def load_lstm_checkpoint(prefix, config=None, name_map=None):
    return _load_by_plan(prefix, lstm_layer_plan(config), lstm_variable_names(config), name_map)


def save_lstm_checkpoint(prefix, weights, config=None):
    names = lstm_variable_names(config)
    return write_bundle(prefix, {names[k]: np.asarray(v, dtype=np.float32) for k, v in weights.items() if k in names})


def save_dnn_checkpoint(prefix, weights, config=None):
    names = dnn_variable_names(config)
    return write_bundle(prefix, {names[k]: np.asarray(v, dtype=np.float32) for k, v in weights.items() if k in names})


def adversarial_slate_layer_plan(config=None):
    """nets/adversarial_slate.py in creation order: id_input_processing over the first 20 cat slots -> Embedding #0; dense
    tower -> Dense #0, #1; sequence_input_concat -> Embedding #1; the unnamed Dense(9, sigmoid) -> Dense #2."""
    cfg = config or {}
    H, E, U = cfg.get("category_hash_size", 100000), cfg.get("emb_size", 128), cfg.get("hidden_units", 128)
    D, S = cfg.get("dense_feature_num", 432), cfg.get("seq_num", 2)
    return [("emb_cat", "embedding", (H, E)), ("dense_w1", "dense", (D, U)), ("dense_b1", "dense", (U,)),
            ("dense_w2", "dense_1", (U, U)), ("dense_b2", "dense_1", (U,)), ("emb_seq", "embedding_1", (H, E)),
            ("rew_w", "dense_2", (S * E + U + E, 9)), ("rew_b", "dense_2", (9,))]


def adversarial_slate_variable_names(config=None):
    inner = {"emb_cat": "embeddings", "emb_seq": "embeddings"}
    return {name: scope + "/" + inner.get(name, "kernel" if name.endswith(("_w", "_w1", "_w2")) else "bias")
            for name, scope, _ in adversarial_slate_layer_plan(config)}


def load_adversarial_slate_checkpoint(prefix, config=None, name_map=None):
    return _load_by_plan(prefix, adversarial_slate_layer_plan(config), adversarial_slate_variable_names(config), name_map)


def save_adversarial_slate_checkpoint(prefix, weights, config=None):
    names = adversarial_slate_variable_names(config)
    return write_bundle(prefix, {names[k]: np.asarray(v, dtype=np.float32) for k, v in weights.items() if k in names})


def save_dien_checkpoint(prefix, weights, config=None):
    """W-table -> Saver-style checkpoint under the expected TF1 variable names (inverse of load_dien_checkpoint)."""
    names = dien_variable_names(config)
    return write_bundle(prefix, {names[k]: np.asarray(v, dtype=np.float32) for k, v in weights.items() if k in names})


def is_saver_prefix(path):
    return isinstance(path, str) and os.path.exists(path + ".index")
