"""Device engine: owns the r4_env handle, the HBM-resident log and the per-step output buffers.

PyTorch is plumbing here (device memory, streams, pinned host staging); all compute is in
librl4rs_b200.so.  One Engine per process / GPU; env rows shard across processes by contiguous
blocks (DESIGN.md section 6), there is no data-path collective.
"""
import ctypes as C

import numpy as np
import torch

from . import _capi
from .synth import Catalog, LogSoA

OBS_DIM = 256


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class Engine(object):
    def __init__(self, config, seq, catalog, weights, log, device=None):
        if not torch.cuda.is_available():
            raise _capi.R4Error("rl4rs_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.lib = _capi.load_library()
        self.config = config
        self.seq = bool(seq)
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.B = int(config["batch_size"])
        self.T = int(config["max_steps"])
        self.P = int(config.get("page_items", 9))
        self.A = int(config["action_size"])
        flags = 0
        for key, bit in (("support_rllib_mask", _capi.FLAG_RLLIB_MASK), ("support_d3rl_mask", _capi.FLAG_D3RL_MASK),
                         ("support_conti_env", _capi.FLAG_CONTI), ("support_onehot_action", _capi.FLAG_ONEHOT),
                         ("rawstate_as_obs", _capi.FLAG_RAWSTATE), ("simulator_info_fetch", _capi.FLAG_INFO_FETCH)):
            if config.get(key, False):
                flags |= bit
        self.flags = flags
        self.conti = bool(flags & _capi.FLAG_CONTI)
        self.raw = bool(flags & _capi.FLAG_RAWSTATE)
        self.rllib = bool(flags & _capi.FLAG_RLLIB_MASK)
        self.d3rl = bool(flags & _capi.FLAG_D3RL_MASK) and not self.rllib   # slate.py:92,98: elif
        self.info_fetch = bool(flags & _capi.FLAG_INFO_FETCH)
        if flags & _capi.FLAG_ONEHOT:                                   # slate.py:22-25
            config["action_emb_size"] = self.A
        self.emb_dim = self.A if flags & _capi.FLAG_ONEHOT else int(config.get("action_emb_size", 32))
        cfg = _capi.R4Config(
            env_kind=_capi.ENV_SEQSLATE if seq else _capi.ENV_SLATE, flags=flags, batch_size=self.B,
            max_steps=self.T, page_items=self.P, action_size=self.A,
            action_emb_size=int(config.get("action_emb_size", 32)), maxlen=int(config.get("maxlen", 64)),
            seq_num=int(config.get("seq_num", 2)), dense_feature_num=int(config.get("dense_feature_num", 432)),
            category_feature_num=int(config.get("category_feature_num", 21)),
            category_hash_size=int(config.get("category_hash_size", 100000)),
            emb_size=int(config.get("emb_size", 128)), hidden_units=int(config.get("hidden_units", 128)),
            max_rows_per_pass=int(config.get("max_rows_per_pass", 0)),
            simulator=_capi.SIMULATORS[config.get("algo", "dien")])
        h = C.c_void_p()
        rc = self.lib.r4_create(C.byref(cfg), self.device.index, C.byref(h))
        _capi.check(self.lib, None, rc, "r4_create")
        self.h = h
        self.obs_dim = int(self.lib.r4_obs_dim(_capi.SIMULATORS[config.get("algo", "dien")]))
        self.stream = torch.cuda.current_stream(self.device)
        self._load_items(catalog)
        self._load_weights(weights)
        self._load_log(log)
        self._alloc_outputs()
        self.env_launches0 = 0

    # ---- static data -------------------------------------------------------------------------
    def _sp(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _load_items(self, catalog):
        assert isinstance(catalog, Catalog)
        if catalog.action_size != self.A:
            raise ValueError("catalog has %d rows, config action_size is %d" % (catalog.action_size, self.A))
        self.catalog = catalog
        self.action_emb = (np.eye(self.A) if self.flags & _capi.FLAG_ONEHOT
                           else catalog.action_emb(self.emb_dim))          # slate.py:21-25,47-52
        vec = np.ascontiguousarray(catalog.item_vec, dtype=np.float64)
        price = np.ascontiguousarray(catalog.price, dtype=np.float64)
        special = np.ascontiguousarray(catalog.special == 2, dtype=np.uint8)
        emb = np.ascontiguousarray(self.action_emb, dtype=np.float64)
        rc = self.lib.r4_load_items(self.h, vec.ctypes.data, vec.shape[1], price.ctypes.data,
                                    special.ctypes.data, emb.ctypes.data, emb.shape[1], self.A)
        _capi.check(self.lib, self.h, rc, "r4_load_items")

    def _load_weights(self, weights):
        for name, arr in weights.items():
            if isinstance(arr, torch.Tensor):        # host or device tensor: r4_load_weight reads either pointer
                a = arr.detach().to(torch.float32).contiguous()
                shape, ptr = (C.c_int64 * a.dim())(*a.shape), a.data_ptr()
            else:
                a = np.ascontiguousarray(arr, dtype=np.float32)
                shape, ptr = (C.c_int64 * a.ndim)(*a.shape), a.ctypes.data
            rc = self.lib.r4_load_weight(self.h, name.encode(), ptr, shape, len(shape))
            _capi.check(self.lib, self.h, rc, "r4_load_weight(%s)" % name)
        rc = self.lib.r4_finalize_weights(self.h, self._sp())
        _capi.check(self.lib, self.h, rc, "r4_finalize_weights")

    def _load_log(self, log):
        assert isinstance(log, LogSoA)
        # Ids index the embedding tables, the price table and action_emb on the device: reject what the reference's
        # TF Embedding lookup / dict lookup would reject on the CPU (out-of-range or negative ids) once, here.
        H = int(self.config.get("category_hash_size", 100000))
        for name, arr, hi in (("user_protrait ids", log.user_cat, H), ("user_seqfeature ids", log.user_seq, H),
                              ("exposed_items", log.items, self.A)):
            a = np.asarray(arr)
            if a.size and (a.min() < 0 or a.max() >= hi):
                raise ValueError("log %s out of range [0, %d): min %d, max %d" % (name, hi, a.min(), a.max()))
        if log.items.shape[1] < (self.P if self.seq else min(self.T, self.P)):
            raise ValueError("log rows carry %d exposed items, the env needs at least %d" % (log.items.shape[1], self.P))
        self.log = log
        dev = self.device
        self.d_cat = torch.from_numpy(np.ascontiguousarray(log.user_cat, dtype=np.int32)).to(dev)
        self.d_dense = torch.from_numpy(np.ascontiguousarray(log.user_dense, dtype=np.float32)).to(dev)
        self.d_seq = torch.from_numpy(np.ascontiguousarray(log.user_seq, dtype=np.int32)).to(dev)
        self.d_items = torch.from_numpy(np.ascontiguousarray(log.items, dtype=np.int32)).to(dev)
        self.d_fb = torch.from_numpy(np.ascontiguousarray(log.feedback, dtype=np.uint8)).to(dev)
        rc = self.lib.r4_load_log(self.h, _ptr(self.d_cat), _ptr(self.d_dense), _ptr(self.d_seq),
                                  _ptr(self.d_items), _ptr(self.d_fb), log.n, log.items.shape[1])
        _capi.check(self.lib, self.h, rc, "r4_load_log")

    def _alloc_outputs(self):
        dev, B = self.device, self.B
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)
        self.rows = z((B,), torch.int32)
        self.obs = None if self.raw else z((B, self.obs_dim), torch.float32)
        self.mask = z((B, self.A), torch.uint8) if self.rllib else None
        self.reward = z((B,), torch.float64)
        self.chosen = z((B,), torch.int32)
        c = self.config
        self.cat = z((B, int(c.get("category_feature_num", 21))), torch.int32) if self.raw else None
        self.dense = z((B, int(c.get("dense_feature_num", 432))), torch.float32) if self.raw else None
        self.seqf = z((B, int(c.get("seq_num", 2)), int(c.get("maxlen", 64))), torch.int32) if self.raw else None
        # one click probability per reward row: a page (SeqSlate) or the whole slate of max_steps items (Slate)
        self.click_p = z((B, self.P if self.seq else self.T), torch.float32) if self.info_fetch else None
        self.masked = z((B, self.P if self.seq else self.T), torch.int32) if self.d3rl else None
        self.out = _capi.R4Out(
            obs=_ptr(self.obs), action_mask=_ptr(self.mask), reward=_ptr(self.reward), done=None,
            chosen=_ptr(self.chosen), cat=_ptr(self.cat), dense=_ptr(self.dense), seq=_ptr(self.seqf),
            click_p=_ptr(self.click_p), masked_actions=_ptr(self.masked))
        self.act_i32 = z((B,), torch.int32)
        self.act_f32 = z((B, self.emb_dim), torch.float32) if self.conti else None
        self.act_f64 = z((B, self.emb_dim), torch.float64) if self.conti else None
        self.pin_act_i32 = torch.zeros((B,), dtype=torch.int32).pin_memory()
        self.pin_rows = torch.zeros((B,), dtype=torch.int32).pin_memory()
        self._ev_rows, self._ev_act = torch.cuda.Event(), torch.cuda.Event()   # guard reuse of the staging buffers
        self.paid = False       # did the last step compute a reward (click_p valid)?

    # ---- episode -----------------------------------------------------------------------------
    def reset(self, rows):
        """rows: int array [B] of log rows (host) or an int32 device tensor."""
        if isinstance(rows, torch.Tensor):
            # device-resident row indices are TRUSTED (checking them would cost a host synchronisation per reset):
            # the caller guarantees 0 <= rows < log.n, as trainer.py / dataset.py do
            self.rows.copy_(rows.to(torch.int32), non_blocking=True)
        else:
            rows = np.asarray(rows)
            if rows.shape != (self.B,):
                raise ValueError("reset needs %d row indices" % self.B)
            if rows.min() < 0 or rows.max() >= self.log.n:
                raise IndexError("log row out of range")
            # the previous episode's copy may still be queued behind its kernels (torch mode never syncs):
            # wait for it before the staging buffer is overwritten
            self._ev_rows.synchronize()
            self.pin_rows.numpy()[:] = rows
            self.rows.copy_(self.pin_rows, non_blocking=True)
            self._ev_rows.record()
        rc = self.lib.r4_reset(self.h, _ptr(self.rows), C.byref(self.out), self._sp())
        _capi.check(self.lib, self.h, rc, "r4_reset")
        self.paid = False

    def step(self, action):
        """action: ints [B] (discrete) or floats [B, emb] (conti); host array/list or device tensor."""
        is_f64 = 0
        if isinstance(action, torch.Tensor) and action.is_cuda:
            if self.conti:
                if action.dtype == torch.float64:
                    a, is_f64 = action.contiguous(), 1
                else:
                    a = action.to(torch.float32).contiguous()
            else:
                a = action.to(torch.int32).contiguous()
        else:
            arr = np.asarray(action)
            if self.conti:
                if arr.shape != (self.B, self.emb_dim):
                    raise ValueError("continuous action must have shape (%d, %d)" % (self.B, self.emb_dim))
                if arr.dtype == np.float32:
                    self.act_f32.copy_(torch.from_numpy(np.ascontiguousarray(arr)), non_blocking=False)
                    a = self.act_f32
                else:
                    self.act_f64.copy_(torch.from_numpy(np.ascontiguousarray(arr, dtype=np.float64)))
                    a, is_f64 = self.act_f64, 1
            else:
                arr = arr.reshape(-1)
                if arr.shape != (self.B,):
                    raise ValueError("discrete action must have %d entries" % self.B)
                if arr.size and (arr.min() < 0 or arr.max() >= self.A):
                    raise IndexError("action id out of range [0, %d)" % self.A)   # slate.py:199 IndexError
                self._ev_act.synchronize()
                self.pin_act_i32.numpy()[:] = arr
                self.act_i32.copy_(self.pin_act_i32, non_blocking=True)
                self._ev_act.record()
                a = self.act_i32
        self._keep = a
        cur = self.cur_steps
        rc = self.lib.r4_step(self.h, _ptr(a), is_f64, C.byref(self.out), self._sp())
        _capi.check(self.lib, self.h, rc, "r4_step")
        nxt = cur + 1
        self.paid = (nxt % self.P == 0) if self.seq else (nxt >= self.T)

    @property
    def cur_steps(self):
        return int(self.lib.r4_cur_steps(self.h))

    def prev_actions(self):
        """Copy of SlateState.prev_actions as a device tensor i32 [B, max_steps]."""
        t = torch.empty((self.B, self.T), dtype=torch.int32, device=self.device)
        rc = self.lib.r4_copy_prev_actions(self.h, _ptr(t), self._sp())
        _capi.check(self.lib, self.h, rc, "r4_copy_prev_actions")
        return t

    def offline_action(self):
        items = torch.empty((self.B,), dtype=torch.int32, device=self.device)
        emb = torch.empty((self.B, self.emb_dim), dtype=torch.float64, device=self.device) if self.conti else None
        rc = self.lib.r4_offline_action(self.h, _ptr(items), _ptr(emb), self._sp())
        _capi.check(self.lib, self.h, rc, "r4_offline_action")
        return items, emb

    def offline_reward(self):
        out = torch.empty((self.B,), dtype=torch.float64, device=self.device)
        rc = self.lib.r4_offline_reward(self.h, _ptr(out), self._sp())
        _capi.check(self.lib, self.h, rc, "r4_offline_reward")
        return out

    def violation(self):
        out = torch.empty((self.B,), dtype=torch.int32, device=self.device)
        rc = self.lib.r4_violation(self.h, _ptr(out), self._sp())
        _capi.check(self.lib, self.h, rc, "r4_violation")
        return out

    def log_row_of(self, record):
        """Row index of a record string in the resident log (text-ingested logs only)."""
        idx = getattr(self, "_line_index", None)
        if idx is None:
            lines = getattr(self.log, "lines", None)
            if lines is None:
                raise ValueError("the log was not ingested from text: pass row indices as records")
            idx = self._line_index = {}
            for i, ln in enumerate(lines):
                idx.setdefault(ln, i)
        return idx[record]

    def features(self):
        """(cat i32[B,21], dense f32[B,432], seq i32[B,2,64]) of the current state, device tensors (r4_features)."""
        c = self.config
        cat = torch.empty((self.B, int(c.get("category_feature_num", 21))), dtype=torch.int32, device=self.device)
        dense = torch.empty((self.B, int(c.get("dense_feature_num", 432))), dtype=torch.float32, device=self.device)
        seq = torch.empty((self.B, int(c.get("seq_num", 2)), int(c.get("maxlen", 64))), dtype=torch.int32, device=self.device)
        rc = self.lib.r4_features(self.h, _ptr(cat), _ptr(dense), _ptr(seq), self._sp())
        _capi.check(self.lib, self.h, rc, "r4_features")
        return cat, dense, seq

    def nearest_neighbor(self, actions):
        a = torch.as_tensor(np.ascontiguousarray(actions, dtype=np.float64)).to(self.device)
        out = torch.empty((a.shape[0],), dtype=torch.int32, device=self.device)
        rc = self.lib.r4_nearest_neighbor(self.h, _ptr(a), 1, a.shape[0], _ptr(out), self._sp())
        _capi.check(self.lib, self.h, rc, "r4_nearest_neighbor")
        return out

    def dien_forward(self, seq, dense, cat):
        """The simulator alone (nets/dien.py:8-45) on explicit feature rows -> (obs, probs)."""
        dev = self.device
        seq = torch.as_tensor(np.ascontiguousarray(seq, dtype=np.int32)).to(dev)
        dense = torch.as_tensor(np.ascontiguousarray(dense, dtype=np.float32)).to(dev)
        cat = torch.as_tensor(np.ascontiguousarray(cat, dtype=np.int32)).to(dev)
        n = seq.shape[0]
        obs = torch.empty((n, self.obs_dim), dtype=torch.float32, device=dev)
        probs = torch.empty((n, 2), dtype=torch.float32, device=dev)
        rc = self.lib.r4_dien_forward(self.h, _ptr(seq), _ptr(dense), _ptr(cat), n, _ptr(obs), _ptr(probs), self._sp())
        _capi.check(self.lib, self.h, rc, "r4_dien_forward")
        return obs, probs

    def to_host(self, **tensors):
        """Device tensors -> NumPy arrays.  Each result lives in a FRESH pinned host block (torch's caching host
        allocator makes that cheap), so the D2H copy lands directly in the array handed to the caller: all copies are
        enqueued asynchronously on the current stream, then ONE synchronisation, no second host memcpy."""
        outs = {}
        for name, t in tensors.items():
            pin = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
            pin.copy_(t, non_blocking=True)
            outs[name] = pin
        torch.cuda.current_stream(self.device).synchronize()
        return {k: v.numpy() for k, v in outs.items()}

    def launch_count(self):
        return int(self.lib.r4_launch_count(self.h))

    def profile(self, mode):
        """0 off / 1 time the AUGRU kernel / 2 time every kernel (CUDA events on the launch stream)."""
        _capi.check(self.lib, self.h, self.lib.r4_profile(self.h, int(mode)), "r4_profile")

    def profile_read(self):
        """-> list of dicts {name, ms, launches, work} for every kernel slot that launched."""
        out = []
        slot = 0
        while True:
            name, ms, n, work = C.c_char_p(), C.c_double(), C.c_int64(), C.c_double()
            rc = self.lib.r4_profile_read(self.h, slot, C.byref(name), C.byref(ms), C.byref(n), C.byref(work))
            if rc == 1:
                break
            _capi.check(self.lib, self.h, rc, "r4_profile_read")
            if n.value:
                out.append({"name": name.value.decode(), "ms": ms.value, "launches": n.value, "work": work.value})
            slot += 1
        return out

    def close(self):
        if getattr(self, "h", None):
            torch.cuda.synchronize(self.device)
            self.lib.r4_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
