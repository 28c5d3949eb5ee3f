"""rl4rs/mdpchecker/decoder.py: token_probs, decode_step and beam_search over a `transformer.get_model` model.

On CUDA a search is one r4_s2s_beam_search call per chunk of rows: the encoder and each decoder block's cross-attention
K / V run once per row, every step is one batched decoder pass over all n * beam prefixes, and the candidate mask, the
top-k per prefix, the top-beam of the beam^2 products and the path gather run on the device; the results come to the
host once.  On the CPU the torch twin runs the same search.  Order is probability descending, ties to the lower
(beam, token) index, as a stable sort gives (the reference's partition / quicksort leaves exact ties unordered)."""
import numpy as np
import torch

from rl4rs_b200 import _capi
from rl4rs_b200.mdpchecker import transformer as tf

START = 1


def token_probs(model, batch_inputs, batch_outputs):
    """The next-token probabilities f32 [n, V] after each prefix batch_outputs [n, t]."""
    return np.array(model.predict([np.array(batch_inputs), np.array(batch_outputs)]))[:, -1]


def _topk_sorted(p, k):
    """(values f64, indices) of the k largest entries of each row of p (f64), ties to the lower index."""
    order = torch.sort(-p, dim=1, stable=True).indices[:, :k]
    return p.gather(1, order), order


def _cand_mask(V, candidates, n, device):
    mask = torch.zeros(n, V, dtype=torch.float64, device=device)
    mask.scatter_(1, candidates.long(), 1.0)
    return mask


def decode_step(model, batch_inputs, batch_outputs, candidates=None, beam_size=1):
    """[n, beam_size, 2] f64 of (probability, token) of the beam_size most probable next tokens, times the candidate mask
    (candidates [n, C] token ids) when given."""
    enc, dec = np.asarray(batch_inputs), np.asarray(batch_outputs)
    n, V = len(enc), model.cfg.Vt
    if model.device.type == "cuda":
        lib = _capi.load_library()
        c = model.cfg.c()
        e32 = torch.as_tensor(enc.astype(np.int32), device=model.device)
        d32 = torch.as_tensor(dec.astype(np.int32), device=model.device)
        cand = None if candidates is None else torch.as_tensor(np.asarray(candidates).astype(np.int32),
                                                                device=model.device).contiguous()
        C = 0 if cand is None else cand.shape[1]
        val = torch.empty(n, beam_size, dtype=torch.float64, device=model.device)
        idx = torch.empty(n, beam_size, dtype=torch.int32, device=model.device)
        m, scr = model._chunk(_capi.S2S_STEP, n, enc.shape[1], dec.shape[1], 1, beam_size)
        for r0 in range(0, n, m):
            k = min(m, n - r0)
            _capi.check(lib, None, lib.r4_s2s_decode_step(
                _capi.C.byref(c), _capi.ptr(model.flat), _capi.ptr(e32[r0:r0 + k]), k, enc.shape[1],
                _capi.ptr(d32[r0:r0 + k]), dec.shape[1], _capi.ptr(cand[r0:r0 + k]) if cand is not None else None, C,
                beam_size, _capi.ptr(val[r0:r0 + k]), _capi.ptr(idx[r0:r0 + k]), _capi.ptr(scr),
                _capi.stream(model.device)), "r4_s2s_decode_step")
    else:
        p = model.predict_tensor(enc, dec)[:, -1].double()
        if candidates is not None:
            p = p * _cand_mask(V, torch.as_tensor(np.asarray(candidates)), n, p.device)
        val, idx = _topk_sorted(p, beam_size)
    return np.stack([val.cpu().numpy(), idx.cpu().numpy().astype(np.float64)], axis=-1)


def _search_twin(model, enc, beam_size, target_len, candidates_size):
    n, V, L = len(enc), model.cfg.Vt, target_len + 1
    path = torch.zeros(n, beam_size, L, dtype=torch.int64)
    path[:, :, 0] = START
    p = model.predict_tensor(enc, path[:, 0, :1].numpy())[:, -1].double().cpu()
    val, idx = _topk_sorted(p, beam_size)
    path[:, :, 1] = idx
    score = val
    mask = None
    if candidates_size:
        mask = _cand_mask(V, _topk_sorted(p, candidates_size)[1], n, p.device)
    encr = np.repeat(np.asarray(enc), beam_size, axis=0)
    for i in range(1, target_len):
        p = model.predict_tensor(encr, path[:, :, :i + 1].reshape(n * beam_size, i + 1).numpy())[:, -1].double().cpu()
        if mask is not None:
            p = p * mask.repeat_interleave(beam_size, 0)
        v, t = _topk_sorted(p, beam_size)
        prod = (score.reshape(n, beam_size, 1) * v.reshape(n, beam_size, beam_size)).reshape(n, -1)
        sv, f = _topk_sorted(prod, beam_size)
        b, j = f // beam_size, f % beam_size
        path = path.gather(1, b.unsqueeze(-1).expand(n, beam_size, L)).clone()
        path[:, :, i + 1] = t.reshape(n, beam_size, beam_size)[torch.arange(n)[:, None], b, j]
        score = sv
    return path.numpy(), score.numpy()


def beam_search(model, encode_input, beam_size, target_len, use_candidates=False, candidates_size=None):
    """(output_topk int [n, beam, target_len + 1], beam_score f64 [n, beam]) of the reference's beam search."""
    enc = np.asarray(encode_input)
    n, Ts = enc.shape
    ncand = int(candidates_size) if use_candidates else 0
    if model.device.type != "cuda":
        return _search_twin(model, enc, beam_size, target_len, ncand)
    lib = _capi.load_library()
    c = model.cfg.c()
    L = target_len + 1
    e32 = torch.as_tensor(enc.astype(np.int32), device=model.device)
    path = torch.empty(n, beam_size, L, dtype=torch.int32, device=model.device)
    score = torch.empty(n, beam_size, dtype=torch.float64, device=model.device)
    m, scr = model._chunk(_capi.S2S_SEARCH, n, Ts, target_len, beam_size, ncand)
    for r0 in range(0, n, m):
        k = min(m, n - r0)
        _capi.check(lib, None, lib.r4_s2s_beam_search(
            _capi.C.byref(c), _capi.ptr(model.flat), _capi.ptr(e32[r0:r0 + k]), k, Ts, beam_size, target_len, ncand,
            _capi.ptr(path[r0:r0 + k]), _capi.ptr(score[r0:r0 + k]), _capi.ptr(scr), _capi.stream(model.device)),
            "r4_s2s_beam_search")
    return path.cpu().numpy().astype(np.int64), score.cpu().numpy()


def path_probs(model, encode_input, output_topk):
    """Experiment I's scores f32 [n, beam, target_len]: entry i the probability of output_topk[., ., i + 1] after the
    prefix output_topk[., ., :i + 1].  The decoder's self-attention is causal, so one pass over each whole path gives
    every prefix's next-token probability (the reference makes one predict call per beam and prefix length)."""
    enc = np.asarray(encode_input)
    paths = np.asarray(output_topk)
    n, beam, L = paths.shape
    T = L - 1
    if model.device.type != "cuda":
        encr = np.repeat(enc, beam, axis=0)
        p = model.predict_tensor(encr, paths[:, :, :T].reshape(n * beam, T)).cpu()
        nxt = torch.as_tensor(paths[:, :, 1:].reshape(n * beam, T, 1).astype(np.int64)).clamp(0, model.cfg.Vt - 1)
        return p.gather(2, nxt).reshape(n, beam, T).numpy()
    lib = _capi.load_library()
    c = model.cfg.c()
    e32 = torch.as_tensor(enc.astype(np.int32), device=model.device)
    p32 = torch.as_tensor(paths.astype(np.int32), device=model.device).contiguous()
    out = torch.empty(n, beam, T, dtype=torch.float32, device=model.device)
    m, scr = model._chunk(_capi.S2S_PREDICT, n, enc.shape[1], T, beam)
    for r0 in range(0, n, m):
        k = min(m, n - r0)
        _capi.check(lib, None, lib.r4_s2s_score(_capi.C.byref(c), _capi.ptr(model.flat), _capi.ptr(e32[r0:r0 + k]), k,
                                                enc.shape[1], _capi.ptr(p32[r0:r0 + k]), beam, T, _capi.ptr(out[r0:r0 + k]),
                                                _capi.ptr(scr), _capi.stream(model.device)), "r4_s2s_score")
    return out.cpu().numpy()
