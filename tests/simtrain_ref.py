"""Shared by the simulator-training tests: synthetic item samples with teacher labels, and the float64 autograd reference of
the kernels' gradient (the torch twin SimulatorNet on a float64 copy of the flat parameters, as learner_ref64.py does for the
learners), with what it takes to run that reference at every shape the C-ABI accepts: a chunked run on any torch device,
embedding tables compacted to the rows a batch touches, the kernel's dropout draw in NumPy, samples at the id and length
edges, and a restatement of the kernel's scratch layout."""
import numpy as np
import torch

from rl4rs_b200 import policy, simtrain, synth


def make_samples(n_records, hash_size, seed=0, pages=True):
    """ItemSamples of n_records random page records: ids in [0, hash_size), histories of 1..80 ids (pre-padded), page numbers
    1..4 with the earlier pages' items as the second sequence."""
    rs = np.random.RandomState(seed)
    N = n_records
    seq = np.zeros((N, 2, 64), np.int32)
    sid = rs.randint(1, 5, N).astype(np.int32) if pages else np.ones(N, np.int32)
    for r in range(N):
        L = rs.randint(1, 81)
        h = rs.randint(1, hash_size, L)[-64:]
        seq[r, 0, 64 - len(h):] = h
        k = 9 * (sid[r] - 1)
        if k:
            seq[r, 1, 64 - k:] = rs.randint(1, hash_size, k)
    return simtrain.ItemSamples(
        hash_size, user_cat=rs.randint(0, hash_size, (N, 10)).astype(np.int32),
        user_dense=np.round(np.maximum(0.0, rs.normal(1.0, 1.0, (N, 32))), 3).astype(np.float32),
        sequence_id=sid, items=rs.randint(1, hash_size, (N, 9)).astype(np.int32),
        feedback=(rs.random_sample((N, 9)) < 0.35).astype(np.uint8),
        item_feature=np.round(rs.normal(0.0, 1.0, (N, 360)), 4).astype(np.float32), seq=seq)


# history lengths of the edge samples: empty, one id, exactly the window, truncated to it, and random ones in between
_HIST = (0, 1, 64, 80, None)
# the second sequence's length at page 1..8 (9 items per earlier page); page 8's 63 is raised to the full window of 64
_PAGE_LEN = (0, 9, 18, 27, 36, 45, 54, 64)


def make_edge_samples(n_records, hash_size, seed=0):
    """ItemSamples at the id and length edges: histories of 0, 1, 64 and 80 (truncated) ids besides random ones; page
    numbers 1..8, so the second sequence runs from empty to the full 64; ids 0 and H - 1 in user_cat, sequence_id, items
    (the query slots) and both sequences; and every third record carries one id in its cat slots, both sequences and the
    query slots at once.  hash_size must be at least 9 (page number 8 is an id of cat slot 10)."""
    assert hash_size >= 9
    rs = np.random.RandomState(seed)
    N, H = n_records, hash_size
    seq = np.zeros((N, 2, 64), np.int32)
    sid = (1 + np.arange(N) % 8).astype(np.int32)
    rs.shuffle(sid)
    ucat = rs.randint(0, H, (N, 10)).astype(np.int32)
    items = rs.randint(0, H, (N, 9)).astype(np.int32)
    for r in range(N):
        L = _HIST[r % len(_HIST)]
        L = rs.randint(2, 64) if L is None else L
        h = rs.randint(0, H, L)[-64:]
        seq[r, 0, 64 - len(h):] = h
        k = _PAGE_LEN[sid[r] - 1]
        if k:
            seq[r, 1, 64 - k:] = rs.randint(0, H, k)
        edge = (0, H - 1)[r % 2]
        ucat[r, r % 10] = edge
        items[r, r % 9] = (0, H - 1)[(r // 2) % 2]
        if len(h):
            seq[r, 0, 64 - 1 - r % len(h)] = edge
        if k:
            seq[r, 1, 64 - 1 - r % k] = H - 1 - edge
        if r % 3 == 0:                                    # one id in a cat slot, both sequences and the query slots
            x = rs.randint(0, H)
            ucat[r, 0] = items[r, 4] = items[r, 8] = x
            seq[r, 0, 63] = seq[r, 1, 63] = x
    sid_id = sid.copy()
    sid_id[5::16] = 0                                     # sequence_id is an id of cat slot 10: its edges too
    sid_id[13::16] = H - 1
    return simtrain.ItemSamples(
        H, user_cat=ucat, user_dense=np.round(np.maximum(0.0, rs.normal(1.0, 1.0, (N, 32))), 3).astype(np.float32),
        sequence_id=sid_id, items=items, feedback=(rs.random_sample((N, 9)) < 0.35).astype(np.uint8),
        item_feature=np.round(rs.normal(0.0, 1.0, (N, 360)), 4).astype(np.float32), seq=seq)


def make_range_samples(n_records, hash_size, lo, hi, seed=0):
    """ItemSamples whose every id, padding included, lies in [lo, hi): both sequences are full, so no slot reads row 0
    unless lo is 0."""
    rs = np.random.RandomState(seed)
    N = n_records
    return simtrain.ItemSamples(
        hash_size, user_cat=rs.randint(lo, hi, (N, 10)).astype(np.int32),
        user_dense=np.round(np.maximum(0.0, rs.normal(1.0, 1.0, (N, 32))), 3).astype(np.float32),
        sequence_id=rs.randint(lo, hi, N).astype(np.int32), items=rs.randint(lo, hi, (N, 9)).astype(np.int32),
        feedback=(rs.random_sample((N, 9)) < 0.35).astype(np.uint8),
        item_feature=np.round(rs.normal(0.0, 1.0, (N, 360)), 4).astype(np.float32),
        seq=rs.randint(lo, hi, (N, 2, 64)).astype(np.int32))


def teacher_labels(samples, config, seed=7, stress=3.0, label_seed=1):
    """Replace the labels by draws from a teacher DIEN's click probabilities (float64 twin, no dropout)."""
    w = synth.make_weights(config, seed=seed, stress=stress, bias_noise=0.2, bounded_scores=True)
    net = simtrain.SimulatorNet(config, simtrain.flatten(w, config), torch.float64)
    idx = np.arange(len(samples))
    p = []
    with torch.no_grad():
        for b in range(0, len(idx), 512):
            cat, dense, seq, _ = samples.features(idx[b:b + 512])
            p.append(net(cat, dense, seq)[0][:, 1].numpy())
    p = np.concatenate(p)
    rs = np.random.RandomState(label_seed)
    samples.feedback = (rs.random_sample(p.shape) < p).astype(np.uint8).reshape(-1, 9)
    return p


def ref_grad(config, flat, samples, idx, keep=None, rate=simtrain.DROPOUT, device="cpu", chunk=512):
    """float64 autograd of the mean loss at flat over samples idx -> (loss, grad f64[np], probs f64[n, 2]).

    Runs on `device` (a CUDA device: torch's float64 kernels, not this project's) in chunks of at most `chunk` samples,
    combined as sum_c (n_c / n) grad_c: the mean loss is linear in the samples, so this is the gradient of the whole batch
    while the saved activations stay those of one chunk."""
    idx = np.asarray(idx, np.int64)
    n = len(idx)
    net = simtrain.SimulatorNet(config, np.asarray(flat, np.float64), torch.float64).to(device)
    loss, probs = 0.0, []
    for b in range(0, n, chunk):
        cat, dense, seq, y = samples.features(idx[b:b + chunk])
        p, _ = net(cat, dense, seq, None if keep is None else keep[b:b + chunk], rate)
        lc = simtrain.keras_bce(p, y) * (len(y) / n)
        lc.backward()
        loss += float(lc.detach())
        probs.append(p.detach().cpu().numpy())
    return loss, net.flat.grad.cpu().numpy(), np.concatenate(probs)


@torch.no_grad()
def ref_probs(config, flat, samples, idx, device="cpu", chunk=2048, keep=None, rate=simtrain.DROPOUT):
    """The float64 twin's click probabilities f64[n, 2], without dropout (r4_simtrain_eval's output) or with keep bits."""
    idx = np.asarray(idx, np.int64)
    net = simtrain.SimulatorNet(config, np.asarray(flat, np.float64), torch.float64).to(device)
    out = []
    for b in range(0, len(idx), chunk):
        cat, dense, seq, _ = samples.features(idx[b:b + chunk])
        out.append(net(cat, dense, seq, None if keep is None else keep[b:b + chunk], rate)[0].cpu().numpy())
    return np.concatenate(out)


def compact(samples, idx):
    """The batch idx over a compacted id space -> (ids, samples', idx').

    ids (int64, ascending) are the distinct ids the batch reads in any slot of either table; samples' holds only the
    batch's records, every id replaced by its position in ids, at hash_size H' = len(ids); idx' are the same samples in it.
    The gradient of an embedding row depends on no other row, so with the rows ids of both tables gathered into tables of
    H' rows, the reference at H' gives the full gradient's rows ids, and every other row of the full gradient is zero."""
    idx = np.asarray(idx, np.int64)
    recs, inv = np.unique(idx // 9, return_inverse=True)
    ids = np.unique(np.concatenate([samples.user_cat[recs].ravel(), samples.sequence_id[recs], samples.items[recs].ravel(),
                                    samples.seq[recs].ravel()]).astype(np.int64))

    def remap(a):
        return np.searchsorted(ids, a).astype(np.int32)
    s = simtrain.ItemSamples(
        len(ids), user_cat=remap(samples.user_cat[recs]), user_dense=samples.user_dense[recs],
        sequence_id=remap(samples.sequence_id[recs]), items=remap(samples.items[recs]), feedback=samples.feedback[recs],
        item_feature=samples.item_feature[recs], seq=remap(samples.seq[recs]))
    return ids, s, (inv * 9 + idx % 9).astype(np.int64)


def compact_weights(weights, ids):
    """The W-table with both embedding tables cut to the rows ids (compact's id space)."""
    return dict(weights, emb_cat=np.asarray(weights["emb_cat"])[ids], emb_seq=np.asarray(weights["emb_seq"])[ids])


def touched_rows(samples, idx):
    """The rows of each embedding table the batch idx reads: emb_cat over the 21 cat slots, emb_seq over both sequences
    and the 10 query slots (cat 11..20)."""
    cat, _, seq, _ = samples.features(idx)
    return {"emb_cat": np.unique(cat), "emb_seq": np.unique(np.concatenate([seq.reshape(-1), cat[:, -10:].reshape(-1)]))}


def keep_bits(seed, counter, n, rate):
    """The kernel's dropout keep bits u8[n, 256] (k_st_gather and drop_u in csrc/r4_simtrain.cuh): unit u of sample s is
    kept when rate <= 0 or u32 = splitmix64(seed ^ splitmix64(splitmix64(counter) + 256 s + u)) >> 40, times 2^-24 in
    float32, is >= rate in float32."""
    s = np.arange(n, dtype=np.uint64)[:, None]
    u = np.arange(256, dtype=np.uint64)[None, :]
    c = policy._splitmix64(np.array([counter], np.uint64))
    r = policy._splitmix64(np.uint64(seed) ^ policy._splitmix64(c + s * np.uint64(256) + u))
    x = (r >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    rate = np.float32(rate)
    if rate <= 0:
        return np.ones((n, 256), np.uint8)
    return (x >= rate).astype(np.uint8)


# ---- the kernel's scratch layout ----
E, NC, ND, U, T, HA, A1, A2, OBS = 128, 21, 432, 128, 64, 256, 64, 16, 256
FEAT = 2 * HA + U + E + NC * E
NSLOT = NC + 2 * T + 10


def scratch_cuts(n):
    """The float count of every plane make_planes (csrc/r4_simtrain.cuh) cuts from the scratch for n samples, in its order.
    This is a copy of its take sequence: a change to that layout has to be made here too."""
    R = n * T
    cuts = [n * NC, n * ND, n * 2 * U, n * U, n * U, n * U, n * FEAT, n * NC * NC, n * E, n * OBS, n * 2, n * 2, n * OBS,
            n * FEAT, n * U, n * U, n * NC * E, n * E, n * 2]
    for _ in range(2):
        cuts += [R * E, R * 2 * E, R * E, R * E, R * E, R * 2 * E, R * E, R * E,
                 R * 4 * E, R * A1, R * A2, R,
                 R * 4 * E, R * 2 * E, R * HA, R * 2 * HA, R * HA, R * HA,
                 R, R * E, R * A2, R * A1, R * 4 * E, R * E, n * E]
    return cuts + [n * NSLOT] * 4


def cub_reserve(n):
    """The radix sort's reserve that follows the planes."""
    return (4 << 20) + 16 * n * NSLOT


def scratch_bytes(n):
    """The bytes a launch over n samples addresses: every plane rounded up to 256 bytes, then the reserve."""
    return sum((4 * k + 255) // 256 * 256 for k in scratch_cuts(n)) + cub_reserve(n)


def num_params(H):
    """The flat parameter count at category_hash_size H (make_layout)."""
    return sum(int(np.prod(s)) for _, s in simtrain.layer_plan({"category_hash_size": H}))


def constant_loss(labels):
    """The loss of the best constant predictor (the label mean)."""
    m = float(np.mean(labels))
    return -(m * np.log(m) + (1 - m) * np.log(1 - m))
