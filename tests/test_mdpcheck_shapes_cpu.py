"""CPU companion of test_gpu_mdpcheck_shapes.py: what its references and planted inputs must be for the GPU checks to mean
anything, shown without a device.

  rejections      every r4_s2s_* entry point refuses one step past each edge on the host (R4_ERR_ARG, no launch), so
                  the GPU module can repeat the calls without ever launching a refused shape
  clipped loss    the planted weights put every loss-position probability at least 100 times from its clip edge, both
                  clip branches are taken, and a loss that drops the clip or lets the gradient through the clipped
                  entries misses the float64 reference by at least 10 times the GPU bars
  planted ties    the twin gives the tied tokens bit-identical probabilities and the zero group exactly 0
  replay          the NumPy replay of the selection rule, fed by the twin's probabilities, equals decoder._search_twin
                  exactly, at ties straddling the beam and with fewer candidates than beam
"""
import ctypes as C

import numpy as np

import mdpcheck_ref64 as ref
from rl4rs_b200 import _capi
from rl4rs_b200.mdpchecker import decoder as dc

LOSS_BAR, GRAD_BAR = 1e-5, 1e-4          # the GPU module's bars


def test_rejections_on_the_host():
    lib = _capi.load_library()
    buf = (C.c_char * 64)()
    n0 = lib.r4_s2s_launch_count()
    got = ref.abi_rejections(lib, C.cast(buf, C.c_void_p))
    assert [x for x in got if x[1] != -1] == []
    assert lib.r4_s2s_launch_count() == n0
    assert len(got) > 150


def test_clip_planting_and_faulty_losses_miss():
    m, enc, dec, y = ref.clip_case()
    loss, g, probs = ref.grad64(m.flat, m.cfg, enc, dec, y)
    assert ref.clip_margin(probs, dec) >= 100.0
    clipped_t, clipped_top = ref.clip_counts(probs, dec, y)
    pos = int((dec != 0).sum())
    assert clipped_t >= 0.3 * pos and clipped_top >= 0.15 * pos, (clipped_t, clipped_top, pos)
    for lf in (ref.loss_noclip, ref.loss_passthrough):
        l2, g2, _ = ref.grad64(m.flat, m.cfg, enc, dec, y, loss_fn=lf)
        worst, _, _ = ref.grad_errors(g2, g, m.cfg)
        miss = max(abs(l2 - loss) / max(1.0, abs(loss)) / LOSS_BAR, worst / GRAD_BAR)
        print("%s: misses the reference by %.0f times the GPU bar" % (lf.__name__, miss))
        assert miss >= 10.0, lf.__name__


TIES = dict(groups=[(3.0, list(range(10, 16))), (2.0, list(range(40, 60)))], zero=list(range(100, 200)))


def test_twin_makes_the_planted_ties():
    m = ref.tie_model(200, 300, 32, 1, 32, 4, **TIES)
    rs = np.random.RandomState(0)
    enc = rs.randint(3, 200, (6, 10))
    enc[:, 0] = 1
    dec = np.concatenate([np.ones((6, 1), int), rs.randint(3, 300, (6, 4))], 1)
    p = m.predict([enc, dec])
    for _, toks in TIES["groups"]:
        assert (p[..., toks] == p[..., toks[:1]]).all()
    assert (p[..., TIES["zero"]] == 0).all() and (np.delete(p, TIES["zero"], -1) > 0).all()


def test_replay_equals_the_twin_search():
    m = ref.tie_model(200, 300, 32, 1, 32, 4, **TIES)
    rs = np.random.RandomState(1)
    enc = rs.randint(3, 200, (6, 10))
    enc[:, 0] = 1
    p = m.predict([enc, np.ones((6, 1), int)])[:, -1]
    # beam 12 cuts the 20-token tie group; 5 candidates < beam 8 leave zero products to the index rule
    for beam, cand, T in ((12, 0, 5), (8, 5, 5), (16, 30, 4), (1, 0, 3)):
        path, score = dc.beam_search(m, enc, beam, T, use_candidates=cand > 0, candidates_size=cand)
        rp, rsc, mask = ref.replay_first(p, beam, cand)
        for t in range(1, T):
            q = m.predict([np.repeat(enc, beam, 0), rp.reshape(-1, t + 1)])[:, -1]
            if cand and cand < beam:       # each prefix's top-beam list ends in zero keys
                keys = q.astype(np.float64) * np.repeat(mask, beam, axis=0)
                assert (ref.top_rule(keys, beam)[0][:, cand:] == 0).all()
            rp, rsc = ref.replay_step(q, rp, rsc, mask)
        assert np.array_equal(rp, path) and np.array_equal(rsc, score), (beam, cand)
