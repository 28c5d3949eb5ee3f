"""CPU, build container only: the oracle env (oracle/env_np.py) against the reference's OWN env classes on RANDOM
scenarios -- env kind, episode length, mask mode, continuous / one-hot actions, raw-state observations, sampling mode,
batch size, and per-step actions (logged, random, repeated, out-of-layer) are drawn from a seed; the reference is rolled
through oracle/ref_harness.py exactly like the committed fixtures were, and everything it exposes per step must equal
what the oracle computes (integers and feature rows bit-exact).  The ten committed fixtures pin ten hand-picked corners;
this sweeps the product of the flags.  What the reference computed is stored under tests/golden/reference/
(golden_util.reference_result; tests/golden/make_reference_golden.py rewrites it), so these run on any machine."""
import os
import sys

import numpy as np
import pytest

from golden_util import GOLDEN_DIR, reference_result
from oracle import ref_harness
from oracle.dnn_np import DnnOracle
from oracle.env_np import OracleEnv
from rl4rs_b200 import synth
from rl4rs_b200.utils.datautil import FeatureUtil

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))

ITEM_FILE = os.path.join(GOLDEN_DIR, "item_info.csv")     # the reference's dataset/item_info.csv (data fixture)


def draw_scenario(seed):
    rs = np.random.RandomState(1000 + seed)
    seq = bool(rs.rand() < 0.5)
    B = int(rs.randint(2, 7))
    cfg = {"epoch": 1, "maxlen": 64, "action_size": 284, "class_num": 2, "dense_feature_num": 432,
           "category_feature_num": 21, "category_hash_size": 5000, "seq_num": 2, "emb_size": 128, "page_items": 9,
           "hidden_units": 128, "action_emb_size": 32, "batch_size": B, "algo": "dnn",     # the cheap network: the env half is under test
           "max_steps": int(rs.choice([9, 18, 27, 36])) if seq else 9}
    mode = rs.choice(["plain", "rllib", "d3rl", "both"])
    if mode in ("rllib", "both"):
        cfg["support_rllib_mask"] = True
    if mode in ("d3rl", "both"):
        cfg["support_d3rl_mask"] = True
    if rs.rand() < 0.35:
        cfg["support_conti_env"] = True
        if rs.rand() < 0.3:
            cfg["support_onehot_action"] = True
    if rs.rand() < 0.25:
        cfg["rawstate_as_obs"] = True
    if rs.rand() < 0.4:
        cfg["simulator_info_fetch"] = True
    train_mode = bool(rs.rand() < 0.4)
    cfg["is_eval"] = not train_mode
    cfg["cache_size"] = int(rs.randint(B, 3 * B + 1)) if train_mode else B
    n_rows = int(rs.randint(cfg["cache_size"], 3 * cfg["cache_size"] + 2))     # small logs wrap around (base.py:85-88)
    episodes = int(rs.randint(1, 4))
    return cfg, seq, n_rows, episodes, int(rs.randint(1 << 30)), train_mode


def action_source(cfg, seed):
    rs = np.random.RandomState(seed)
    B = cfg["batch_size"]
    emb = cfg["action_size"] if cfg.get("support_onehot_action") else 32

    def pick(env, ep, t, off):
        if cfg.get("support_conti_env"):
            a = rs.uniform(-1, 1, (B, emb))
            a[rs.rand(B) < 0.15] = 0.0                              # all-zero rows: every score ties
            keep = rs.rand(B) < 0.3
            a[keep] = np.asarray(off, dtype=np.float64)[keep]       # the logged item's own embedding
            return a
        off = np.asarray(off)
        r = rs.rand(B)
        rand = rs.randint(0, cfg["action_size"], B)                 # often outside the layer, or a repeat
        prev = env.samples.prev_actions[:, max(t - 1, 0)]
        return np.where(r < 0.6, off, np.where(r < 0.85, rand, prev)).astype(np.int64)
    return pick


# The configuration edges r4_create admits, as a fixed list rather than a draw, so every value is covered by construction:
# action_size 149 (layer 2 holds item 148 alone), 150, 160, 255-257, 288 and 511 / 512 (the last and the 16th mask word,
# full or partial), Slate lengths 3-11 (post-padded and post-truncated feature rows, layer 3 at steps 9 and 10), SeqSlate
# 9 to 81 (more than 64 previous items, Q9 walking pages 4-8), and category_hash_size == action_size.  The log carries
# ceil(T / 9) pages, so the reference finds a logged slot at every step.  A Slate slate of 11 always violates (steps 9 and
# 10 may only hold item 0, and twice in a row is a repeat), so there the reward pass is held to the record by click_p.
SHAPE_SCENARIOS = [
    dict(A=149, seq=False, T=10, B=3, mode="rllib", conti=True),
    dict(A=150, seq=False, T=3, B=2, mode="plain", H=150),
    dict(A=160, seq=False, T=4, B=5, mode="d3rl", info=True),
    dict(A=255, seq=False, T=5, B=4, mode="rllib", raw=True, train=True),
    dict(A=256, seq=False, T=8, B=3, mode="both", conti=True, info=True),
    dict(A=257, seq=False, T=11, B=4, mode="rllib", info=True),
    dict(A=288, seq=False, T=11, B=2, mode="d3rl", conti=True),
    dict(A=511, seq=False, T=10, B=5, mode="plain", info=True, train=True),
    dict(A=512, seq=False, T=8, B=3, mode="rllib", conti=True, onehot=True),
    dict(A=256, seq=False, T=3, B=2, mode="rllib", raw=True, info=True, H=256),
    dict(A=288, seq=True, T=9, B=2, mode="rllib", conti=True, info=True),
    dict(A=511, seq=True, T=18, B=5, mode="d3rl", info=True),
    dict(A=160, seq=True, T=45, B=3, mode="plain", raw=True),
    dict(A=512, seq=True, T=45, B=3, mode="rllib", conti=True, onehot=True),
    dict(A=512, seq=True, T=81, B=2, mode="plain", info=True, train=True),
    dict(A=149, seq=True, T=81, B=4, mode="both", conti=True),
]


def shape_scenario(i):
    s = dict({"H": 5000, "conti": False, "onehot": False, "raw": False, "info": False, "train": False}, **SHAPE_SCENARIOS[i])
    B = s["B"]
    cfg = {"epoch": 1, "maxlen": 64, "action_size": s["A"], "class_num": 2, "dense_feature_num": 432,
           "category_feature_num": 21, "category_hash_size": s["H"], "seq_num": 2, "emb_size": 128, "page_items": 9,
           "hidden_units": 128, "action_emb_size": 32, "batch_size": B, "algo": "dnn", "max_steps": s["T"],
           "is_eval": not s["train"], "cache_size": 2 * B if s["train"] else B}
    for key, on in (("support_rllib_mask", s["mode"] in ("rllib", "both")), ("support_d3rl_mask", s["mode"] in ("d3rl", "both")),
                    ("support_conti_env", s["conti"]), ("support_onehot_action", s["onehot"]),
                    ("rawstate_as_obs", s["raw"]), ("simulator_info_fetch", s["info"])):
        if on:
            cfg[key] = True
    episodes = 2 if s["T"] <= 18 else 1
    return cfg, s["seq"], 2 * cfg["cache_size"] + 1, episodes, 3000 + i, (300 + i if s["train"] else None)


def scenario(kind, i):
    """Inputs of random_scenario_NN / shape_scenario_NN and what the reference's own env computed on them:
    (cfg, seq, catalog, records, dnn weights, episodes, numpy seed of the sampler or None, record)."""
    import make_golden
    if kind == "random":
        cfg, seq, n_rows, episodes, aseed, train_mode = draw_scenario(i)
        cat = synth.make_catalog()
        log = synth.make_log(n_rows, pages=4 if seq else 1, catalog=cat, hash_size=5000, corrupt_frac=0.25, keep_hist=True,
                             seed=synth.LOG_SEED + i)
        np_seed = 77 + i if train_mode else None
        w = synth.make_dnn_weights(cfg, stress=2.0, bias_noise=0.2)
    else:
        cfg, seq, n_rows, episodes, aseed, np_seed = shape_scenario(i)
        cat = synth.make_catalog(n_items=cfg["action_size"] - 1)
        log = synth.make_log(n_rows, pages=-(-cfg["max_steps"] // 9), catalog=cat, hash_size=cfg["category_hash_size"],
                             corrupt_frac=0.25, keep_hist=True, seed=synth.LOG_SEED + 100 + i)
        w = synth.make_dnn_weights(cfg, stress=1.0, bias_noise=0.2)     # the env's edges are under test, not the network's
    records = synth.render_records(log, cat)
    rec = reference_result("%s_scenario_%02d" % (kind, i), lambda: make_golden.run_reference(
        dict(cfg), records, cat.to_text(), w, seq, action_source(cfg, aseed), n_episodes=episodes, seed=np_seed,
        net=DnnOracle(w, np.float32)))
    return cfg, seq, cat, records, w, episodes, np_seed, rec


def check_scenario(kind, i, fmt):
    """The oracle env, then the product's own env classes (gym layer, sampler, obs / reward formatting) over the engine
    stand-in, against the stored reference record of one scenario."""
    from test_oracle_golden import check_oracle_against_record
    cfg, seq, cat, records, w, episodes, np_seed, rec = scenario(kind, i)
    if np_seed is not None:
        np.random.seed(np_seed)
    env = OracleEnv(dict(cfg), FeatureUtil.parse_log(records, 64), cat, DnnOracle(w, np.float32), seq=seq)
    check_oracle_against_record(env, cfg, rec, episodes, "%s scenario %d" % (kind, i))
    import rl4rs_b200.engine as engine_mod
    from oracle_engine import OracleEngine
    from test_host_layer_cpu import make_env, replay_through_host_layer
    real = engine_mod.Engine
    engine_mod.Engine = OracleEngine
    try:
        if np_seed is not None:
            np.random.seed(np_seed)
        host_env = make_env(dict(cfg), seq, cat, FeatureUtil.parse_log(records, 64), w, output_format=fmt)
        replay_through_host_layer(host_env, cfg, rec, episodes, "%s scenario %d (host layer, %s)" % (kind, i, fmt), fmt)
    finally:
        engine_mod.Engine = real


@pytest.mark.parametrize("seed", range(32))
def test_oracle_env_equals_the_reference_env_on_a_random_scenario(seed):
    check_scenario("random", seed, ("list", "numpy", "torch")[seed % 3])


@pytest.mark.parametrize("idx", range(len(SHAPE_SCENARIOS)))
def test_oracle_env_equals_the_reference_env_on_a_shape_scenario(idx):
    check_scenario("shape", idx, ("list", "numpy", "torch")[idx % 3])


@pytest.mark.parametrize("seed", range(8))
def test_ingest_equals_the_reference_preprocessing_on_random_sessions(seed, tmp_path):
    """n3: rl4rs_b200/utils/ingest.py against the reference's own script/data_preprocess.py (run as its own CLI, like
    tests/golden/make_ingest_golden.py does) on random session tables: `data_augment` pads sessions of 1-4 pages to 4 with
    the GLOBAL numpy RNG, `slate2trajectory` joins 4-page sessions and drops the last one."""
    import runpy
    from rl4rs_b200.utils import ingest

    def run_stage(stage, lines):
        ref_harness.install_stubs()
        script = os.path.join(ref_harness.REFERENCE_ROOT, "script", "data_preprocess.py")
        src, dst = str(tmp_path / "in.csv"), str(tmp_path / ("out_%s.csv" % stage))
        open(src, "w").write("\n".join(lines))
        argv, sys.argv = sys.argv, [script, src, dst, stage]
        try:
            runpy.run_path(script, run_name="__main__")
        finally:
            sys.argv = argv
        return [x for x in open(dst).read().split("\n") if x]

    rs = np.random.RandomState(500 + seed)
    n_sess = int(rs.randint(3, 10))
    cat = synth.make_catalog()
    recs = synth.render_records(synth.make_log(4 * n_sess, pages=1, catalog=cat, keep_hist=True, seed=900 + seed), cat)
    header = "timestamp@session_id@sequence_id@exposed_items@user_feedback@user_seqfeature@user_protrait@item_feature@behavior_policy_id"
    ragged = [header]
    for s in range(n_sess):
        base = recs[4 * s].split("@")
        for p in range(int(rs.randint(1, 5))):               # 1..4 pages of this session survive
            f = recs[4 * s + p].split("@")
            ragged.append("@".join([str(1000 * s + p), base[1], str(p + 1), f[3], f[4], base[5], base[6], f[7], base[8]]))
    ragged.append("")

    def reference():
        np.random.seed(40 + seed)
        aug = run_stage("data_augment", ragged)
        full_ = [header] + aug[1:] + [""] if aug[0] == header else [header] + aug + [""]
        return {"aug": aug, "traj": run_stage("slate2trajectory", full_)}
    want = reference_result("ingest_%d" % seed, reference)
    want_aug, want_traj = want["aug"], want["traj"]
    np.random.seed(40 + seed)
    got_aug = ingest.data_augment(ragged)
    assert got_aug == want_aug
    full = [header] + want_aug[1:] + [""] if want_aug[0] == header else [header] + want_aug + [""]
    assert ingest.slate2trajectory(full) == want_traj
    assert 1 <= len(want_traj) < n_sess                      # the script drops the last session (and any it merges)


def test_trainer_defaults_are_the_reference_scripts_hyper_parameters():
    """a23: the RLlib config dicts of script/modelfree_train.py (PPO :179-217, A2C :248-268, common :390-415), read out of
    the script's own source with `ast`, against the defaults rl4rs_b200/trainer.py trains with."""
    import ast
    from rl4rs_b200 import trainer

    def literal(node):
        """A dict literal with non-literal values (config[...] expressions) left out."""
        out = {}
        for k, v in zip(node.keys, node.values):
            if k is None:
                continue
            try:
                out[ast.literal_eval(k)] = ast.literal_eval(v)
            except Exception:
                pass
        return out

    def reference():
        src = open(os.path.join(ref_harness.REFERENCE_ROOT, "script", "modelfree_train.py")).read()
        tree = ast.parse(src)
        branches = {}
        for node in ast.walk(tree):
            if isinstance(node, ast.If) and isinstance(node.test, ast.Compare) and isinstance(node.test.left, ast.Constant) \
                    and node.test.left.value in ("PPO", "A2C"):
                first = node.body[0]
                assert isinstance(first, ast.Assign) and first.targets[0].id == "cfg"
                branches[node.test.left.value] = literal(first.value)
        common = [literal(n) for n in ast.walk(tree) if isinstance(n, ast.Dict)]
        return {"branches": branches, "common": [d for d in common if d.get("batch_mode") == "complete_episodes"],
                "softq": '"type": "SoftQ"' in src}
    stored = reference_result("modelfree_train_configs", reference)
    branches, common = stored["branches"], stored["common"]
    assert set(branches) == {"PPO", "A2C"}
    for algo, ours in (("PPO", trainer.PPO_DEFAULTS), ("A2C", trainer.A2C_DEFAULTS)):
        ref = branches[algo]
        shared = sorted(set(ref) & set(ours))
        assert len(shared) >= 5, shared
        for k in shared:
            assert ours[k] == ref[k], (algo, k, ours[k], ref[k])
    assert trainer.PPO_DEFAULTS["grad_clip"] is None and "grad_clip" not in branches["PPO"]       # commented out there
    # the dict every algorithm is merged into: gamma 1, SoftQ exploration, complete episodes
    assert len(common) == 1 and common[0]["gamma"] == 1 and common[0]["explore"] is True
    assert trainer.PPO_DEFAULTS["gamma"] == trainer.A2C_DEFAULTS["gamma"] == 1.0
    assert stored["softq"]


def test_static_helpers_on_the_real_catalog_and_random_knn_queries():
    """slate.py:28-65,180-191: the item table, action embeddings, location mask and special items read from the
    reference's own dataset/item_info.csv, and the two nearest-neighbour statics on random queries (incl. ties and
    fully masked rows), reference class against mirror class."""
    from rl4rs_b200.env.slate import SlateState

    def queries(emb):
        rs = np.random.RandomState(4)
        for trial in range(20):
            q = rs.uniform(-1, 1, (16, 32))
            q[0] = 0.0                                        # every score ties at 0: lowest index wins
            q[1] = emb[1 + trial]                             # an item's own embedding
            mask = (rs.rand(16, 284) < 0.3).astype(np.int64)
            mask[2] = 0                                       # nothing allowed: all scores -2**31, index 0
            yield q, mask

    def reference():
        ref_slate = ref_harness.install_stubs()[1]
        item_file = os.path.join(ref_harness.REFERENCE_ROOT, "dataset", "item_info.csv")
        info, emb = ref_slate.SlateState.get_iteminfo_from_file(item_file, 284)
        loc, sp = ref_slate.SlateState.get_mask_from_file(item_file, 284)
        keys = sorted(info, key=int)
        nn = [(ref_slate.SlateState.get_nearest_neighbor(q, emb), ref_slate.SlateState.get_nearest_neighbor_with_mask(q, emb, m))
              for q, m in queries(emb)]
        return {"keys": [int(k) for k in keys], "price": np.array([info[k]["price"] for k in keys], np.float64),
                "location": np.array([info[k]["location"] for k in keys], np.int64),
                "item_vec": np.array([np.asarray(info[k]["item_vec"], float) for k in keys]), "emb": np.asarray(emb),
                "loc": np.asarray(loc), "special": [int(x) for x in sp],
                "nn": np.array([a for a, _ in nn]), "nn_mask": np.array([b for _, b in nn])}
    ref = reference_result("static_helpers", reference)
    info_o, emb_o = SlateState.get_iteminfo_from_file(ITEM_FILE, 284)
    np.testing.assert_array_equal(emb_o, ref["emb"])
    assert sorted(int(k) for k in info_o) == ref["keys"]
    for i, k in enumerate(sorted(info_o, key=int)):
        assert info_o[k]["price"] == ref["price"][i] and info_o[k]["location"] == ref["location"][i], k
        np.testing.assert_array_equal(np.asarray(info_o[k]["item_vec"], float), ref["item_vec"][i])
    loc_o, sp_o = SlateState.get_mask_from_file(ITEM_FILE, 284)
    np.testing.assert_array_equal(loc_o, ref["loc"])
    assert [int(x) for x in sp_o] == ref["special"] and len(ref["special"]) > 0
    for trial, (q, mask) in enumerate(queries(emb_o)):
        np.testing.assert_array_equal(SlateState.get_nearest_neighbor(q, emb_o), ref["nn"][trial])
        np.testing.assert_array_equal(SlateState.get_nearest_neighbor_with_mask(q, emb_o, mask), ref["nn_mask"][trial])


def test_feature_extraction_mirror_on_random_ragged_rows():
    """datautil.py:34-69: FeatureUtil.feature_extraction, reference method against the host mirror, on raw state rows
    with empty / short / over-long sequences, short and over-long dense and category lists."""
    from rl4rs_b200.utils.datautil import FeatureUtil
    cfg = {"maxlen": 64, "batch_size": 5, "class_num": 2, "dense_feature_num": 432, "category_feature_num": 21,
           "category_hash_size": 100000, "seq_num": 2}

    def trials():
        rs = np.random.RandomState(8)
        for trial in range(12):
            rows = []
            for i in range(5):
                seqs = [list(rs.randint(1, 284, rs.choice([0, 1, 7, 64, 65, 130]))) for _ in range(2)]
                dense = list(rs.normal(0, 1, rs.choice([32, 72, 432, 440])).astype(np.float64))
                cat = list(rs.randint(0, 100000, rs.choice([10, 12, 21, 25])).astype(np.float64))       # floats in the reference too
                rows.append([0, seqs, dense, cat, [0] * 9, int(rs.randint(2))])
            yield rows

    def reference():
        ref = ref_harness.install_stubs()[3].FeatureUtil(cfg)
        out = {}
        for trial, rows in enumerate(trials()):
            (s2, d2, c2, l2), y2 = ref.feature_extraction(rows)
            out.update({"s%d" % trial: s2, "d%d" % trial: d2, "c%d" % trial: c2, "l%d" % trial: np.asarray(l2),
                        "y%d" % trial: np.asarray(y2)})
        return out
    ref = reference_result("feature_extraction", reference)
    ours = FeatureUtil(cfg)
    for trial, rows in enumerate(trials()):
        (s1, d1, c1, l1), y1 = ours.feature_extraction(rows)
        np.testing.assert_array_equal(s1, ref["s%d" % trial]); np.testing.assert_array_equal(d1, ref["d%d" % trial])
        np.testing.assert_array_equal(c1, ref["c%d" % trial]); np.testing.assert_array_equal(l1, ref["l%d" % trial])
        np.testing.assert_array_equal(np.asarray(y1), ref["y%d" % trial])
        assert d1.dtype == ref["d%d" % trial].dtype and c1.dtype == ref["c%d" % trial].dtype and s1.shape == (5, 2, 64)
