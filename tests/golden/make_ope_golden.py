"""Write tests/golden/reference/ope_{metrics,behavior,flow}.npz from the reference's own code:

  ope_metrics   rl4rs/utils/offline_policy_metrics.py (NumPy / SciPy only) over a grid: B in {2, 7, 2048}, T in
                {1, 9, 36}; plain ratios, ratios on both edges of the [0.1, 10] clip, negative (log-)probabilities, and
                B = 2 cases whose int(n_e) - 1 is 0.
  ope_behavior  rl4rs/policy/behavior_model.py with keras.models.load_model stubbed by oracle/dnn_np.py (D = 50, C = 284)
                over synthetic Slate (9 items) and SeqSlate (36 items) records: every layer 1..12, pages 0..3, the edge
                actions 0, 1, 39, 40, 147, 148, 283.
  ope_flow      script/offline_evaluation.py:ope_eval with policy_model, behavior_model and the env replaced by recorders
                replaying fixed arrays: what it computes and prints.

    python tests/golden/make_ope_golden.py      (needs the reference tree; RL4RS_REFERENCE_ROOT)
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_harness  # noqa: E402
from oracle.dnn_np import DnnOracle  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference")
H, C = 1000, 284
EDGE_ACTIONS = (0, 1, 39, 40, 147, 148, 283)


def _exec(rel, g):
    src = os.path.join(ref_harness.REFERENCE_ROOT, rel)
    exec(compile(open(src).read(), os.path.basename(src), "exec"), g)
    return g


def metric_cases():
    """[(name, B, T, pol [B, T] f32, beh f32, off_rewards [B, T] f64, rewards_hat f64, q f32, episode_reward f64)]."""
    rs = np.random.RandomState(7)
    out = []
    for B in (2, 7, 2048):
        for T in (1, 9, 36):
            for kind in ("plain", "edges", "logprob"):
                beh = rs.uniform(0.005, 0.02, (B, T)).astype(np.float32)
                if kind == "plain":
                    pol = rs.uniform(0.005, 0.02, (B, T)).astype(np.float32)
                elif kind == "edges":
                    f = rs.choice(np.array([0.1, 10.0, 0.0999, 0.1001, 9.999, 10.001, 1.0]), (B, T))
                    pol = (beh * f).astype(np.float32)
                else:
                    pol = np.log(rs.uniform(0.2, 0.99, (B, T))).astype(np.float32)
                off = rs.uniform(0, 5, (B, T))
                hat = rs.uniform(0, 5, (B, T))
                q = rs.uniform(-1, 8, (B, T)).astype(np.float32)
                out.append(("%s_%d_%d" % (kind, B, T), pol, beh, off, hat, q, hat.sum(1)))
    # int(n_e) - 1 == 0: two episodes whose clipped ratios are 10 and 0.1 apart
    pol = np.array([[0.5], [0.001]], np.float32)
    beh = np.array([[0.01], [0.01]], np.float32)
    out.append(("ne1_2_1", pol, beh, np.array([[1.0], [2.0]]), np.array([[0.5], [1.5]]), np.array([[1.0], [2.0]], np.float32),
                np.array([0.5, 1.5])))
    return out


def metric_inputs():
    """[(name, inputs)] for ope_metrics: metric_cases with the episode products -- the step products where they stay
    finite, else products with the same kind of ratios.  Seeded, so the tests rebuild them."""
    rs = np.random.RandomState(8)
    out = []
    for name, pol, beh, off, hat, q, ep in metric_cases():
        bpm = np.multiply.reduce(beh * 100, axis=1)
        if name.startswith("plain") or name.startswith("ne1"):
            apm = np.multiply.reduce(pol * 100, axis=1)
        elif name.startswith("edges"):
            apm = (bpm * rs.choice(np.array([0.1, 10.0, 0.0999, 0.1001, 9.999, 10.001, 1.0]), len(bpm))).astype(np.float32)
        else:
            apm = -rs.uniform(0.5, 50, len(bpm)).astype(np.float32)
        out.append((name, dict(pol=pol, beh=beh, off=off, hat=hat, q=q, ep=ep, apm=apm, bpm=bpm, offs=np.sum(off, axis=1))))
    return out


def metric_calls(g, x):
    """The estimator calls of ope_metrics, over the functions of namespace g."""
    return {"IPS": lambda: g["eval_IPS"](x["offs"], x["apm"], x["bpm"]),
            "CIPS": lambda: g["eval_CIPS"](x["offs"], x["apm"], x["bpm"]),
            "SNIPS": lambda: g["eval_SNIPS"](x["offs"], x["apm"], x["bpm"]),
            "DR": lambda: g["eval_doubly_robust"](x["ep"], np.average(x["q"], 1), x["offs"], x["apm"], x["bpm"]),
            "WIPS": lambda: g["eval_WIPS"](x["off"], x["pol"], x["beh"]),
            "SeqDR": lambda: g["eval_seq_doubly_robust"](x["hat"], x["q"], x["off"], x["pol"], x["beh"])}


def make_metrics():
    g = _exec("rl4rs/utils/offline_policy_metrics.py", {"__name__": "ref_ope"})
    out = {}
    for name, x in metric_inputs():
        for k, f in metric_calls(g, x).items():
            try:
                out[name + "/" + k] = np.asarray(f(), np.float64)
            except ValueError as exc:           # int(n_e) of a NaN n_e: the reference raises
                out[name + "/" + k + "_raises"] = np.array(str(exc))
        if len(x["pol"]) <= 7:
            out[name + "/seqw"] = g["_calc_sequential_weigths"](x["pol"], x["beh"], a_min=0.1, a_max=10)
        r, n_e, cv = g["_calc_sample_weigths"](x["apm"], x["bpm"], a_min=0.1, a_max=10)
        out[name + "/ne_cv"] = np.array([n_e, cv], np.float64)
    np.savez_compressed(os.path.join(OUT, "ope_metrics.npz"), **out)


def dnn_weights(seed=3):
    rs = np.random.RandomState(seed)
    shapes = {"emb_cat": (H, 128), "dense_w1": (50, 128), "dense_b1": (128,), "dense_w2": (128, 128), "dense_b2": (128,),
              "fc_w": (256, 256), "fc_b": (256,), "obs_w": (256, 256), "obs_b": (256,), "rew_w": (256, C), "rew_b": (C,)}
    return {k: (rs.standard_normal(s) * (0.3 if k == "emb_cat" else 1.0 / np.sqrt(s[0]) if len(s) == 2 else 0.1))
            .astype(np.float32) for k, s in shapes.items()}


def records(n, pages, seed):
    """Synthetic log records in the reference's '@' format (datautil.record_split), item_feature 40 per item."""
    rs = np.random.RandomState(seed)
    out = []
    for i in range(n):
        items = rs.randint(1, C, 9 * pages)
        fb = rs.randint(0, 2, 9 * pages)
        hist = rs.randint(1, C, rs.randint(1, 20))
        portrait = list(rs.randint(0, H - 1, 10).astype(float)) + list(rs.standard_normal(32).round(4))
        feat = ";".join(",".join("%.5f" % x for x in rs.standard_normal(40)) for _ in range(9 * pages))
        out.append("@".join([str(i), str(1000 + i), str(rs.randint(0, 40)), ",".join(map(str, items)), ",".join(map(str, fb)),
                             ",".join(map(str, hist)), ",".join("%g" % x for x in portrait), feat, "0"]))
    return out


class _Keras(object):
    def __init__(self, w):
        self.m = DnnOracle(w, np.float32)

    def predict(self, x):
        return self.m.forward(x[0], x[1], x[2])[1]


def make_behavior():
    ref_harness.install_stubs()
    w = dnn_weights()
    tf = sys.modules["tensorflow"]

    class _Sess(object):
        def as_default(self):
            return types.SimpleNamespace(__enter__=lambda *a: None, __exit__=lambda *a: False)

    class _Ctx(object):
        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

    tf.Session = lambda: types.SimpleNamespace(as_default=lambda: _Ctx())
    tf.keras.models = types.SimpleNamespace(load_model=lambda f: _Keras(w))
    from rl4rs.utils.datautil import FeatureUtil
    g = {"__name__": "ref_behavior"}
    src = open(os.path.join(ref_harness.REFERENCE_ROOT, "rl4rs", "policy", "behavior_model.py")).read()
    src = src.replace("from tensorflow import keras", "keras = tf.keras")
    src = src.replace("from rl4rs.utils.datautil import FeatureUtil", "")
    g["FeatureUtil"] = FeatureUtil
    exec(compile(src, "behavior_model.py", "exec"), g)
    out = {}                      # the weights are dnn_weights(), rebuilt by the tests
    rs = np.random.RandomState(5)
    for kind, pages, B in (("slate", 1, 7), ("seqslate", 4, 7)):
        recs = records(B, pages, 11 + pages)
        out[kind + "/records"] = np.array(recs)
        bm = g["behavior_model"]({"batch_size": B, "page_items": 9, "maxlen": 64, "class_num": 2, "category_hash_size": H, "seq_num": 2}, "logged_policy.h5")
        for page in range(pages):
            for layer in range(1, 13):
                act = np.array(list(EDGE_ACTIONS) * 2)[:B] if layer % 2 else rs.randint(0, C, B)
                out["%s/%d/%d/action" % (kind, page, layer)] = act
                out["%s/%d/%d/probs" % (kind, page, layer)] = np.asarray(bm.action_probs(recs, act, layer, page=page))
            out["%s/%d/edges" % (kind, page)] = np.stack([np.asarray(bm.action_probs(recs, np.full(B, a), layer, page=page))
                                                          for layer in (1, 2, 3) for a in EDGE_ACTIONS])
    np.savez_compressed(os.path.join(OUT, "ope_behavior.npz"), **out)


def flow_arrays(B=6, T=9, A=20, epochs=2, seed=9):
    rs = np.random.RandomState(seed)
    return {"probs": rs.dirichlet(np.ones(A), (epochs, T, B)).astype(np.float32),
            "actions": rs.randint(0, A, (epochs, T, B)), "off_action": rs.randint(0, A, (epochs, T, B)),
            "q": rs.uniform(0, 5, (epochs, T, B)).astype(np.float32), "beh": rs.uniform(0.02, 0.2, (epochs, T, B)).astype(np.float32),
            "reward": rs.uniform(0, 3, (epochs, T, B)), "off_reward": rs.uniform(0, 3, (epochs, T, B))}


class FlowEnv(object):
    """Replays offline actions, rewards and the offline rewards of fixed arrays; records the actions it is given."""

    def __init__(self, arr):
        self.a, self.e, self.t, self.taken = arr, -1, 0, []
        self.samples = types.SimpleNamespace(records=None)

    def reset(self):
        self.e, self.t = self.e + 1, 0
        self.samples = types.SimpleNamespace(records=["episode %d" % self.e])
        return np.full((self.a["probs"].shape[2], 3), float(self.e))

    @property
    def offline_action(self):
        return self.a["off_action"][self.e, self.t]

    @property
    def offline_reward(self):
        return self.a["off_reward"][self.e, self.t - 1]

    def step(self, action):
        self.taken.append(np.asarray(action))
        r = self.a["reward"][self.e, self.t]
        self.t += 1
        return np.full((len(r), 3), float(self.t)), r, [self.t == self.a["probs"].shape[1]] * len(r), {}


class FlowPolicy(object):
    """policy_model's surface over the arrays: predict_with_mask, action_probs [B, A], predict_q [B]."""

    def __init__(self, env):
        self.env = env

    def predict_with_mask(self, obs):
        return self.env.a["actions"][self.env.e, self.env.t]

    def action_probs(self, obs):
        return self.env.a["probs"][self.env.e, self.env.t]

    def predict_q(self, obs, action):
        assert np.array_equal(action, self.env.a["actions"][self.env.e, self.env.t])
        return self.env.a["q"][self.env.e, self.env.t]


class FlowBehavior(object):
    def __init__(self, env):
        self.env, self.calls = env, []

    def action_probs(self, records, action, layer, page=0):
        self.calls.append((self.env.e, self.env.t, layer, page))
        assert np.array_equal(action, self.env.a["off_action"][self.env.e, self.env.t])
        return self.env.a["beh"][self.env.e, self.env.t]


def make_flow():
    arr = flow_arrays()
    env = FlowEnv(arr)
    printed = []
    pm = types.ModuleType("rl4rs.policy.policy_model")
    pm.policy_model = lambda algo, config: FlowPolicy(env)
    bm = types.ModuleType("rl4rs.policy.behavior_model")
    bm.behavior_model = FlowBehavior
    saved = {k: sys.modules.get(k) for k in ("rl4rs.policy.policy_model", "rl4rs.policy.behavior_model")}
    sys.modules.update({"rl4rs.policy.policy_model": pm, "rl4rs.policy.behavior_model": bm, "gym": types.ModuleType("gym")})
    if ref_harness.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, ref_harness.REFERENCE_ROOT)
    g = _exec("script/offline_evaluation.py", {"__name__": "ref_flow", "print": lambda *a, **k: printed.append(a)})
    E, T, B = arr["probs"].shape[:3]
    config = {"epoch": E, "batch_size": B, "max_steps": T, "page_items": 4}
    sm = FlowBehavior(env)
    g["ope_eval"](config, env, None, sample_model=sm)
    for k, v in saved.items():
        if v is not None:
            sys.modules[k] = v
    out = dict(arr)
    out["printed_avg"], out["printed_std"] = np.asarray(printed[-2][0]), np.asarray(printed[-1][0])
    out["header"] = np.array(" ".join(printed[-3]))
    out["calls"] = np.array(sm.calls)
    out["taken"] = np.array(env.taken)
    np.savez_compressed(os.path.join(OUT, "ope_flow.npz"), **out)


if __name__ == "__main__":
    make_metrics()
    make_behavior()
    make_flow()
    print("wrote ope_metrics.npz, ope_behavior.npz, ope_flow.npz under", OUT)
