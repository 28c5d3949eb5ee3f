"""GPU: the CUDA path (through the reference-facing env API and the C-ABI) against
 (a) the fixtures produced by the reference's own code (tests/golden/*.npz), and
 (b) the CPU oracle on seeded synthetic inputs, incl. size-independent properties at full batch.
Integer outputs (masks, chosen items, done, features, violation) bit-exact; observations and
rewards within 1e-4 relative (golden_util.assert_close_rel states the exact bound)."""
import numpy as np
import pytest

from golden_util import Golden, golden_names, assert_close_rel

pytestmark = pytest.mark.gpu


def make_env(cfg, seq, catalog, log, weights, **extra):
    from rl4rs_b200 import gymshim
    from rl4rs_b200.env.slate import SlateRecEnv, SlateState
    from rl4rs_b200.env.seqslate import SeqSlateRecEnv, SeqSlateState
    cfg = dict(cfg, catalog=catalog, log=log, weights=weights, **extra)
    if seq:
        sim = SeqSlateRecEnv(cfg, state_cls=SeqSlateState)
        return gymshim.make("SeqSlateRecEnv-v0", recsim=sim)
    sim = SlateRecEnv(cfg, state_cls=SlateState)
    return gymshim.make("SlateRecEnv-v0", recsim=sim)


def obs_arrays(obs):
    if isinstance(obs, list) and isinstance(obs[0], dict):
        return {k: np.stack([np.asarray(o[k]) for o in obs]) for k in obs[0]}
    if isinstance(obs, dict):
        return obs
    return {"obs": np.asarray(obs)}


@pytest.mark.parametrize("fmt", ["list", "numpy"])
@pytest.mark.parametrize("name", golden_names())
def test_cuda_env_matches_reference_fixture(name, fmt):
    if fmt == "numpy" and name not in ("slate_rllib_replay", "seqslate36_rllib_replay"):
        pytest.skip("numpy format checked on two fixtures")
    g = Golden(name)
    cfg, a = g.config, g.arr
    if "np_seed" in g.meta:
        np.random.seed(g.meta["np_seed"])
    env = make_env(cfg, g.seq, g.catalog, g.log, g.weights, output_format=fmt)
    T = cfg["max_steps"]
    k = 0
    for ep in range(g.n_episodes):
        obs = obs_arrays(env.reset())
        np.testing.assert_array_equal(np.asarray([int(u) for u in env.user_id]), a["reset_user"][ep])
        for key, val in obs.items():
            ref = a["reset_" + key][ep]
            if key == "obs":
                assert_close_rel(val, ref, what="%s reset obs" % name)
            else:
                np.testing.assert_array_equal(val, ref, err_msg="reset " + key)
        for t in range(T):
            off = np.asarray(env.offline_action)
            np.testing.assert_array_equal(off, a["offline_action"][k], err_msg="offline_action %d" % k)
            obs, reward, done, info = env.step(a["action_in"][k])
            obs = obs_arrays(obs)
            np.testing.assert_array_equal(env.samples.prev_actions, a["prev_actions"][k], err_msg="prev_actions %d" % k)
            np.testing.assert_array_equal(env.samples.get_violation(), a["violation"][k], err_msg="violation %d" % k)
            np.testing.assert_array_equal(np.asarray(done), a["done"][k])
            for key, val in obs.items():
                ref = a["step_" + key][k]
                if key == "obs":
                    assert_close_rel(val, ref, what="%s obs step %d" % (name, k))
                else:
                    np.testing.assert_array_equal(val, ref, err_msg="%s step %d" % (key, k))
            if "category_feature" in obs:      # rawstate fixtures: the assembled features themselves
                np.testing.assert_array_equal(obs["category_feature"], a["cat"][k])
                np.testing.assert_array_equal(obs["dense_feature"], a["dense"][k])
                np.testing.assert_array_equal(obs["sequence_feature"], a["seq"][k])
                assert obs["dense_feature"].dtype == np.float32
            assert_close_rel(np.asarray(reward, dtype=np.float64), a["reward"][k], what="%s reward step %d" % (name, k))
            assert_close_rel(np.asarray(env.offline_reward, dtype=np.float64), a["offline_reward"][k], rtol=1e-12,
                             what="offline_reward")
            if "click_p" in a and t == T - 1:
                cp = np.stack([i["click_p"] for i in info]) if isinstance(info, list) else info["click_p"]
                assert_close_rel(cp, a["click_p"][ep], what="click_p")
            k += 1
        with pytest.raises(Exception):           # stepping past max_steps raises (slate.py:198 IndexError)
            env.step(a["action_in"][k - 1])


def test_feature_assembly_bit_exact_against_reference_fixture():
    """Feature rows (a9: seq/dense/cat) of every step, bit-exact, via rawstate_as_obs."""
    for name in ("slate_rllib_replay", "seqslate36_rllib_replay", "seqslate27_plain_mixed"):
        g = Golden(name)
        cfg = dict(g.config, rawstate_as_obs=True, support_rllib_mask=False, support_d3rl_mask=False,
                   simulator_info_fetch=False, output_format="numpy")
        env = make_env(cfg, g.seq, g.catalog, g.log, g.weights)
        k = 0
        for ep in range(g.n_episodes):
            env.reset()
            for t in range(cfg["max_steps"]):
                obs, _, _, _ = env.step(g.arr["action_in"][k])
                np.testing.assert_array_equal(obs["category_feature"], g.arr["cat"][k], err_msg="%s cat %d" % (name, k))
                np.testing.assert_array_equal(obs["dense_feature"], g.arr["dense"][k], err_msg="%s dense %d" % (name, k))
                np.testing.assert_array_equal(obs["sequence_feature"], g.arr["seq"][k], err_msg="%s seq %d" % (name, k))
                k += 1


def _synthetic(B, seq, hash_size=5000, pages=None, n_log=None, **flags):
    from rl4rs_b200 import synth
    cfg = {"maxlen": 64, "batch_size": B, "action_size": 284, "class_num": 2, "dense_feature_num": 432,
           "category_feature_num": 21, "category_hash_size": hash_size, "seq_num": 2, "emb_size": 128,
           "hidden_units": 128, "max_steps": 27 if seq else 9, "page_items": 9, "action_emb_size": 32,
           "is_eval": True, "cache_size": B}
    cfg.update(flags)
    cat = synth.make_catalog()
    log = synth.make_log(n_log or 4 * B, pages=pages or (4 if seq else 1), catalog=cat, hash_size=hash_size,
                         corrupt_frac=0.1)
    w = synth.make_weights(cfg, stress=2.0, bias_noise=0.1, bounded_scores=True)
    return cfg, cat, log, w


@pytest.mark.parametrize("seq", [False, True])
def test_cuda_env_matches_oracle_synthetic(seq):
    """Seeded synthetic rows, B=48 (ragged against the 32/64-row kernel tiles), policy = logged
    actions with 20% random replacements; compared step by step with the CPU oracle."""
    from oracle.dien_np import DienOracle
    from oracle.env_np import OracleEnv
    B = 48
    cfg, cat, log, w = _synthetic(B, seq, support_rllib_mask=True, simulator_info_fetch=True)
    env = make_env(cfg, seq, cat, log, w, output_format="numpy")
    ref = OracleEnv(cfg, log, cat, DienOracle(w, np.float32), seq=seq)
    rs = np.random.RandomState(0)
    for ep in range(2):
        o, r = env.reset(), ref.reset()
        assert_close_rel(o["obs"], r["obs"], what="reset obs")
        np.testing.assert_array_equal(o["action_mask"], r["action_mask"])
        for t in range(cfg["max_steps"]):
            a = np.where(rs.rand(B) < 0.8, ref.offline_action, rs.randint(0, 284, B))
            o, rew, done, info = env.step(a)
            r, rrew, rdone, rinfo = ref.step(a)
            np.testing.assert_array_equal(o["action_mask"], r["action_mask"], err_msg="mask %d" % t)
            np.testing.assert_array_equal(done, rdone)
            assert_close_rel(o["obs"], r["obs"], what="obs %d" % t)
            assert_close_rel(rew, rrew, what="reward %d" % t)
            np.testing.assert_array_equal(env.samples.get_violation(), ref.samples.get_violation())
        assert (np.asarray(rrew) != 0).any()


def test_conti_knn_matches_oracle_synthetic():
    """Masked kNN item search (K2): chosen items bit-exact incl. all-zero ties and f32/f64 inputs."""
    from oracle.dien_np import DienOracle
    from oracle.env_np import OracleEnv
    B = 64
    cfg, cat, log, w = _synthetic(B, False, support_rllib_mask=True, support_conti_env=True)
    env = make_env(cfg, False, cat, log, w, output_format="numpy")
    ref = OracleEnv(cfg, log, cat, DienOracle(w, np.float32))
    rs = np.random.RandomState(1)
    env.reset(); ref.reset()
    for t in range(9):
        a = rs.uniform(-1, 1, (B, 32))
        a[0] = 0.0
        a[1] = 1.0
        a[2:10] = ref.offline_action[2:10]
        a = a.astype(np.float32) if t % 2 else a
        o, rew, _, _ = env.step(a)
        r, rrew, _, _ = ref.step(a)
        np.testing.assert_array_equal(env.samples.prev_actions, ref.samples.prev_actions, err_msg="kNN step %d" % t)
        np.testing.assert_array_equal(o["action_mask"], r["action_mask"])
    assert_close_rel(rew, rrew, what="conti reward")
    # unmasked static variant (slate.py:180-184; tutorial.ipynb:251-254)
    q = rs.uniform(-1, 1, (33, 32))
    got = env.sim.engine.nearest_neighbor(q).cpu().numpy()
    np.testing.assert_array_equal(got, env.samples.get_nearest_neighbor(q, env.samples.action_emb))


def test_onehot_action_mode():
    from oracle.dien_np import DienOracle
    from oracle.env_np import OracleEnv
    B = 16
    cfg, cat, log, w = _synthetic(B, False, support_conti_env=True, support_onehot_action=True)
    env = make_env(dict(cfg), False, cat, log, w, output_format="numpy")
    ref = OracleEnv(dict(cfg), log, cat, DienOracle(w, np.float32))
    rs = np.random.RandomState(2)
    env.reset(); ref.reset()
    for t in range(9):
        a = rs.uniform(0, 1, (B, 284))
        env.step(a); ref.step(a)
        np.testing.assert_array_equal(env.samples.prev_actions, ref.samples.prev_actions)


def test_dien_forward_alone_matches_oracle():
    """The simulator network by itself (K4-K10) on random feature rows, 200 rows (ragged tiles)."""
    from oracle.dien_np import DienOracle
    cfg, cat, log, w = _synthetic(8, False)
    env = make_env(cfg, False, cat, log, w, output_format="numpy")
    rs = np.random.RandomState(3)
    R = 200
    seq = np.zeros((R, 2, 64), np.int32)
    for i in range(R):
        for s in range(2):
            n = rs.randint(0, 65)
            if n:
                seq[i, s, 64 - n:] = rs.randint(1, 284, n)
    dense = rs.normal(0, 2, (R, 432)).astype(np.float32)
    catf = rs.randint(0, 5000, (R, 21)).astype(np.int32)
    obs, probs = env.sim.engine.dien_forward(seq, dense, catf)
    o_ref, p_ref = DienOracle(w, np.float32).forward(seq, dense, catf)
    assert_close_rel(obs.cpu().numpy(), o_ref, what="dien obs")
    assert_close_rel(probs.cpu().numpy(), p_ref, what="dien probs")
    o64, _ = DienOracle(w, np.float64).forward(seq, dense, catf)
    assert_close_rel(obs.cpu().numpy(), o64, what="dien obs vs f64")


def test_batch_size_one_returns_scalars():
    cfg, cat, log, w = _synthetic(1, False, support_rllib_mask=True)
    env = make_env(cfg, False, cat, log, w)
    obs = env.reset()
    assert isinstance(obs, dict) and obs["obs"].shape == (256,)
    a = env.offline_action
    assert isinstance(a, int)
    obs, reward, done, info = env.step(a)
    assert isinstance(reward, float) and done == 0 and isinstance(info, dict)


def test_full_batch_properties():
    """BASELINE config 2 size (B=4096): size-independent properties instead of an oracle run.
    * determinism / idempotence: replaying the same rows and actions reproduces obs and rewards bit-exact;
    * row independence (the sharding premise): a row's outputs do not depend on its batch neighbours
      -- compare against a B=64 env fed a slice of the same rows/actions.  Integer outputs must be identical; float
      outputs are compared at the parity tolerance, because the launch geometry picks the AUGRU kernel (2-CTA pair
      kernel for launches that would leave SMs idle, one-CTA kernel for multi-wave launches such as the B=4096
      reward pass) and the two round differently in the last bits;
    * mask algebra: chosen items are cleared, popcounts follow the layer sizes;
    * rewards are 0 before the last step and bounded by sum(price) after it."""
    B = 4096
    cfg, cat, log, w = _synthetic(B, False, n_log=B, support_rllib_mask=True)
    env = make_env(cfg, False, cat, log, w, output_format="numpy")
    runs = []
    for rep in range(2):
        o = env.reset(reset_file=True)
        traj = [o["obs"].copy()]
        for t in range(9):
            a = env.offline_action
            o, rew, done, _ = env.step(a)
            traj.append(o["obs"].copy())
            m = o["action_mask"]
            assert not m[np.arange(B), a].any()
            if t < 8:
                assert (np.asarray(rew) == 0).all() and not done.any()
        assert done.all()
        runs.append((np.stack(traj), np.asarray(rew)))
    np.testing.assert_array_equal(runs[0][0], runs[1][0])
    np.testing.assert_array_equal(runs[0][1], runs[1][1])
    rew = runs[0][1]
    pa = env.samples.prev_actions
    assert (rew >= 0).all() and (rew <= cat.price[pa].sum(1) + 1e-9).all() and (rew > 0).mean() > 0.5
    small_cfg = dict(cfg, batch_size=64, cache_size=64)
    small = make_env(small_cfg, False, cat, log, w, output_format="numpy")
    small.sim._recData.pos = 0
    o = small.reset(reset_file=True)
    assert_close_rel(o["obs"], runs[0][0][0][:64], what="row independence: reset obs")
    for t in range(9):
        a = small.offline_action
        o, srew, _, _ = small.step(a)
        assert_close_rel(o["obs"], runs[0][0][t + 1][:64], what="row independence: obs %d" % t)
    np.testing.assert_array_equal(small.samples.prev_actions, pa[:64])
    assert_close_rel(np.asarray(srew), rew[:64], what="row independence: reward")


def test_row_chunking_is_invisible():
    """max_rows_per_pass bounds the simulator rows per launch group (obs and reward passes are chunked);
    results must not depend on it.  40-row chunks: ragged obs chunks (40 + 8 / 40 + 7); reward chunks of 4 envs (Slate 9,
    SeqSlate pages), and of 3 envs with a ragged last chunk of 2 at Slate 11."""
    for seq, T, B in ((False, 9, 48), (False, 11, 47), (True, 81, 47)):
        cfg, cat, log, w = _synthetic(B, seq, pages=-(-T // 9), support_rllib_mask=True, simulator_info_fetch=True,
                                      max_steps=T)
        runs = []
        for mr in (0, 40):
            env = make_env(dict(cfg, max_rows_per_pass=mr), seq, cat, log, w, output_format="numpy")
            o = env.reset(reset_file=True)
            tr = [o["obs"].copy()]
            for t in range(T):
                o, rew, _, info = env.step(env.offline_action)
                tr.append(o["obs"].copy())
            runs.append((np.stack(tr), np.asarray(rew), info["click_p"].copy()))
        for what, a, b in zip(("obs", "reward", "click_p"), runs[0], runs[1]):
            np.testing.assert_array_equal(a, b, err_msg="%s, %s %d, B=%d" % (what, "SeqSlate" if seq else "Slate", T, B))
