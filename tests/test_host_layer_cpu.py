"""CPU: the product's HOST layer (rl4rs_b200/env/{base,slate,seqslate}.py, gymshim, sampler, output formats) end to end
against the fixtures made by the reference's own env code -- with the device engine replaced by an oracle-backed
stand-in (tests/oracle_engine.py).  The GPU suite runs the same replay through the CUDA library
(tests/test_gpu_parity.py::test_cuda_env_matches_reference_fixture); this one keeps the Python half honest on boxes
without a GPU.  Integers bit-exact; observations / rewards at the oracle's own f32 distance from the fixtures."""
import numpy as np
import pytest

from golden_util import Golden, golden_names, assert_close_rel
from oracle_engine import OracleEngine


@pytest.fixture()
def oracle_engine(monkeypatch):
    import rl4rs_b200.engine as engine_mod
    monkeypatch.setattr(engine_mod, "Engine", OracleEngine)


def make_env(cfg, seq, catalog, log, weights, **extra):
    from rl4rs_b200 import gymshim
    from rl4rs_b200.env.slate import SlateRecEnv, SlateState
    from rl4rs_b200.env.seqslate import SeqSlateRecEnv, SeqSlateState
    cfg = dict(cfg, catalog=catalog, log=log, weights=weights, **extra)
    if seq:
        return gymshim.make("SeqSlateRecEnv-v0", recsim=SeqSlateRecEnv(cfg, state_cls=SeqSlateState))
    return gymshim.make("SlateRecEnv-v0", recsim=SlateRecEnv(cfg, state_cls=SlateState))


def obs_arrays(obs):
    if isinstance(obs, list) and isinstance(obs[0], dict):
        return {k: np.stack([np.asarray(o[k]) for o in obs]) for k in obs[0]}
    if isinstance(obs, dict):
        return {k: np.asarray(v) for k, v in obs.items()}
    return {"obs": np.asarray(obs)}


def host(x):
    return x.cpu().numpy() if hasattr(x, "is_cuda") else np.asarray(x)


def replay_through_host_layer(env, cfg, a, n_episodes, name, fmt, floor_rewards=False):
    """Replay recorded actions through the product's env classes and hold what they hand out to the record.
    floor_rewards: a step's rewards are bounded like an observation row, 1e-4 of max(|ref|, rms of the step's rewards)."""
    def arrays(obs):
        if fmt == "torch" and not isinstance(obs, dict):
            obs = {"obs": host(obs)}
        return obs_arrays({k_: host(v) for k_, v in obs.items()} if isinstance(obs, dict) else obs)

    T, k = cfg["max_steps"], 0
    for ep in range(n_episodes):
        obs = arrays(env.reset())
        np.testing.assert_array_equal(np.asarray([int(u) for u in env.user_id]), a["reset_user"][ep])
        for key, val in obs.items():
            ref = a["reset_" + key][ep]
            if key == "obs":
                assert_close_rel(val, ref, what="host %s reset obs" % name)
            else:
                np.testing.assert_array_equal(val, ref, err_msg="reset " + key)
        for t in range(T):
            np.testing.assert_array_equal(host(env.offline_action), a["offline_action"][k], err_msg="offline_action %d" % k)
            obs, reward, done, info = env.step(a["action_in"][k])
            obs = arrays(obs)
            np.testing.assert_array_equal(env.samples.prev_actions, a["prev_actions"][k])
            np.testing.assert_array_equal(env.samples.get_violation(), a["violation"][k])
            np.testing.assert_array_equal(host(done), a["done"][k])
            for key, val in obs.items():
                ref = a["step_" + key][k]
                if key == "obs":
                    assert_close_rel(val, ref, what="host %s obs step %d" % (name, k))
                else:
                    np.testing.assert_array_equal(val, ref, err_msg="%s step %d" % (key, k))
            rew = np.asarray(host(reward), dtype=np.float64).reshape(-1)
            assert_close_rel(rew[None] if floor_rewards else rew, a["reward"][k][None] if floor_rewards else a["reward"][k],
                             what="host %s reward step %d" % (name, k))
            assert_close_rel(np.asarray(host(env.offline_reward), dtype=np.float64), a["offline_reward"][k], rtol=1e-12,
                             what="host offline_reward")
            if "click_p" in a and t == T - 1:
                cp = np.stack([i["click_p"] for i in info]) if isinstance(info, list) else info["click_p"]
                assert_close_rel(cp, a["click_p"][ep], what="host click_p")
            k += 1
        with pytest.raises(Exception):
            env.step(a["action_in"][k - 1])


@pytest.mark.parametrize("fmt", ["list", "numpy", "torch"])
@pytest.mark.parametrize("name", golden_names())
def test_host_layer_replays_reference_fixture(oracle_engine, name, fmt):
    g = Golden(name)
    if fmt != "list" and name not in ("slate_rllib_replay", "seqslate36_d3rl_conti", "slate_rawstate_replay", "slate_plain_random"):
        pytest.skip("array formats checked on four fixtures (one per observation layout)")
    if "np_seed" in g.meta:
        np.random.seed(g.meta["np_seed"])
    env = make_env(g.config, g.seq, g.catalog, g.log, g.weights, output_format=fmt)
    assert env.observation_space is not None and env.action_space is not None
    replay_through_host_layer(env, g.config, g.arr, g.n_episodes, name, fmt)


def test_batch_size_one_in_every_format(oracle_engine):
    """base.py:9-23: a batch of one hands out bare elements -- in the list format (the reference's), and element by
    element in the array formats (advisor finding of round 1)."""
    g = Golden("slate_rllib_replay")
    for fmt in ("list", "numpy", "torch"):
        cfg = dict(g.config, batch_size=1, cache_size=1, is_eval=True)
        env = make_env(cfg, g.seq, g.catalog, g.log, g.weights, output_format=fmt)
        obs = env.reset()
        assert isinstance(obs, dict) and tuple(obs["obs"].shape) == (256,) and tuple(obs["action_mask"].shape) == (284,)
        a = env.offline_action
        assert np.ndim(host(a)) == 0
        obs, reward, done, info = env.step(a)
        assert tuple(obs["obs"].shape) == (256,) and np.ndim(host(reward)) == 0 and int(host(done)) == 0
        assert isinstance(info, dict)
        assert env.cur_step == 1 and isinstance(env.user_id, str)


def test_custom_obs_fn_plugin_reads_the_raw_state_rows(oracle_engine):
    """base.py:160,174 + slate.py:244-249: a RecSimBase subclass with its own obs_fn(state) gets the reference's raw
    6-field rows and can run them through self.FeatureUtil.feature_extraction exactly like the reference's obs_fn does;
    what comes out are the feature rows the engine assembled for that state."""
    from rl4rs_b200 import gymshim
    from rl4rs_b200.env.slate import SlateRecEnv, SlateState

    class PluginEnv(SlateRecEnv):
        def obs_fn(self, state):
            feat, _ = self.FeatureUtil.feature_extraction(state["state"])        # the reference's own first line
            self.last_feat = feat
            return [[len(r), int(np.sum(r[3])), float(np.sum(r[2]))] for r in state["state"]]

    g = Golden("slate_rllib_replay")
    cfg = dict(g.config, catalog=g.catalog, log=g.log, weights=g.weights)
    sim = PluginEnv(cfg, state_cls=SlateState)
    env = gymshim.make("SlateRecEnv-v0", recsim=sim)
    env.reset()
    for t in range(3):
        obs, _, _, _ = env.step(g.arr["action_in"][t])
        assert len(obs) == cfg["batch_size"] and all(o[0] == 6 for o in obs)
        seqs, dense, cat, _ = sim.last_feat
        np.testing.assert_array_equal(seqs, g.arr["seq"][t])
        np.testing.assert_array_equal(dense, g.arr["dense"][t])
        np.testing.assert_array_equal(cat, g.arr["cat"][t])


@pytest.mark.parametrize("seq,conti", [(False, False), (False, True), (True, False)])
def test_dataset_writer_host_loop(oracle_engine, seq, conti, tmp_path):
    """n2 (batchrl_trainer.py:172-320): rl4rs_b200/dataset.py's rollout / shuffle / flatten over the stand-in engine
    against the same loop written over the oracle env (the GPU twin is tests/test_gpu_dataset.py)."""
    from test_gpu_dataset import _oracle_dataset
    from test_gpu_parity import _synthetic
    from rl4rs_b200 import dataset
    B, epochs = 8, 3
    cfg, cat, log, w = _synthetic(B, seq)
    fn = {(False, False): dataset.data_generate_rl4rs_a, (False, True): dataset.data_generate_rl4rs_a_conti,
          (True, False): dataset.data_generate_rl4rs_b}[(seq, conti)]
    path = str(tmp_path / "ds.npz")
    np.random.seed(11)
    got = fn(dict(cfg, catalog=cat, log=log, weights=w), path, epochs=epochs)
    np.random.seed(11)
    O, A, R, D = _oracle_dataset(cfg, seq, conti, log, cat, w, epochs)
    T = cfg["max_steps"]
    assert got["observations"].shape == (epochs * B * (T + 1), 266) and got["observations"].dtype == np.float32
    np.testing.assert_allclose(got["observations"], O, rtol=0, atol=1e-6)
    np.testing.assert_array_equal(got["actions"], A)
    np.testing.assert_allclose(got["rewards"], R, rtol=1e-6)
    np.testing.assert_array_equal(got["terminals"], D)
    assert bool(got["discrete_action"]) == (not conti) and got["terminals"].sum() == epochs * B
    np.testing.assert_array_equal(np.load(path)["actions"], got["actions"])


def test_ppo_learns_on_the_env_through_the_host_layer(oracle_engine):
    """a23 end to end on CPU: the PPO trainer (torch twin of the kernels) driving SlateRecEnv-v0 in the 'torch' format
    through the product's env classes; the simulator behind them is the oracle.  Six iterations on 16 fixed users lift
    the greedy episode reward by 20-70 % depending on the seed (measured 262.9 -> 376.8 for seed 0); the test asks for 10 %."""
    import torch
    from test_gpu_parity import _synthetic
    from rl4rs_b200.trainer import get_rl_model
    torch.manual_seed(0)
    np.random.seed(0)
    cfg, cat, log, w = _synthetic(16, False, support_rllib_mask=True)
    env = make_env(cfg, False, cat, log, w, output_format="torch")
    tr = get_rl_model("PPO", {"lr": 3e-3, "sgd_minibatch_size": 48}, env=env, device="cpu", seed=0)
    before = tr.evaluate(1)
    stats = [tr.train() for _ in range(6)]
    after = tr.evaluate(1)
    assert all(np.isfinite(s["episode_reward_mean"]) for s in stats) and stats[-1]["timesteps_total"] == 6 * 16 * 9
    assert after > 1.1 * before, (before, after)
    # every action the policy took was legal: the reward of a slate with a violation is zeroed (slate.py:303-306)
    assert (tr.buf.reward[-1] > 0).all()
