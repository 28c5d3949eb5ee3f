"""CPU: the learner fronts share their code instead of copying it -- no method borrowed by class-attribute assignment, the
replay learners as siblings over one skeleton, one ctypes calling convention in _capi, one checkpoint path -- and each
algorithm family's checkpoint keeps its file format."""
import ast
import os
import tempfile

import pytest
import torch

from rl4rs_b200 import trainer
from test_trainer_conti_cpu import FakeContiEnv
from test_trainer_cpu import FakeEnv
from test_trainer_rainbow_cpu import FakeEnv as PlainEnv

PKG = os.path.dirname(os.path.abspath(trainer.__file__))
CTYPES_FRONTS = ("trainer.py", "batchrl.py", "simtrain.py", "engine.py")


def _modules():
    return {f: open(os.path.join(PKG, f)).read() for f in sorted(os.listdir(PKG)) if f.endswith(".py")}


def test_no_method_is_borrowed_from_a_learner_front():
    trees = {f: ast.parse(src) for f, src in _modules().items()}
    classes = {n.name for n in ast.walk(trees["trainer.py"]) if isinstance(n, ast.ClassDef)}
    borrowed = ["%s: %s.%s = %s.%s" % (f, c.name, s.targets[0].id, s.value.value.id, s.value.attr)
                for f, t in trees.items() for c in ast.walk(t) if isinstance(c, ast.ClassDef) for s in c.body
                if isinstance(s, ast.Assign) and isinstance(s.targets[0], ast.Name) and isinstance(s.value, ast.Attribute)
                and isinstance(s.value.value, ast.Name) and s.value.value.id in classes]
    assert not borrowed, borrowed


def test_replay_learners_are_siblings():
    assert not issubclass(trainer.RainbowTrainer, trainer.DDPGTrainer)
    for cls in (trainer.DDPGTrainer, trainer.TD3Trainer, trainer.RainbowTrainer):
        assert issubclass(cls, trainer._ReplayTrainer), cls


def test_one_ctypes_calling_convention():
    src = _modules()
    pointer_helpers = [f for f, s in src.items() if "c_void_p(t.data_ptr()" in s]
    assert pointer_helpers == ["_capi.py"], pointer_helpers
    assert [f for f in CTYPES_FRONTS if "cuda_stream" in src[f]] == []
    assert [f for f, s in src.items() if "failed (%d)" in s] == ["_capi.py"]


def test_one_checkpoint_path():
    tree = ast.parse(_modules()["trainer.py"])
    defs = [n.name for n in ast.walk(tree) if isinstance(n, ast.FunctionDef)]
    assert defs.count("save") == 1 and defs.count("restore") == 1


ON_POLICY = {"algo", "flat", "opt", "kernel_adam", "iteration", "timesteps_total", "extra"}
DDPG = {"algo", "flat", "target", "opt_actor", "opt_critic", "kernel_adam", "ou_state", "ou_slot", "counter", "policy_ts",
        "actor_steps", "critic_steps", "gen", "iteration", "timesteps_total"}
RAINBOW = {"algo", "flat", "target", "opt", "kernel_adam", "counter", "policy_ts", "last_target_update", "sgd_steps", "gen",
           "iteration", "timesteps_total"}


@pytest.mark.parametrize("algo,env,keys", [("PPO", FakeEnv, ON_POLICY), ("A2C_conti", FakeContiEnv, ON_POLICY),
                                           ("PG", FakeEnv, ON_POLICY), ("IMPALA", FakeEnv, ON_POLICY),
                                           ("DDPG", FakeContiEnv, DDPG), ("TD3", FakeContiEnv, DDPG),
                                           ("RAINBOW", PlainEnv, RAINBOW)])
def test_checkpoint_keys(algo, env, keys):
    tr = trainer.get_rl_model(algo, {}, env=env(8), device="cpu")
    st = torch.load(tr.save(tempfile.mkdtemp()), map_location="cpu")
    assert set(st) == keys and st["algo"] == algo and st["kernel_adam"] is None
