"""CPU: the batch-RL front keeps one copy of what the discrete and continuous learners share -- one device dataset, one
model base, one flat-parameter builder for the twins and one epoch driver in the host code -- and each family's
checkpoint keeps its keys."""
import ast
import inspect
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _source(*parts):
    with open(os.path.join(ROOT, *parts)) as f:
        return f.read()


def _methods(tree):
    """(class name, name) of every method a class of the module defines, by def or by assignment."""
    out = []
    for c in (c for c in tree.body if isinstance(c, ast.ClassDef)):
        for f in c.body:
            if isinstance(f, ast.FunctionDef):
                out.append((c.name, f.name))
            elif isinstance(f, ast.Assign):
                out += [(c.name, t.id) for t in f.targets if isinstance(t, ast.Name)]
    return out


# ---- one copy of each shared part ------------------------------------------------------------------------
def test_one_device_dataset():
    from rl4rs_b200 import batchrl
    assert "ContiDeviceDataset" not in _source("rl4rs_b200", "batchrl.py")
    assert not hasattr(batchrl, "ContiDeviceDataset")


@pytest.mark.parametrize("name", ["fit", "save_model", "load_model", "_device_data", "_epoch_twin", "fit_reward_scaler"])
def test_one_model_base(name):
    tree = ast.parse(_source("rl4rs_b200", "batchrl.py"))
    assert len([c for c, f in _methods(tree) if f == name]) == 1


def test_one_device_rule_and_memory_check():
    src = _source("rl4rs_b200", "batchrl.py")
    assert src.count("mem_get_info") == 1
    assert src.count('torch.cuda.is_available() and config.get("gpu", True)') == 1


def test_no_method_borrowed_from_another_class():
    tree = ast.parse(_source("rl4rs_b200", "batchrl.py"))
    classes = {c.name for c in tree.body if isinstance(c, ast.ClassDef)}
    borrowed = [(c.name, ast.unparse(a)) for c in tree.body if isinstance(c, ast.ClassDef)
                for a in c.body if isinstance(a, ast.Assign)
                for v in ast.walk(a.value) if isinstance(v, ast.Attribute) and isinstance(v.value, ast.Name)
                and v.value.id in classes]
    assert borrowed == []


def test_one_init_loop_among_the_twins():
    from rl4rs_b200 import policy
    classes = {k for c in (policy.BatchRLNet, policy.BatchRLContiNet, policy.BatchRLContiBCQNet)
               for k in inspect.getmro(c) if k is not object}
    src = "".join(inspect.getsource(k) for k in classes)
    assert src.count("torch.Generator(") == 1
    assert src.count("torch.rand(shape, generator=g)") == 1


def test_one_epoch_driver():
    src = _source("rl4rs_b200", "csrc", "r4_learn.cu")
    assert src.count("too many steps") == 1
    assert src.count("r4cqlc::Data{") == 1


# ---- what each family writes -------------------------------------------------------------------------------
SHARED = {"algo", "obs_dim", "params", "target", "m", "v", "step", "reward_scaler", "reward_mean", "reward_std"}


@pytest.mark.parametrize("algo", ["BC", "BCQ", "CQL", "BCQ-conti", "CQL-conti"])
def test_checkpoint_keys(algo, tmp_path):
    from rl4rs_b200 import batchrl, synth
    if algo.endswith("conti"):
        from test_batchrl_conti_cpu import conti_dataset
        cfg = {"action_size": 284, "action_emb_size": 3, "support_conti_env": True, "gpu": False}
        ds, extra = conti_dataset(20, 3, E=2, L=6), {"action_dim", "act_counter", "gen"}
    else:
        from test_batchrl_cpu import synthetic_dataset
        cfg = {"action_size": 284, "page_items": 9, "catalog": synth.make_catalog(), "gpu": False}
        ds, extra = synthetic_dataset(E=2), {"action_size"}
    m = batchrl.get_model(cfg, algo)
    m.build_with_dataset(ds)
    path = str(tmp_path / "m.pt")
    m.save_model(path)
    assert set(torch.load(path)) == SHARED | extra
