"""Rewrites tests/golden/reference/batchrl_*.npz: what the reference's own batch-RL code computes for
tests/test_batchrl_cpu.py::test_reference_encoder_and_eval_rule_against_the_twin -- rl4rs/nets/cql/encoder.py
CustomVectorEncoder.forward and rl4rs/policy/policy_model.py policy_model.predict_with_mask, run from the reference tree.
Needs the reference tree (RL4RS_REFERENCE_ROOT); the test itself reads the stored results.

d3rlpy 0.91 and Ray are not installable here, so the names those two files import are stood in for below: d3rlpy's
VectorEncoder (restated from its published 0.91 code: the Linear + activation stack the custom encoder builds on), the
d3rlpy.algos class names policy_model dispatches on, and RLlib's Trainer class name.  Everything the files compute
themselves -- the location / prev-action / special-item masking, the embedding of the last ten columns, fc2, the zeroing,
the -2^15 eval masking and the argmax -- is the reference's own code.

    python tests/golden/make_batchrl_golden.py
"""
import contextlib
import importlib.util
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
TESTS = ["tests/test_batchrl_cpu.py::test_reference_encoder_and_eval_rule_against_the_twin"]


def _d3rlpy_stand_in():
    import torch.nn as nn

    class Encoder(nn.Module):
        pass

    class EncoderFactory(object):
        pass

    class VectorEncoder(Encoder):
        """d3rlpy 0.91 models/encoders.py VectorEncoder (the parts CustomVectorEncoder uses): hidden Linear layers with the
        activation, optional batch norm / dropout / dense skip, _feature_size = the last hidden width."""

        def __init__(self, observation_shape, hidden_units=None, use_batch_norm=False, dropout_rate=None, use_dense=False,
                     activation=nn.ReLU()):
            super().__init__()
            self._observation_shape = observation_shape
            hidden_units = [256, 256] if hidden_units is None else hidden_units
            self._use_batch_norm, self._dropout_rate, self._use_dense = use_batch_norm, dropout_rate, use_dense
            self._feature_size = hidden_units[-1]
            self._activation = activation
            in_units = [observation_shape[0]] + list(hidden_units[:-1])
            self._fcs, self._bns, self._dropouts = nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
            for i, (in_unit, out_unit) in enumerate(zip(in_units, hidden_units)):
                if use_dense and i > 0:
                    in_unit += observation_shape[0]
                self._fcs.append(nn.Linear(in_unit, out_unit))
                if use_batch_norm:
                    self._bns.append(nn.BatchNorm1d(out_unit))
                if dropout_rate is not None:
                    self._dropouts.append(nn.Dropout(dropout_rate))

        def _fc_encode(self, x):
            h = x
            for i, fc in enumerate(self._fcs):
                if self._use_dense and i > 0:
                    h = __import__("torch").cat([h, x], dim=1)
                h = self._activation(fc(h))
                if self._use_batch_norm and i != len(self._fcs) - 1:
                    h = self._bns[i](h)
                if self._dropout_rate is not None and i != len(self._fcs) - 1:
                    h = self._dropouts[i](h)
            return h

    def _create_activation(name):
        return {"relu": nn.ReLU(), "tanh": nn.Tanh()}[name]

    enc = types.ModuleType("d3rlpy.models.encoders")
    enc.Encoder, enc.EncoderFactory, enc.VectorEncoder = Encoder, EncoderFactory, VectorEncoder
    enc.VectorEncoderWithAction, enc._create_activation = VectorEncoder, _create_activation

    algos = types.ModuleType("d3rlpy.algos")

    class AlgoBase(object):
        pass
    algos.AlgoBase = AlgoBase
    for name in ("DiscreteBC", "DiscreteBCQ", "DiscreteCQL"):
        setattr(algos, name, type(name, (AlgoBase,), {}))
    models = types.ModuleType("d3rlpy.models")
    models.encoders = enc
    d3 = types.ModuleType("d3rlpy")
    d3.models, d3.algos = models, algos

    trainer = types.ModuleType("ray.rllib.agents.trainer")
    trainer.Trainer = type("Trainer", (object,), {})
    mods = {"d3rlpy": d3, "d3rlpy.models": models, "d3rlpy.models.encoders": enc, "d3rlpy.algos": algos,
            "ray": types.ModuleType("ray"), "ray.rllib": types.ModuleType("ray.rllib"),
            "ray.rllib.agents": types.ModuleType("ray.rllib.agents"), "ray.rllib.agents.trainer": trainer}
    return mods


@contextlib.contextmanager
def _stand_ins():
    mods = _d3rlpy_stand_in()
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update(mods)
    try:
        yield mods
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def _load(rel):
    from oracle import ref_harness
    path = os.path.join(ref_harness.REFERENCE_ROOT, rel)
    spec = importlib.util.spec_from_file_location("_r4_ref_" + rel.replace("/", "_").replace(".py", ""), path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def reference_encoder(config, obs, w1, b1, emb, w2, b2):
    """CustomVectorEncoder(config, action_size, mask_size = 10, with_q=True, hidden_units=[256]).forward(obs) in float64
    with the given weights (w1 [K, 256], emb [A, 32], w2 [576, A], in the y = x W + b orientation) -> [n, A]."""
    import numpy as np
    import torch
    with _stand_ins():
        mod = _load("rl4rs/nets/cql/encoder.py")
        A = emb.shape[0]
        enc = mod.CustomVectorEncoderFactory(config, action_size=A, mask_size=10, with_q=True,
                                             hidden_units=[256]).create((obs.shape[1],))
        enc = enc.double()
        with torch.no_grad():
            enc._fcs[0].weight.copy_(torch.as_tensor(w1.T))
            enc._fcs[0].bias.copy_(torch.as_tensor(b1))
            enc.emb_layer.weight.copy_(torch.as_tensor(emb))
            enc.fc2.weight.copy_(torch.as_tensor(w2.T))
            enc.fc2.bias.copy_(torch.as_tensor(b2))
            enc.location_mask = enc.location_mask.cpu()
            return np.asarray(enc(torch.as_tensor(obs, dtype=torch.float64)).numpy())


def reference_predict_with_mask(config, algo, obs, net_output):
    """policy_model(model, config).predict_with_mask(obs) for a d3rlpy model of class Discrete<algo> whose imitator (BC)
    or Q function (BCQ, CQL) outputs net_output [n, A] on obs -> actions [n]."""
    import numpy as np
    import torch
    with _stand_ins() as mods:
        mod = _load("rl4rs/policy/policy_model.py")
        model = getattr(mods["d3rlpy.algos"], "Discrete" + algo)()
        out = lambda x: torch.as_tensor(np.asarray(net_output))
        model._impl = types.SimpleNamespace(_imitator=out, _q_func=out)
        return np.asarray(mod.policy_model(model, config).predict_with_mask(obs))


if __name__ == "__main__":
    env = dict(os.environ, RL4RS_WRITE_GOLDEN="1")
    sys.exit(subprocess.call([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "not gpu"] + TESTS,
                             cwd=ROOT, env=env))
