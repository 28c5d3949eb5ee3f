"""rl4rs_b200 -- H100-native batched SlateRecEnv / SeqSlateRecEnv (the RL4RS hot path).

Importing the package does not need a GPU; constructing an env does (no CPU fallback).
Env ids are registered like rl4rs/__init__.py:10-18.
"""
from . import gymshim

gymshim.register(id="SlateRecEnv-v0", entry_point="rl4rs_b200.env:RecEnvBase")
gymshim.register(id="SeqSlateRecEnv-v0", entry_point="rl4rs_b200.env:RecEnvBase")

__version__ = "0.1.0"
