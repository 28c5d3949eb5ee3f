"""Rewrites tests/golden/reference/*.npz: what the reference's own code computes for the tests that compare against it
(golden_util.reference_result).  Needs the reference tree (RL4RS_REFERENCE_ROOT); the tests themselves do not.

    python tests/golden/make_reference_golden.py
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
TESTS = ["tests/test_oracle_vs_reference_random.py", "tests/test_env_base_cpu.py",
         "tests/test_reference_graph.py::test_the_references_own_stack_with_the_other_simulators",
         "tests/test_reference_graph.py::test_rllib_policy_models_of_the_reference_against_the_torch_twins"]

if __name__ == "__main__":
    env = dict(os.environ, RL4RS_WRITE_GOLDEN="1")
    sys.exit(subprocess.call([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "not gpu"] + TESTS,
                             cwd=ROOT, env=env))
