"""CPU: the simulator trainer has one host path for every (net, head): one embedding-gradient sort, one Adam launch, and
the r4_simtrain_head_* entry points are r4_simtrain_net_* with net 0.  The learner families share one tiled GEMM, one
weight-gradient kernel with one job tiler, and one Keras Adam (r4_dense.cuh)."""
import os
import re

from test_learner_launch_path_cpu import CSRC, _body, _code

LEARN = os.path.join(CSRC, "r4_learn.cu")
SIMTRAIN = os.path.join(CSRC, "r4_simtrain.cuh")


def _functions(text):
    """The name and brace-balanced body of every top-level function definition."""
    out = []
    for m in re.finditer(r"^[A-Za-z][\w:<>, *&]*?\b(\w+)\([^;{]*?\)\s*(?=\{)", text, flags=re.M):
        out.append((m.group(1), _body(text[m.start():], re.escape(m.group(0)))))
    return out


def test_one_radix_sort_and_one_keras_adam_launch_per_family():
    learn = _code(LEARN)
    sorts = [name for name, body in _functions(learn) if "cub::DeviceRadixSort::SortPairs" in body]
    assert len(sorts) == 1, sorts
    # the Keras Adam: one launch in the simulator trainer's host path (st_apply), one in Exact-K's
    adams = [(name, len(re.findall(r"\bk_keras_adam\b", body))) for name, body in _functions(learn) if "k_keras_adam" in body]
    assert adams == [("st_apply", 1), ("r4_exactk_adam", 1)], adams
    assert len(re.findall(r"\bk_keras_adam\b", learn)) == 2


def test_the_duplicate_paths_are_gone():
    both = _code(LEARN) + _code(SIMTRAIN)
    for name in ("k_st_nembkeys", "k_st_nembsum", "apply_layout", "ncub_reserve", "st_net_classes", "sn_apply"):
        assert not re.search(r"\b%s\b" % name, both), name


def test_one_gemm_and_one_weight_gradient_kernel():
    files = sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h")))
    text = {f: open(os.path.join(CSRC, f)).read() for f in files}
    for name in ("k_gauss_wgrad", "k_ddpg_wgrad", "k_st_gemm", "k_ek_gemm", "k_st_apply", "k_ek_adam"):
        assert not any(re.search(r"\b%s\b" % name, t) for t in text.values()), name
    kernels = []
    for f in files:
        if f != "r4_gemm_tc.cuh":       # the env's tensor-core GEMM
            kernels += re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(", _code(os.path.join(CSRC, f)))
    assert [k for k in kernels if "gemm" in k] == ["k_dense_gemm"], kernels
    assert [k for k in kernels if "wgrad" in k] == ["k_dense_wgrad"], kernels
    tilers = sum(len(re.findall(r"\btile0\s*=(?!=)", _code(os.path.join(CSRC, f)))) for f in files)
    assert tilers == 1, tilers


def test_head_entry_points_forward_to_net():
    learn = _code(LEARN)
    for op in ("num_params", "scratch_size", "grad", "apply", "step", "eval"):
        body = _body(learn, r"\br4_simtrain_head_%s\(int head[^)]*\)" % op)
        inner = body[body.index("{") + 1:body.rindex("}")].strip()
        assert re.fullmatch(r"return r4_simtrain_net_%s\(R4_SIM_DIEN, head,[^;]*\);" % op, inner, flags=re.S), inner
