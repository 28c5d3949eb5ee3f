"""CPU: the simulator trainer has one host path for every (net, head): one embedding-gradient sort, one Adam launch, and
the r4_simtrain_head_* entry points are r4_simtrain_net_* with net 0."""
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


def test_one_radix_sort_and_one_adam_launch():
    learn = _code(LEARN)
    sorts = [name for name, body in _functions(learn) if "cub::DeviceRadixSort::SortPairs" in body]
    assert len(sorts) == 1, sorts
    assert len(re.findall(r"\bk_st_apply\b", learn)) == 1


def test_the_duplicate_paths_are_gone():
    both = _code(LEARN) + _code(SIMTRAIN)
    for name in ("k_st_nembkeys", "k_st_nembsum", "apply_layout", "ncub_reserve", "st_net_classes", "sn_apply"):
        assert not re.search(r"\b%s\b" % name, both), name


def test_head_entry_points_forward_to_net():
    learn = _code(LEARN)
    for op in ("num_params", "scratch_size", "grad", "apply", "step", "eval"):
        body = _body(learn, r"\br4_simtrain_head_%s\(int head[^)]*\)" % op)
        inner = body[body.index("{") + 1:body.rindex("}")].strip()
        assert re.fullmatch(r"return r4_simtrain_net_%s\(R4_SIM_DIEN, head,[^;]*\);" % op, inner, flags=re.S), inner
