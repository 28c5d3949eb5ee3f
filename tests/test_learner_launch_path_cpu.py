"""CPU: the learner entry points launch their kernels through one launcher (csrc/r4_host.h: r4h::launch), which sets the
shared-memory opt-in and PDL and counts every launch; the shared dense kernels have one host front in r4_learn.cu; every
header includes what it uses at its head; the env's translation unit holds no learner code, and the trainers read the
launch count from the library instead of re-deriving it."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rl4rs_b200", "csrc")


def _src(path):
    """The source without its comments."""
    text = open(path).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def _code(path):
    """The source without its comments and string literals."""
    return re.sub(r'"(?:\\.|[^"\\])*"', '""', _src(path))


def _body(text, signature):
    """The brace-balanced body of the first definition whose head matches `signature`."""
    m = re.search(signature, text)
    assert m, signature
    i = text.index("{", m.end())
    depth = 0
    for j in range(i, len(text)):
        depth += {"{": 1, "}": -1}.get(text[j], 0)
        if depth == 0:
            return text[m.start():j + 1]
    raise AssertionError("unbalanced " + signature)


def test_learner_kernels_launch_only_through_the_launcher():
    learn = _code(os.path.join(CSRC, "r4_learn.cu"))
    assert "<<<" not in learn
    for api in ("cudaFuncSetAttribute", "cudaLaunchKernelEx"):
        assert api not in learn, api
    host = _code(os.path.join(CSRC, "r4_host.h"))
    launcher = _body(host, r"int launch\(") + _body(host, r"cudaError_t smem_optin\(")
    for api in ("cudaFuncSetAttribute", "cudaLaunchKernelEx"):
        assert host.count(api) == launcher.count(api) == 1, api
    assert "launch(" in learn and "count_launch(FAM_SIMTRAIN)" in learn     # the radix sort, counted once


def test_env_translation_unit_names_no_learner():
    capi = _src(os.path.join(CSRC, "r4_capi.cu"))
    for ns in ("r4ppo::", "r4gauss::", "r4ddpg::", "r4rb::", "r4bq::", "r4st::", "r4comm::", "r4dense::"):
        assert ns not in capi, ns


def test_learn_unit_includes_the_thirteen_learner_headers_and_the_env_unit_none():
    sources = [f for f in os.listdir(CSRC) if f.endswith(".cu")]
    assert sorted(sources) == ["r4_capi.cu", "r4_learn.cu"]
    includes = {f: set(re.findall(r'#include "(r4_\w+\.cuh)"', _src(os.path.join(CSRC, f)))) for f in sources}
    assert includes["r4_learn.cu"] == {"r4_ppo.cuh", "r4_comm.cuh", "r4_gauss.cuh", "r4_ddpg.cuh", "r4_rainbow.cuh",
                                       "r4_batchrl.cuh", "r4_cqlconti.cuh", "r4_bcqconti.cuh", "r4_simtrain.cuh",
                                       "r4_dense.cuh", "r4_exactk.cuh", "r4_seq2seq.cuh", "r4_ope.cuh"}
    assert not includes["r4_capi.cu"] & includes["r4_learn.cu"]


def test_headers_include_only_at_their_head():
    for f in sorted(f for f in os.listdir(CSRC) if f.endswith(".cuh")):
        lines = [l.strip() for l in _src(os.path.join(CSRC, f)).splitlines()]
        first = next(i for i, l in enumerate(lines) if l and not l.startswith("#"))
        assert not [l for l in lines[first:] if l.startswith("#include")], f


def test_the_dense_kernels_have_one_host_front():
    src = _src(os.path.join(CSRC, "r4_learn.cu"))
    for token in ("gemm_kernel(", '"k_dense_gemm"', '"k_dense_wgrad"'):
        assert src.count(token) == 1, token
    code = _code(os.path.join(CSRC, "r4_learn.cu"))
    for name in ("cq_gemm", "st_gemm", "ek_mm", "ek_bmm", "s2_mm", "s2_bmm", "ope_mm", "st_wgrad", "s2_wgrad", "cq_blocks",
                 "s2_blocks", "s2_rm", "s2_tr"):
        assert not re.search(r"\b%s\b" % name, code), name
    assert not re.search(r"\bStats\s+none\b", code)


def test_trainers_do_not_count_launches_by_hand():
    trainer = open(os.path.join(ROOT, "rl4rs_b200", "trainer.py")).read()
    assert "launches +=" not in trainer and "_chunks" not in trainer
    assert "r4_learner_launch_count" in trainer
