import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


_KEEP = []


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")
    # The CPU suite is hundreds of small NumPy / torch products (the oracles).  With a BLAS thread per core they spend
    # their time handing 100-microsecond products to spinning worker threads, and glibc returns every temporary above
    # 128 KB to the kernel: on the 8-core build container the same suite takes 24 minutes that way and about 4 with two
    # threads and a heap that keeps its blocks (oracle/cpu_arm.py measured the same effect on the CPU arm).  Numerics are
    # unaffected; the GPU suite does no CPU BLAS work worth threading.
    try:
        import numpy  # noqa: F401  -- the limits below apply to the BLAS libraries that are loaded when they are set
        import torch
        torch.set_num_threads(2)
    except Exception:
        pass
    try:
        from threadpoolctl import threadpool_limits
        _KEEP.append(threadpool_limits(limits=2))
    except Exception:
        pass
    try:
        from oracle.cpu_arm import _tune_malloc
        _tune_malloc()
    except Exception:
        pass


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def pytest_sessionfinish(session, exitstatus):
    """Parity margins of this session (golden_util.MARGINS): printed, and kept as gpurun_out/parity_margins.json."""
    try:
        import json
        import golden_util
        if not golden_util.MARGINS:
            return
        out = os.path.join(ROOT, "gpurun_out")
        os.makedirs(out, exist_ok=True)
        import torch
        # the CUDA suite's margins are the judged artifact; a CPU session (oracle vs fixtures) must not overwrite them
        name = "parity_margins.json" if torch.cuda.is_available() else "parity_margins_cpu.json"
        with open(os.path.join(out, name), "w") as f:
            json.dump(golden_util.MARGINS, f, indent=1, sort_keys=True)
        tr = session.config.pluginmanager.get_plugin("terminalreporter")
        if tr:
            tr.write_line("")
            tr.write_line("parity margins (floored err/bound <= 1 is the assertion; plain = element-wise |err|/|ref|):")
            for k, m in sorted(golden_util.MARGINS.items()):
                tr.write_line("  %-44s n=%-9d floored %.3f  plain rel max %.3g at |ref|=%.3g (row rms %.3g)" % (
                    k[:44], m["n"], m["floored_err_over_bound"], m["plain_rel_max"], m["plain_rel_at_abs_ref"], m["row_rms_there"]))
    except Exception as exc:      # never turn a reporting problem into a test failure
        print("parity margin report failed:", exc)
