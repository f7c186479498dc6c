"""CPU: mixed batches (r8bgpu_batch_create_mixed) as the header declares them, as the binding binds them, their argument
checks (which run before any device is touched), the absence of a CPU fallback, and the mapped conversion kernels."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("r8bgpu_batch_create_mixed", "r8bgpu_batch_max_out_len", "r8bgpu_batch_flush_max_out_len", "r8bgpu_batch_part")


def _pkg():
    from __graft_entry__ import load_package
    return load_package()


@pytest.mark.parametrize("name", NAMES)
def test_declared_exported_bound(name):
    with open(os.path.join(ROOT, "include", "r8bgpu.h")) as f:
        assert re.search(r"R8BGPU_API\s+[\w\s\*]+\b" + name + r"\s*\(", f.read()), name + " is not declared"
    p = _pkg()
    assert name in p._SYMBOLS
    assert getattr(C.CDLL(p.lib_path()), name) is not None


def _create(p, plans, plan_of, device=-2):
    hs = (C.c_void_p * len(plans))(*[q._h for q in plans])
    po = np.ascontiguousarray(plan_of, dtype=np.int32)
    h = p.lib().r8bgpu_batch_create_mixed(hs, len(plans), po.ctypes.data, len(po), device)
    return h, p._err()


@pytest.mark.parametrize("case,words", [
    ("device_all", "R8BGPU_DEVICE_ALL"),
    ("max_in_len", "MaxInLen"),
    ("fasttiming", "FASTTIMING"),
    ("plan_of", "plan_of[2]"),
    ("empty_plan", "no channel"),
])
def test_refused_arguments(case, words):
    p = _pkg()
    a = p.Plan(44100.0, 48000.0, 4096)
    b = p.Plan(48000.0, 16000.0, 4096)
    plans, plan_of, dev = [a, b], [0, 1, 0], -2
    if case == "device_all":
        dev = p.DEVICE_ALL
    elif case == "max_in_len":
        plans = [a, p.Plan(48000.0, 16000.0, 2048)]
    elif case == "fasttiming":
        plans = [a, p.Plan(48000.0, 47999.0, 4096, fasttiming=1)]
    elif case == "plan_of":
        plan_of = [0, 1, 2]
    elif case == "empty_plan":
        plans = [a, b, p.Plan(8000.0, 16000.0, 4096)]
    h, err = _create(p, plans, plan_of, dev)
    assert not h and words in err, err


def test_no_cpu_fallback():
    p = _pkg()
    if p.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    plans = [p.Plan(44100.0, 48000.0, 4096), p.Plan(16000.0, 16000.0, 4096)]
    h, err = _create(p, plans, [1, 0, 1])
    assert not h and "no CUDA device" in err
    with pytest.raises(p.R8bGpuError):
        p.Batch.mixed(plans, [1, 0, 1])


def test_batch_caps_rule():
    # r8bgpu_batch_max_out_len / _flush_max_out_len of a mixed batch are the largest of its plans' values (restated
    # here: without a device no batch exists); a one-plan set gives the plan's own values, as an ordinary batch does
    p = _pkg()
    sets = [[(44100.0, 96000.0), (48000.0, 44100.0), (16000.0, 16000.0)], [(2822400.0, 44100.0), (8000.0, 16000.0)],
            [(48000.0, 47999.0)]]
    for s in sets:
        plans = [p.Plan(a, b, 16384) for a, b in s]
        mo = max(q.max_out_len for q in plans)
        fo = max(q.flush_max_out_len for q in plans)
        for q in plans:
            assert q.max_out_len <= mo and q.flush_max_out_len <= fo
            # every default flush of every plan fits the batch-level bound
            assert q.simulate_flush([16384, 7, 0])[1] <= fo
    assert p.Plan(16000.0, 16000.0, 16384).flush_max_out_len == 0


def test_map_kernels_compile_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("no nvcc")
    src = os.path.join(ROOT, "r8brain-free-src_b200", "csrc", "r8b_format.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c", src,
                        "-o", str(tmp_path / "f.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = r.stderr.splitlines()
    found = 0
    for i, line in enumerate(lines):
        if "Function properties for" in line and "MapRec" in line:
            found += 1
            assert "0 bytes spill stores, 0 bytes spill loads" in lines[i + 1], (line, lines[i + 1])
    assert found == 20  # 5 formats x 2 directions x planar / interleaved
