"""The per-clip-rate long-clip calls from C++ (CDSPResamplerBatch::oneshotLong / oneshotLongAdjoint overloads) and the
r8bgpu_batch_oneshot_mixed* C entry points, compiled and linked against libr8bgpu.so.  Without a device every call
fails cleanly, with a message; with one, the clips at known rate pairs run and an unknown pair is refused."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cpp_mixed_oneshot_calls(pkg, tmp_path):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no g++")
    lib_dir = os.path.dirname(pkg.lib_path())
    exe = str(tmp_path / "oneshot_mixed_demo")
    subprocess.run([gxx, "-O1", "-std=c++11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "oneshot_mixed_demo.cpp"), "-o", exe, "-L", lib_dir, "-lr8bgpu",
                    "-Wl,-rpath," + lib_dir], check=True)
    res = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    rows = {}
    for line in res.stdout.strip().split("\n"):
        name, rc, msg = line.split(" ", 2)
        rows[name] = (int(rc), msg)
    assert set(rows) == {"long", "long_unknown_pair", "adjoint_unknown_pair", "c_mixed", "c_mixed_host", "c_adjoint_mixed"}
    for name in ("c_mixed", "c_mixed_host", "c_adjoint_mixed"):
        assert rows[name][0] == -1 and "bad arguments" in rows[name][1], (name, rows[name])
    if pkg.device_count() < 1:
        for name in ("long", "long_unknown_pair", "adjoint_unknown_pair"):
            assert rows[name][0] == -1 and "no CUDA device" in rows[name][1], (name, rows[name])
    else:
        assert rows["long"] == (0, "-")
        for name in ("long_unknown_pair", "adjoint_unknown_pair"):
            assert rows[name][0] == -1 and "not a plan index" in rows[name][1], (name, rows[name])
