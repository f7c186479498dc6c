"""CDSPResamplerBatch::oneshotCrops from C++, both overloads, compiled and linked against libr8bgpu.so.  Without a device
each call fails cleanly with a message; with one, every crop is bit for bit what Batch.oneshot_crops returns."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 20000
LENS = [N, 15000]
CROPS = [(1, 100, 160), (0, 2000, 2100), (0, 6000, 6060)]


def test_cpp_oneshot_crops(pkg, tmp_path):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no g++")
    lib_dir = os.path.dirname(pkg.lib_path())
    exe = str(tmp_path / "oneshot_crops_demo")
    subprocess.run([gxx, "-O1", "-std=c++11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "oneshot_crops_demo.cpp"), "-o", exe, "-L", lib_dir, "-lr8bgpu",
                    "-Wl,-rpath," + lib_dir], check=True)
    res = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    rows = {}
    for line in res.stdout.strip().split("\n"):
        name, k, rest = (line.split(" ", 2) + [""])[:3]
        rows[(name, int(k))] = rest
    if pkg.device_count() < 1:
        assert set(rows) == {("one_pair", -1), ("per_clip", -1)}
        assert all(m for m in rows.values())  # a message from batch creation
        return
    i = np.arange(N)
    x = np.stack([((i * 7 + r * 3) % 101 - 50) / 64.0 for r in range(2)])
    p48 = pkg.Plan(48000.0, 16000.0, 4096, 2.0, 206.91)
    p44 = pkg.Plan(44100.0, 16000.0, 4096, 2.0, 206.91)
    want = {"one_pair": pkg.Batch(p48, 4, device=0).oneshot_crops(x, CROPS, LENS)}
    mixed = pkg.Batch.mixed([p48, p44], [0, 0, 1, 1], device=0)
    want["per_clip"] = mixed.oneshot_crops(x, CROPS, LENS, plan_of=[1, 0])
    for name, y in want.items():
        for k, (_, o0, o1) in enumerate(CROPS):
            got = np.array([float.fromhex(v) for v in rows[(name, k)].split()])
            assert got.tobytes() == np.ascontiguousarray(y[k, :o1 - o0]).tobytes(), (name, k)
