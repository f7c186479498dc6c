"""CPU: the v2 fused kernel's per-call tile table against the per-tile bookkeeping it replaces.

k_up2_frac2 computes a tile's interpolation bookkeeping (first output, output count, stepping-cycle range, window
offset; for the order-2 bank the call's first outputs at the tile's two ends) once per tile index of the call, in its
prologue, and every channel's tile reads that entry.  tests/cpp/fused2_tiles.cpp checks on the host that each entry
equals what every tile of every channel computes for itself, for linear and ring destinations, over every kind of
pair the planner fuses into that kernel: the 2x BlockConvolver before a whole-stepping interpolator (plain and padded
y layout), the 1x pair at the tail of a decimating chain, and the 2x pair before the order-2 bank.  (The lone 2x
BlockConvolver has no interpolation bookkeeping and no table.)  Calls of ragged lengths shift every tile boundary,
and tiny calls put the first tile's window into the history ring before the caller's block.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "r8brain-free-src_b200", "csrc")


def _cuda_include():
    for d in (os.environ.get("CUDA_HOME"), "/usr/local/cuda"):
        if d and os.path.exists(os.path.join(d, "include", "cuda_runtime.h")):
            return os.path.join(d, "include")
    return None


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    inc = _cuda_include()
    if inc is None:
        pytest.skip("CUDA headers not found")
    so = str(tmp_path_factory.mktemp("f2tiles") / "libf2tiles.so")
    srcs = [os.path.join(HERE, "cpp", "fused2_tiles.cpp")] + [os.path.join(CSRC, f) for f in
                                                              ("r8b_plan.cpp", "r8b_design.cpp", "r8b_hosttab.cpp")]
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + inc, "-o", so] + srcs,
                   check=True)
    L = C.CDLL(so)
    L.f2tiles_check.restype = C.c_int
    L.f2tiles_check.argtypes = [C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_void_p, C.c_int,
                                C.c_void_p]
    return L


def _check(L, src, dst, max_len, lens, atten=180.15, tb=2.0):
    lens = np.asarray(lens, dtype=np.int32)
    stats = np.zeros(5, dtype=np.int64)
    bad = L.f2tiles_check(src, dst, max_len, tb, atten, lens.ctypes.data, len(lens), stats.ctypes.data)
    assert bad != -1, "rate pair has no fused BlockConvolver -> interpolator pair"
    assert bad == 0, "%d tile-table entries differ from the per-tile bookkeeping" % bad
    assert stats[0] > 0
    return stats


def _lens(max_len):
    # full blocks, tiny and empty calls (the next call's first tile then starts in the history ring), odd lengths
    return [max_len, 1, 0, 3, max_len, max_len - 1, max_len // 3 + 7, 777 % max_len + 1, max_len]


@pytest.mark.parametrize("max_len", [4096, 65536, 300000])
@pytest.mark.parametrize("src,dst", [(44100.0, 96000.0),     # 2x pair, whole stepping (the benchmark's chain)
                                     (48000.0, 44100.0),     # 2x pair, padded y layout
                                     (44100.0, 48000.0)])
def test_whole_stepping_2x_pairs(lib, src, dst, max_len):
    st = _check(lib, src, dst, max_len, _lens(max_len))
    assert st[1] >= 1
    assert st[3] >= 1, "no call's first tile reached into the history ring"


@pytest.mark.parametrize("max_len", [4096, 65536])
@pytest.mark.parametrize("src,dst", [(192000.0, 44100.0), (96000.0, 44100.0), (100000.0, 44100.0)])
def test_whole_stepping_1x_pairs(lib, src, dst, max_len):
    st = _check(lib, src, dst, max_len, _lens(max_len))
    assert st[1] >= 1


@pytest.mark.parametrize("max_len", [4096, 65536])
@pytest.mark.parametrize("src,dst", [(48000.0, 47999.0), (44100.0, 44099.5)])
def test_order2_bank_pairs(lib, src, dst, max_len):
    st = _check(lib, src, dst, max_len, _lens(max_len))
    assert st[2] >= 1


def test_tile_counts_span_the_table_sizes(lib):
    # a 65536-sample call of the benchmark's chain has about 20 tiles; the longest blocks need hundreds of entries
    assert 15 <= _check(lib, 44100.0, 96000.0, 65536, [65536])[4] <= 30
    assert _check(lib, 44100.0, 96000.0, 1 << 20, [1 << 20])[4] > 300
