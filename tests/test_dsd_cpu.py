"""One-bit DSD input on the host (no GPU): the layout, restated with np.unpackbits and pinned to hand anchors; the
__host__ __device__ decode of r8b_dsd.cuh, compiled for the host, against that restatement for every byte, both bit
orders and both layouts; the refusal of DSD by the host quantiser; and what the compiler makes of the kernels -- the
conversion kernels without spills, and every kernel of r8b_kernels.cu that predates DSD with the registers and spills
it had before (tests/golden/r8b_kernels_ptxas.json), since the DSD instantiations of the half-band decimators must
leave their fp64 instantiations as they were.
"""
import ctypes as C
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "r8brain-free-src_b200", "csrc")
DSD_LSB, DSD_MSB = 16, 17


def nvcc():
    n = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if n is None:
        pytest.skip("no nvcc")
    return n


def decode_planar(byt, scale, msb):
    """Planar DSD bytes [n_ch, w] -> samples [n_ch, 8 w]: bit i % 8 (LSB order) or 7 - i % 8 (MSB) of byte i / 8."""
    bits = np.unpackbits(np.asarray(byt, dtype=np.uint8), axis=-1, bitorder="big" if msb else "little")
    return np.where(bits != 0, scale, -scale)


def decode_interleaved(byt, scale, msb):
    """Interleaved DSD bytes [w, n_ch] (byte frame f, channel c) -> planar samples [n_ch, 8 w]."""
    return decode_planar(np.asarray(byt).T, scale, msb)


def test_layout_anchors():
    assert list(decode_planar([[0x01]], 1.0, False)[0]) == [1.0] + [-1.0] * 7
    assert list(decode_planar([[0x80]], 1.0, True)[0]) == [1.0] + [-1.0] * 7
    assert list(decode_planar([[0x80]], 1.0, False)[0]) == [-1.0] * 7 + [1.0]
    assert list(decode_planar([[0x03, 0xFE]], 0.5, False)[0]) == [0.5, 0.5] + [-0.5] * 6 + [-0.5] + [0.5] * 7
    il = np.array([[0x01, 0x80], [0xFF, 0x00]], dtype=np.uint8)  # byte frames 0 and 1 of channels 0 and 1
    y = decode_interleaved(il, 1.0, False)
    assert list(y[0]) == [1.0] + [-1.0] * 7 + [1.0] * 8
    assert list(y[1]) == [-1.0] * 7 + [1.0] + [-1.0] * 8


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("dsd") / "libdsd.so")
    subprocess.run([nvcc(), "-std=c++17", "-O2", "--shared", "-Xcompiler", "-fPIC", "-o", so,
                    os.path.join(HERE, "cpp", "dsd_decode.cu")], check=True)
    L = C.CDLL(so)
    L.dsd_decode.restype = None
    L.dsd_decode.argtypes = [C.c_void_p, C.c_int, C.c_longlong, C.c_int, C.c_longlong, C.c_longlong, C.c_int, C.c_double,
                             C.c_void_p]
    return L


@pytest.mark.parametrize("msb", [False, True])
@pytest.mark.parametrize("interleaved", [False, True])
def test_host_decode_matches_restatement(lib, msb, interleaved):
    n_ch, scale, i0 = 3, 0.5, 13  # an odd start index: the decode is relative to the buffer's first sample
    rng = np.random.default_rng(3)
    planar = np.stack([np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8)[::-1],
                       rng.permutation(256).astype(np.uint8)])  # every byte value in every channel
    want = decode_planar(planar, scale, msb)
    raw = np.ascontiguousarray(planar.T if interleaved else planar)
    stride = n_ch if interleaved else planar.shape[1]
    n = want.shape[1] - i0
    for c in range(n_ch):
        got = np.zeros(n)
        lib.dsd_decode(raw.ctypes.data, int(interleaved), stride, c, i0, n, int(msb), scale, got.ctypes.data)
        np.testing.assert_array_equal(got, want[c, i0:])


def test_quantiser_refuses_dsd(pkg):
    assert (pkg.DSD_LSB, pkg.DSD_MSB) == (DSD_LSB, DSD_MSB)
    assert pkg.FORMAT_BYTES[pkg.DSD_LSB] == 1 and pkg.FORMAT_SAMPLES[pkg.DSD_MSB] == 8
    with open(os.path.join(ROOT, "include", "r8bgpu.h")) as f:
        h = f.read()
    assert "R8BGPU_DSD_LSB = 16" in h and "R8BGPU_DSD_MSB = 17" in h
    for fmt in (DSD_LSB, DSD_MSB):
        with pytest.raises(pkg.R8bGpuError, match="fmt must be"):
            pkg.dither_quantize(np.zeros(4), fmt, 1)


# A name in an anonymous namespace carries a hash of the compiled file's path: keep only the namespace's marker.
ANON = re.compile(r"\d+_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]{8}")


def ptxas(src, tmp_path):
    r = subprocess.run([nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                        os.path.join(CSRC, src), "-o", str(tmp_path / "k.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = r.stderr.splitlines()
    out = {}
    for i, line in enumerate(lines):
        m = re.search(r"Function properties for (\S+)", line)
        if not m:
            continue
        sp = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", lines[i + 1])
        regs = next((int(g.group(1)) for g in (re.search(r"Used (\d+) registers", x) for x in lines[i + 1:i + 5]) if g), None)
        out[ANON.sub("_GLOBAL__N_", m.group(1))] = [regs, int(sp.group(1)), int(sp.group(2))]
    return out


def test_conversion_kernels_compile_without_spills(tmp_path):
    figs = {k: v for k, v in ptxas("r8b_format_dsd.cu", tmp_path).items() if "k_dsd_" in k}
    assert len(figs) == 6, sorted(figs)  # (plain, ragged, mapped) x (planar, interleaved)
    for k, (regs, st, ld) in figs.items():
        assert st == 0 and ld == 0, (k, st, ld)


def test_existing_kernels_keep_their_figures(tmp_path):
    with open(os.path.join(HERE, "golden", "r8b_kernels_ptxas.json")) as f:
        want = json.load(f)
    got = ptxas("r8b_kernels.cu", tmp_path)
    for name, fig in want.items():
        assert got.get(name) == fig, (name, got.get(name), fig)
    # what is new: the DSD instantiations of the two half-band decimators and of the history copy
    assert len(got) - len(want) == 3, sorted(set(got) - set(want))
