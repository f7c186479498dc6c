"""One-byte sample formats on the host (no GPU): U8 and G.711 mu-law / A-law through r8bgpu_dither_quantize_host, the
quantiser a batch runs on the device, against a numpy restatement of G.711 written from its definition (segment ends and
biases of Sun's g711.c, as CPython's audioop uses them), pinned to fixed anchors and cross-checked against audioop where
it can still be imported.
"""
import os
import shutil
import subprocess
import warnings

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ULAW_SEG_END = np.array([0x3F, 0x7F, 0xFF, 0x1FF, 0x3FF, 0x7FF, 0xFFF, 0x1FFF])  # 14-bit magnitude + bias 33
ALAW_SEG_END = np.array([0x1F, 0x3F, 0x7F, 0xFF, 0x1FF, 0x3FF, 0x7FF, 0xFFF])  # 13-bit magnitude


def ulaw_encode(s):
    s = np.asarray(s, dtype=np.int64) >> 2
    mask = np.where(s < 0, 0x7F, 0xFF)
    mag = np.minimum(np.abs(s), 8159) + 33
    seg = np.searchsorted(ULAW_SEG_END, mag)
    code = np.where(seg >= 8, 0x7F, (seg << 4) | ((mag >> np.minimum(seg + 1, 8)) & 0x0F))
    return (code ^ mask).astype(np.uint8)


def alaw_encode(s):
    s = np.asarray(s, dtype=np.int64) >> 3
    neg = s < 0
    mag = np.where(neg, -s - 1, s)
    mask = np.where(neg, 0x55, 0xD5)
    seg = np.searchsorted(ALAW_SEG_END, mag)
    code = np.where(seg >= 8, 0x7F, (seg << 4) | ((mag >> np.where(seg < 2, 1, seg)) & 0x0F))
    return (code ^ mask).astype(np.uint8)


def ulaw_decode(c):
    u = ~np.asarray(c, dtype=np.int64) & 0xFF
    t = (((u & 0x0F) << 3) + 0x84) << ((u & 0x70) >> 4)
    return np.where(u & 0x80, 0x84 - t, t - 0x84)


def alaw_decode(c):
    a = np.asarray(c, dtype=np.int64) ^ 0x55
    seg = (a & 0x70) >> 4
    t = (a & 0x0F) << 4
    t = np.where(seg == 0, t + 8, (t + 0x108) << np.maximum(seg - 1, 0))
    return np.where(a & 0x80, t, -t)


ALL16 = np.arange(-32768, 32768, dtype=np.int64)
CODES = np.arange(256, dtype=np.int64)


def audioop():
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        try:
            import audioop as a
        except ImportError:
            pytest.skip("audioop is not available in this Python")
    return a


def test_restatement_anchors():
    assert list(ulaw_decode([0x00, 0x7F, 0x80, 0xFF])) == [-32124, 0, 32124, 0]
    assert list(alaw_decode([0x2A, 0x55, 0xAA, 0xD5])) == [-32256, -8, 32256, 8]
    s = [0, -1, 32767, -32768, 1000, -1000]
    assert list(ulaw_encode(s)) == [0xFF, 0x7E, 0x80, 0x00, 0xCE, 0x4E]
    assert list(alaw_encode(s)) == [0xD5, 0x55, 0xAA, 0x2A, 0xFA, 0x7A]


def test_restatement_matches_audioop():
    a = audioop()
    pcm = ALL16.astype("<i2").tobytes()
    np.testing.assert_array_equal(np.frombuffer(a.lin2ulaw(pcm, 2), np.uint8), ulaw_encode(ALL16))
    np.testing.assert_array_equal(np.frombuffer(a.lin2alaw(pcm, 2), np.uint8), alaw_encode(ALL16))
    codes = CODES.astype(np.uint8).tobytes()
    np.testing.assert_array_equal(np.frombuffer(a.ulaw2lin(codes, 2), "<i2"), ulaw_decode(CODES))
    np.testing.assert_array_equal(np.frombuffer(a.alaw2lin(codes, 2), "<i2"), alaw_decode(CODES))


def test_constants(pkg):
    assert (pkg.U8, pkg.ULAW, pkg.ALAW) == (5, 6, 7)
    assert pkg.FORMAT_BYTES[pkg.U8] == pkg.FORMAT_BYTES[pkg.ULAW] == pkg.FORMAT_BYTES[pkg.ALAW] == 1
    with open(os.path.join(ROOT, "include", "r8bgpu.h")) as f:
        h = f.read()
    for name, v in (("U8", 5), ("ULAW", 6), ("ALAW", 7)):
        assert "R8BGPU_%s = %d" % (name, v) in h


def cast(pkg, y, fmt):
    q, st = pkg.dither_quantize(np.asarray(y, dtype=np.float64), fmt, 0, kind=pkg.DITHER_OFF)
    assert q.dtype == np.uint8 and q.shape == (len(y),)
    assert not st.any()
    return q


@pytest.mark.parametrize("fmt,enc", [(6, ulaw_encode), (7, alaw_encode)])
def test_every_int16_encodes(pkg, fmt, enc):
    np.testing.assert_array_equal(cast(pkg, ALL16, fmt), enc(ALL16))


@pytest.mark.parametrize("fmt,enc", [(6, ulaw_encode), (7, alaw_encode)])
def test_cast_takes_the_s16_rule_first(pkg, fmt, enc):
    y = np.array([0.7, -0.7, 999.9, -999.9, 32767.9, -32768.9, 32768.0, -32769.0, 1e9, -1e9, np.inf, -np.inf, np.nan, -0.0])
    s16, _ = pkg.dither_quantize(y, pkg.S16, 0, kind=pkg.DITHER_OFF)
    assert list(s16) == [0, 0, 999, -999, 32767, -32768, 32767, -32768, 32767, -32768, 32767, -32768, 0, 0]
    np.testing.assert_array_equal(cast(pkg, y, fmt), enc(s16))


def test_u8_cast(pkg):
    v = np.arange(-200, 201, dtype=np.float64)
    np.testing.assert_array_equal(cast(pkg, v, pkg.U8), np.clip(v, -128, 127).astype(np.int64) + 128)
    y = np.array([0.9, -0.9, 127.99, -128.99, np.inf, -np.inf, np.nan])
    assert list(cast(pkg, y, pkg.U8)) == [128, 128, 255, 0, 255, 0, 128]
    # scale applies before the cast, as for the other integer formats
    q, _ = pkg.dither_quantize(np.array([0.5, -0.5, 1.0]), pkg.U8, 0, scale=128.0, kind=pkg.DITHER_OFF)
    assert list(q) == [192, 64, 255]


TAPS = [2.033, -2.165, 1.959, -1.590, 0.6149, -0.2, 0.1, -0.05, 0.01]


def dithered_signal(n):
    rng = np.random.default_rng(11)
    y = rng.uniform(-300, 300, n) + np.sin(np.arange(n) * 0.003) * 20000.0
    y[::211] = rng.uniform(-40000, 40000, len(y[::211]))
    y[7], y[13], y[19] = np.nan, np.inf, -np.inf
    return y


@pytest.mark.parametrize("taps", [None, TAPS])
@pytest.mark.parametrize("fmt,enc", [(6, ulaw_encode), (7, alaw_encode)])
def test_companded_dither_is_the_s16_dither_encoded(pkg, taps, fmt, enc):
    y = dithered_signal(5000)
    st0 = np.random.default_rng(3).uniform(-1, 1, 16)
    s16, st16 = pkg.dither_quantize(y, pkg.S16, 77, taps, first_index=999, state=st0.copy())
    q, st = pkg.dither_quantize(y, fmt, 77, taps, first_index=999, state=st0.copy())
    np.testing.assert_array_equal(q, enc(s16))
    np.testing.assert_array_equal(st, st16)


@pytest.mark.parametrize("taps", [None, TAPS])
def test_u8_dither_is_int8(pkg, taps):
    y = dithered_signal(5000) / 256.0
    s16, st16 = pkg.dither_quantize(y, pkg.S16, 5, taps, first_index=3)
    q, st = pkg.dither_quantize(y, pkg.U8, 5, taps, first_index=3)
    np.testing.assert_array_equal(q.astype(np.int64), np.clip(s16.astype(np.int64), -128, 127) + 128)
    np.testing.assert_array_equal(st, st16)


def test_refusals(pkg):
    for fmt in (8, 99, -1, pkg.F32, pkg.F64):
        with pytest.raises(pkg.R8bGpuError, match="fmt must be"):
            pkg.dither_quantize(np.zeros(4), fmt, 1)


def test_byte_format_kernels_compile_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("no nvcc")
    src = os.path.join(ROOT, "r8brain-free-src_b200", "csrc", "r8b_format_bytes.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c", src,
                        "-o", str(tmp_path / "f.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = r.stderr.splitlines()
    found = 0
    for i, line in enumerate(lines):
        if "Function properties for" in line and "k_cvt_" in line:
            found += 1
            assert "0 bytes spill stores, 0 bytes spill loads" in lines[i + 1], (line, lines[i + 1])
    assert found == 36  # 3 formats x (plain, ragged, mapped) x 2 directions x planar / interleaved
