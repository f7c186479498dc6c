"""CPU: the large-tile BlockConvolver (16384 .. 65536-point tiles) without a GPU.

* The host tile choice over a grid of rate pairs, transition bands, attenuations and R8B_EXTFFT: every BlockConvolver
  stage gets a supported tile, and every stage that the in-shared-memory tiles already served keeps exactly the tile,
  half support and view it had (the rule those tiles follow is restated here independently).
* The per-thread steps of k_bcl_gather / k_bcl_conv / k_bcl_scatter (csrc/r8b_bclarge.cuh), run thread by thread on the
  host by tests/cpp/bclarge_emul.cpp on the engine's own one-stage plan, schedule and tables, against the compiled
  reference's own BlockConvolver stage: equal per-call counts, <= 32 eps max and <= 4 eps rms, ragged calls.
"""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

import oracle_util

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "r8brain-free-src_b200", "csrc")
EPS = 2.0 ** -52

RATES = [8000.0, 11025.0, 16000.0, 22050.0, 32000.0, 44100.0, 44101.0, 47999.0, 48000.0, 64000.0, 88200.0, 96000.0,
         176400.0, 192000.0, 352800.0, 384000.0]
TBS = [0.5, 0.75, 1.0, 1.5, 2.0, 45.0]
ATTENS = [49.0, 109.56, 136.45, 180.15, 206.91, 218.0]


def _cuda_include():
    for d in (os.environ.get("CUDA_HOME"), "/usr/local/cuda"):
        if d and os.path.exists(os.path.join(d, "include", "cuda_runtime.h")):
            return os.path.join(d, "include")
    return None


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    inc = _cuda_include()
    if inc is None:
        pytest.skip("CUDA headers not found")
    so = str(tmp_path_factory.mktemp("bclemul") / "libbclemul.so")
    srcs = [os.path.join(HERE, "cpp", "bclarge_emul.cpp")] + [os.path.join(CSRC, f) for f in
                                                              ("r8b_plan.cpp", "r8b_design.cpp", "r8b_hosttab.cpp")]
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + inc, "-o", so] + srcs,
                   check=True)
    L = C.CDLL(so)
    dp = C.POINTER(C.c_double)
    L.bclemul_tiles.argtypes = [C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_int, C.POINTER(C.c_int),
                                C.c_int]
    L.bclemul_find.argtypes = [C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_int, dp]
    L.bclemul_create.restype = C.c_void_p
    L.bclemul_create.argtypes = [dp, C.c_int, C.c_int]
    L.bclemul_destroy.argtypes = [C.c_void_p]
    L.bclemul_info.restype = C.c_double
    L.bclemul_info.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
    L.bclemul_process.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    return L


def _old_rule(up, down, block_exact, half_len, prev_len, blk_log2):
    """The in-shared-memory tile rule the engine had before the large-tile path: (fft_log2 or -1, lg, virt_up)."""
    virt_up, up_eff = (up, 1) if up > 2 else (1, up)
    if block_exact:
        lo, hi = (6, 13) if up_eff == 1 else (10, 12)
        return (blk_log2 if lo <= blk_log2 <= hi else -1), prev_len - half_len, virt_up
    lg = (half_len + up_eff - 1) // up_eff
    best, best_cost = -1, 0.0
    for b in range(10, (13 if up_eff == 1 else 12) + 1):
        m = 1 << b
        valid = m - 2 * lg
        if valid < 64:
            continue
        cost = b * m / valid
        if best < 0 or cost < best_cost:
            best, best_cost = b, cost
    return best, lg, virt_up


def test_tile_choice_covers_the_parameter_space_and_keeps_every_existing_tile(emul):
    buf = (C.c_int * 200)()
    n_cfg = n_large = n_stages = 0
    for (src, dst), tb, atten, ext in itertools.product(itertools.permutations(RATES, 2), TBS, ATTENS, (0, 1)):
        if src / dst > 40 or dst / src > 40:
            continue
        n = emul.bclemul_tiles(src, dst, 4096, tb, atten, ext, buf, 20)
        assert n >= 0, (src, dst, tb, atten, ext)
        n_cfg += 1
        for i in range(n):
            up, down, be, half_len, prev_len, blk, fl, large, lg, vup = buf[10 * i:10 * i + 10]
            cfg = (src, dst, tb, atten, ext, i, up, down, be, half_len)
            n_stages += 1
            old_fl, old_lg, old_vup = _old_rule(up, down, be, half_len, prev_len, blk)
            if old_fl >= 0:
                assert (fl, lg, vup, large) == (old_fl, old_lg, old_vup, 0), cfg
                continue
            n_large += 1
            assert large == 1 and 14 <= fl <= 16, cfg
            if be:
                assert fl == blk and lg == prev_len - half_len and vup == max(1, up if up > 2 else 1), cfg
            else:
                assert vup == (up if up > 1 else 1) and lg == half_len, cfg
                assert (1 << fl) - 2 * lg >= 64, cfg
    assert n_cfg > 10000 and n_large > 1000, (n_cfg, n_large, n_stages)


def _run(L, src, dst, max_len, tb, atten, ext, lens, want_log2=None, want_block_exact=None, seed=11):
    flavor = "e1" if ext else "e0"
    if not oracle_util.have_ref(flavor):
        pytest.skip("oracle/_ref not built (needs /root/reference at build time)")
    ref = oracle_util.RefOracle(flavor)
    a = (C.c_double * 6)()
    in_max = L.bclemul_find(src, dst, max_len, tb, atten, ext, a)
    assert in_max > 0, "no BlockConvolver stage of this plan takes the large-tile path"
    h = L.bclemul_create(a, in_max, ext)
    assert h
    info = (C.c_int * 4)()
    spectrum_ms = L.bclemul_info(h, info)
    if want_log2 is not None:
        assert info[0] == want_log2, list(info)
    if want_block_exact is not None:
        assert info[3] == int(want_block_exact), list(info)
    rs = ref.stage_blockconv(a[0], a[1], a[2], a[3], int(a[4]), int(a[5]))
    rng = np.random.default_rng(seed)
    worst = se = sy = 0.0
    total = 0
    for n in lens:
        n = min(n, in_max)
        x = rng.uniform(-1.0, 1.0, n)
        out = np.zeros(int(n * a[4] / a[5]) + 64)
        k = L.bclemul_process(h, x.ctypes.data, n, out.ctypes.data, len(out))
        yr = rs.process(x)
        assert k == len(yr), (k, len(yr))
        if k:
            d = out[:k] - yr
            worst = max(worst, float(np.max(np.abs(d))) / float(np.max(np.abs(yr))))
            se += float(np.sum(d * d))
            sy += float(np.sum(yr * yr))
            total += k
    L.bclemul_destroy(h)
    assert total > 0
    assert worst <= 32 * EPS, worst / EPS
    assert (se / sy) ** 0.5 <= 4 * EPS, (se / sy) ** 0.5 / EPS
    return info[0], spectrum_ms


RAGGED = [4096, 0, 1, 4095, 3, 9000, 65536, 777, 65536, 2, 30000]


@pytest.mark.parametrize("src,dst,tb,atten,ext,log2,block_exact", [
    (11025.0, 8000.0, 0.5, 218.0, 0, 16, False),       # 2x on the zero-stuffed view
    (48000.0, 32000.0, 0.5, 180.15, 0, 16, False),     # 2/3 on the zero-stuffed view
    (48000.0, 6003.0, 0.5, 218.0, 0, None, False),     # 1x, the longest half support (lg 6813)
    (48000.0, 16000.0, 0.5, 180.15, 0, None, False),   # 1/3
    (96000.0, 48000.0, 0.5, 180.15, 1, None, True),    # reference-exact 1/2
    (64000.0, 48000.0, 0.5, 218.0, 1, 16, True),       # reference-exact 3/4 on 65536-point blocks
])
def test_large_tile_stage_against_the_reference(emul, src, dst, tb, atten, ext, log2, block_exact):
    _run(emul, src, dst, 65536, tb, atten, ext, RAGGED, want_log2=log2, want_block_exact=block_exact)


def test_spectrum_of_the_largest_plan_is_built_in_reasonable_time(emul):
    """build_spectrum_large at M = 65536 for the longest kernel: half the bins, symmetric taps, one cosine sum each."""
    a = (C.c_double * 6)()
    in_max = emul.bclemul_find(64000.0, 48000.0, 65536, 0.5, 218.0, 1, a)
    h = emul.bclemul_create(a, in_max, 1)
    info = (C.c_int * 4)()
    ms = emul.bclemul_info(h, info)
    emul.bclemul_destroy(h)
    assert info[0] == 16
    assert ms < 20000.0, ms
