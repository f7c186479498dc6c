"""CPU: phase C of the flagship kernel on the filter spectrum's symmetric half-size form, without a GPU.

k_up2_frac2 keeps the 2x pair's filter spectrum in shared memory as the pairs (a0[k], a1[k]), k = 0..2048
(csrc/r8b_fused2_core.cuh, cs_entry / cd1s_compute), where the plan has room for them beside its phase-group bank.
tests/cpp/fused2_sym_emul.cpp runs the kernel's per-thread functions with that table on the host.  Checked here:
* every bin of G rebuilt from the table with the kernel's own arithmetic equals build_spectrum()'s table within 2 ulp of
  max |G|, over the presets, transition bands 0.5-45 % and the four attenuations;
* the table's index algebra: every bin is read exactly where it is stored, and both reads of a warp are conflict-free;
* the whole kernel emulated with the new phase C against the oracle (cfg 2, cfg 3, a ragged sweep);
* the per-plan shared-memory decision over the rate pairs, transition bands and attenuations of the tile-choice sweep.
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
PRESET_ATTENS = [136.45, 180.15, 206.91, 218.0]   # CDSPResampler16 / 24 / 24 at 0.5 % ... and the reference's maximum

FN, HT, CS_PAIRS = 2048, 256, 2049
# dynamic shared memory of k_up2_frac2 (bytes): 2 padded tile buffers, [q][r] twiddles, the bank, the spectrum pairs
TILE_BUFS, TWIDDLES, SMEM_MAX = 2 * (4096 + 256 + 16) * 16, 512 * 16, 227 * 1024 - 1024


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
    so = str(tmp_path_factory.mktemp("f2semul") / "libf2semul.so")
    srcs = [os.path.join(HERE, "cpp", "fused2_sym_emul.cpp")] + [os.path.join(CSRC, f) for f in
                                                                 ("r8b_plan.cpp", "r8b_design.cpp", "r8b_hosttab.cpp")]
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + inc, "-o", so] + srcs, check=True)
    L = C.CDLL(so)
    L.f2semul_create.restype = C.c_void_p
    L.f2semul_create.argtypes = [C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_int]
    L.f2semul_process.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    L.f2semul_destroy.argtypes = [C.c_void_p]
    L.f2semul_table_err.argtypes = [C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_int, C.POINTER(C.c_double)]
    L.f2semul_entries.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.f2semul_fit.argtypes = [C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_int, C.POINTER(C.c_int), C.c_int]
    return L


def _entry(k):
    """Where bin k's pair is stored: thread order [t][16 q1 + q2] for k = q1 + 16 q2 + 256 t, then k = N."""
    if k == FN:
        return FN
    return 256 * (k >> 8) + 16 * (k & 15) + ((k >> 4) & 15)


def test_rebuilt_bins_match_the_full_spectrum(emul):
    out = (C.c_double * 1)()
    worst, n = 0.0, 0
    for (src, dst), tb, atten in itertools.product([(44100.0, 96000.0), (48000.0, 44100.0), (44100.0, 48000.0),
                                                   (22050.0, 48000.0), (48000.0, 88200.0)],
                                                  [0.5, 1.0, 2.0, 3.0, 7.5, 20.0, 45.0], PRESET_ATTENS):
        k = emul.f2semul_table_err(src, dst, 4096, tb, atten, 0, out)
        assert k >= 0, (src, dst, tb, atten)
        if k:
            assert out[0] <= 2.0, (src, dst, tb, atten, out[0])
            worst = max(worst, out[0])
            n += k
    assert n >= 60, n


def test_table_index_algebra(emul):
    first, second = (C.c_int * HT)(), (C.c_int * HT)()
    emul.f2semul_entries(first, second)
    seen = np.zeros(CS_PAIRS, dtype=int)
    for g in range(HT):
        q1, q2 = g >> 4, g & 15
        for t in range(8):
            kap = q1 + 16 * q2 + 256 * t
            assert first[g] + 256 * t == _entry(kap), (g, t)
            assert second[g] - 256 * t == _entry(FN - kap), (g, t)
            seen[_entry(kap)] += 1
            seen[_entry(FN - kap)] += 1
    # every pair is read: k = 0 and N once each from both sides' special lanes, the rest once as kappa, once as N - kappa
    assert np.all(seen >= 1) and seen.sum() == 2 * 8 * HT
    # 16-byte loads: a quarter-warp (8 lanes) is one wavefront when its 8 entries sit on 8 different 16-byte bank groups
    for w in range(HT // 32):
        for t in range(8):
            for qw in range(4):
                lanes = range(32 * w + 8 * qw, 32 * w + 8 * qw + 8)
                assert len({(first[g] + 256 * t) % 8 for g in lanes}) == 8, (w, t, qw)
                assert len({(second[g] - 256 * t) % 8 for g in lanes}) == 8, (w, t, qw)
            # and a warp's 32 reads of each kind lie in one 512-byte run, except warp 0's q1 = 0 lanes
            s = sorted(second[g] - 256 * t for g in range(32 * w, 32 * w + 32) if w > 0)
            if s:
                assert s[-1] - s[0] == 31, (w, t)


def _run(L, src, dst, max_len, lens, glog=-1, atten=180.15, tb=2.0, seed=7):
    ref = oracle_util.best_oracle()
    h = L.f2semul_create(src, dst, max_len, tb, atten, glog)
    assert h, "rate pair does not plan to BlockConv(2x) -> whole-stepping interpolator"
    rs = ref.Resampler(src, dst, max_len, tb, atten)
    rng = np.random.default_rng(seed)
    worst = se = sy = 0.0
    total = 0
    for n in lens:
        x = rng.uniform(-1.0, 1.0, n)
        out = np.zeros(int(n * dst / src * 1.25) + 4096)
        k = L.f2semul_process(h, x.ctypes.data, n, out.ctypes.data, len(out))
        yr = rs.process(x)
        assert k == len(yr), (k, len(yr))
        if k:
            d = out[:k] - yr
            worst = max(worst, float(np.max(np.abs(d))) / float(np.max(np.abs(yr))))
            se += float(np.sum(d * d))
            sy += float(np.sum(yr * yr))
            total += k
    L.f2semul_destroy(h)
    assert total > 0
    assert worst <= 32 * EPS, worst / EPS
    assert (se / sy) ** 0.5 <= 4 * EPS, (se / sy) ** 0.5 / EPS


@pytest.mark.parametrize("glog", [0, 8])
def test_cfg2_chain(emul, glog):
    _run(emul, 44100.0, 96000.0, 8192, [8192, 8192, 8192], glog=glog)


@pytest.mark.parametrize("glog", [-1, 8])
def test_cfg3_chain_padded_y_layout(emul, glog):
    _run(emul, 48000.0, 44100.0, 8191, [8191, 8191, 4000], glog=glog)


def test_ragged_blocks_history_ring_and_misaligned_rows(emul):
    _run(emul, 44100.0, 96000.0, 8192, [1, 0, 4097, 777, 8192, 3, 8191, 5000], glog=8)


def test_seeded_sweep_of_rate_pairs_presets_and_ragged_calls(emul):
    rng = np.random.default_rng(9191)
    pairs = [(44100.0, 96000.0), (48000.0, 44100.0), (44100.0, 48000.0), (32000.0, 44100.0), (48000.0, 88200.0),
             (88200.0, 48000.0), (44100.0, 64000.0), (22050.0, 32000.0)]
    done = 0
    for src, dst in pairs:
        att = float(rng.choice(PRESET_ATTENS[:3]))
        tb = float(rng.choice([2.0, 3.0, 6.0]))
        max_len = int(rng.choice([2048, 4096, 8192]))
        lens = [max_len, max_len] + [int(v) for v in rng.integers(0, max_len + 1, 4)] + [max_len]
        glog = int(rng.choice([-1, 8]))
        h = emul.f2semul_create(src, dst, max_len, tb, att, glog)
        if not h:
            continue
        emul.f2semul_destroy(h)
        _run(emul, src, dst, max_len, lens, glog=glog, atten=att, tb=tb, seed=int(rng.integers(1 << 30)))
        done += 1
    assert done >= 5, done


def test_shared_memory_fit_decision(emul):
    buf = (C.c_int * 80)()
    n_plans = n_stages = n_fit = 0
    for (src, dst), tb, atten, ext in itertools.product(itertools.permutations(RATES, 2), TBS, ATTENS, (0, 1)):
        if src / dst > 40 or dst / src > 40:
            continue
        n = emul.f2semul_fit(src, dst, 4096, tb, atten, ext, buf, 20)
        assert 0 <= n <= 20, (src, dst, tb, atten, ext)
        n_plans += 1
        for i in range(n):
            kind, bank, fits, smem = buf[4 * i:4 * i + 4]
            cfg = (src, dst, tb, atten, ext, i)
            assert kind in (1, 2) and bank >= 0, cfg
            if kind == 2:
                assert bank == 0, cfg
            want = TILE_BUFS + TWIDDLES + ((bank + 1) & ~1) * 8 + CS_PAIRS * 16
            assert smem == want, cfg
            assert fits == int(want <= SMEM_MAX), cfg
            n_stages += 1
            n_fit += fits
    assert n_plans > 10000 and n_stages > 1000 and n_fit > 0, (n_plans, n_stages, n_fit)
    # the flagship keeps its spectrum on chip; 48000->44100 does not (its 10-phase FMA bank, 6600 doubles, leaves no room)
    assert emul.f2semul_fit(44100.0, 96000.0, 65536, 2.0, 180.15, 0, buf, 20) == 1
    assert buf[0] == 1 and buf[2] == 1, list(buf[:4])
    assert emul.f2semul_fit(48000.0, 44100.0, 65536, 2.0, 180.15, 0, buf, 20) == 1
    assert buf[0] == 1 and buf[1] == 6600 and buf[2] == 0, list(buf[:4])
