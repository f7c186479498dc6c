"""Dithered integer output on the host (no GPU): the quantiser r8bgpu_dither_quantize_host, which a batch runs on the
device, against a numpy restatement of the contract in include/r8bgpu.h written from that text alone, and its statistics.
"""
import numpy as np
import pytest

RANGE = {2: (-32768, 32767), 3: (-8388608, 8388607), 4: (-2147483648, 2147483647)}


def tpdf(seed, n):
    """d for output indices n (int64 array): SplitMix64 on seed + (n + 1) * gamma, mod 2^64 (numpy wraps uint64)."""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + (np.asarray(n, dtype=np.uint64) + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
        z = z ^ (z >> np.uint64(30))
        z = z * np.uint64(0xBF58476D1CE4E5B9)
        z = z ^ (z >> np.uint64(27))
        z = z * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(32)).astype(np.float64) * 2.0 ** -32 - (z & np.uint64(0xFFFFFFFF)).astype(np.float64) * 2.0 ** -32


def restate(y, fmt, seed, taps=(), scale=1.0, first=0, hist=None):
    """The contract, one sample at a time.  hist: e[first-1], e[first-2], ... (newest first); returns (ints, hist)."""
    lo, hi = RANGE[fmt]
    taps = [float(t) for t in taps]
    K = len(taps)
    e = list(hist) if hist is not None else [0.0] * 16
    d = tpdf(seed, np.arange(first, first + len(y), dtype=np.int64))
    out = np.zeros(len(y), dtype=np.int64)
    for i, yi in enumerate(np.asarray(y, dtype=np.float64)):
        v = np.float64(yi) * np.float64(scale)
        if not np.isfinite(v):
            out[i] = 0 if np.isnan(v) else (hi if v > 0 else lo)
            e.insert(0, 0.0)
        else:
            s = np.float64(0.0)
            for k in range(K, 0, -1):
                s = s + np.float64(taps[k - 1]) * np.float64(e[k - 1])
            w = v - s
            q = np.rint(w + d[i])
            e.insert(0, float(q - w))
            out[i] = int(min(max(q, lo), hi))
        del e[16:]
    return out, e


def as_ints(q, fmt):
    if fmt == 3:
        b = q.astype(np.int32)
        v = b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)
        return np.where(v >= 1 << 23, v - (1 << 24), v).astype(np.int64)
    return q.astype(np.int64)


def signal(rng, n, fmt, scale=1.0):
    lo, hi = RANGE[fmt]
    y = rng.uniform(-6, 6, n) + np.sin(np.arange(n) * 0.01) * 40.0
    y[::97] = rng.uniform(lo * 1.5, hi * 1.5, len(y[::97]))  # at and beyond full scale
    y[5], y[11], y[17], y[23] = hi + 0.5, lo - 0.5, hi, lo
    y[31], y[37], y[41] = np.nan, np.inf, -np.inf
    return y / scale


TAPS = {0: [], 1: [1.0], 9: [2.033, -2.165, 1.959, -1.590, 0.6149, -0.2, 0.1, -0.05, 0.01],
        16: list(np.random.default_rng(7).uniform(-0.6, 0.6, 16))}


@pytest.mark.parametrize("fmt", [2, 3, 4])
@pytest.mark.parametrize("K", [0, 1, 9, 16])
@pytest.mark.parametrize("scale", [1.0, 32767.0])
def test_host_quantiser_matches_contract(pkg, fmt, K, scale):
    rng = np.random.default_rng(fmt * 100 + K)
    y = signal(rng, 3000, fmt, scale)
    seed = 0xDEADBEEF12345678 + K
    ref, _ = restate(y, fmt, seed, TAPS[K], scale, first=12345)
    q, _ = pkg.dither_quantize(y, fmt, seed, TAPS[K], scale=scale, first_index=12345)
    np.testing.assert_array_equal(as_ints(q, fmt), ref)


@pytest.mark.parametrize("K", [0, 9, 16])
def test_split_blocks_carry_state(pkg, K):
    rng = np.random.default_rng(K)
    y = signal(rng, 5000, 2)
    whole, st_whole = pkg.dither_quantize(y, pkg.S16, 99, TAPS[K])
    cuts = np.sort(rng.choice(np.arange(1, len(y)), 12, replace=False))
    st = np.zeros(16)
    parts = []
    for a, b in zip(np.r_[0, cuts], np.r_[cuts, len(y)]):
        q, st = pkg.dither_quantize(y[a:b], pkg.S16, 99, TAPS[K], first_index=int(a), state=st)
        parts.append(q)
    np.testing.assert_array_equal(np.concatenate(parts), whole)
    np.testing.assert_array_equal(st, st_whole)


def test_off_is_the_cast(pkg):
    y = np.array([0.9, -0.9, 1.5, -1.5, 40000.0, -40000.0, np.nan, np.inf, -np.inf, 32766.99])
    q, st = pkg.dither_quantize(y, pkg.S16, 5, kind=pkg.DITHER_OFF)
    np.testing.assert_array_equal(q, [0, 0, 1, -1, 32767, -32768, 0, 32767, -32768, 32766])
    assert not st.any()


def test_noise_statistics():
    d = tpdf(0x1234, np.arange(1 << 20, dtype=np.int64))
    assert abs(d.mean()) < 2e-3
    assert abs(d.var() - 1.0 / 6.0) < 2e-3
    assert d.min() > -1.0 and d.max() < 1.0


def test_flat_tpdf_is_unbiased_where_the_cast_is_not(pkg):
    v = np.linspace(-4.0, 4.0, 1 << 18)
    q, _ = pkg.dither_quantize(v, pkg.S32, 42)
    err = q.astype(np.float64) - v
    bins = np.minimum(((v + 4.0) * 2.0).astype(int), 15)  # 16 bins of half an LSB
    for b in np.unique(bins):
        m = bins == b
        assert abs(err[m].mean()) < 0.02, b
        assert abs(err[m].var() - 0.25) < 0.03, b
    qc, _ = pkg.dither_quantize(v, pkg.S32, 42, kind=pkg.DITHER_OFF)
    ec = qc.astype(np.float64) - v
    assert ec[v > 1].mean() < -0.4 and ec[v < -1].mean() > 0.4  # truncation toward zero


def test_first_order_shaping_moves_error_up(pkg):
    rng = np.random.default_rng(3)
    v = rng.uniform(-100, 100, 1 << 16)
    q, _ = pkg.dither_quantize(v, pkg.S32, 8, taps=[1.0])
    p = np.abs(np.fft.rfft(q - v)) ** 2
    half = len(p) // 2
    assert p[half:].sum() > 3.0 * p[:half].sum()


@pytest.mark.parametrize("cfg,msg", [
    (dict(kind=7), "unknown kind"),
    (dict(taps=[0.1] * 17), "n_taps"),
    (dict(taps=[0.5], kind=0), "taps with kind OFF"),
    (dict(taps=[float("nan")]), "not finite"),
])
def test_host_refusals(pkg, cfg, msg):
    with pytest.raises(pkg.R8bGpuError) as ei:
        pkg.dither_quantize(np.zeros(4), pkg.S16, 1, **cfg)
    assert msg in str(ei.value)
    with pytest.raises(pkg.R8bGpuError):
        pkg.dither_quantize(np.zeros(4), pkg.F32, 1)


def test_symbols_bound(pkg):
    for name in ("r8bgpu_batch_set_dither", "r8bgpu_dither_quantize_host"):
        assert name in pkg._SYMBOLS
        getattr(pkg.lib(), name)


def test_history_kept_across_a_gap(pkg):
    """Outputs the channel does not dither (float-output calls, OFF) leave its error history as it was: e[n-k] is the
    error of its k-th most recent dithered output, across the gap in the output index."""
    rng = np.random.default_rng(11)
    a, b = signal(rng, 1000, 2)[50:], rng.uniform(-30, 30, 777)
    qa, st = pkg.dither_quantize(a, pkg.S16, 5, TAPS[9])
    ra, hist = restate(a, 2, 5, TAPS[9])
    gap = len(a) + 37  # 37 outputs went out undithered in between
    qb, _ = pkg.dither_quantize(b, pkg.S16, 5, TAPS[9], first_index=gap, state=st)
    rb, _ = restate(b, 2, 5, TAPS[9], first=gap, hist=hist)
    np.testing.assert_array_equal(qa, ra)
    np.testing.assert_array_equal(qb, rb)


def test_library_noise_is_triangular(pkg):
    """The pinned function on silence: q = rint(d), so P(q = +1) = P(q = -1) = P(d > 1/2) = 1/8 for a triangular d on
    (-1, 1) (1/4 for a uniform one), and the mean of q is 0."""
    q, _ = pkg.dither_quantize(np.zeros(1 << 20), pkg.S32, 0xABCDEF)
    p_up, p_dn = np.mean(q == 1), np.mean(q == -1)
    assert abs(p_up - 0.125) < 2e-3 and abs(p_dn - 0.125) < 2e-3
    assert abs(q.mean()) < 2e-3 and np.all(np.abs(q) <= 1)
