"""One-bit DSD output on the host (no GPU): the modulator r8bgpu_dsd_modulate_host, which a batch with DSD output on runs
on the device, against a restatement of the recursion in include/r8bgpu.h written from that text alone, its noise
shaping and overload behaviour at 2.8224 MHz, and a round trip 44100 -> DSD64 -> 44100 through the reference resampler.
"""
import numpy as np
import pytest
from scipy.signal import windows

FS = 2822400
# the loop filter's coefficients as include/r8bgpu.h lists them (17 significant digits: the exact doubles)
G = [-0.52235343612653207, 3.000835998986414, -7.1916327798335757, 9.2026607872978481, -6.631444183027881,
     2.5513679570436851, -0.40943457836890584]
A = [-6.4737547313163422, 17.979709100302625, -27.769461679678152, 25.758433672213886, -14.349100916261154,
     4.4447402103991882, -0.59056542163109382]


def restate(y, scale=1.0, state=None):
    """The header's steps 1-5, one output at a time (Python floats: IEEE doubles, no FMA).  Returns (bits, state, ov)."""
    ep, p = (0.0, [0.0] * 7) if state is None else (state[0], list(state[1:]))
    bits = np.zeros(len(y), dtype=np.uint8)
    ov = 0
    for i, yi in enumerate(np.asarray(y, dtype=np.float64).tolist()):
        v = yi * scale
        if not np.isfinite(v):
            v = 0.0
        v = min(max(v, -0.5), 0.5)
        u = G[0] * ep + (v + p[0])
        bit = u >= 0.0
        bits[i] = bit
        if not abs(u) <= 4.0:
            ep, p = 0.0, [0.0] * 7
            ov += 1
            continue
        e = (1.0 if bit else -1.0) - u
        f = G[0] * ep + p[0]
        r = [None] + [G[k] * ep + p[k] for k in range(1, 7)]
        p = [r[k + 1] + (-A[k]) * f for k in range(6)] + [(-A[6]) * f]
        ep = e
    return bits, [ep] + p, ov


def sine(f, amp, n, fs=FS):
    return amp * np.sin(2 * np.pi * f * np.arange(n) / fs)


def test_host_modulator_matches_contract(pkg):
    rng = np.random.default_rng(11)
    n = 50000
    y = np.concatenate([
        sine(997.0, 0.5, n // 5),
        rng.uniform(-0.5, 0.5, n // 5),
        np.zeros(n // 5),
        sine(3000.0, 0.9, n // 5),  # beyond 0.5: clamped
        rng.uniform(-0.3, 0.3, n // 5)])
    y[n // 5 + 17::997] = np.nan
    y[3 * n // 5 + 5::1511] = np.inf
    y[3 * n // 5 + 9::1709] = -np.inf
    y[4 * n // 5 + 3::2003] = 1e300
    for scale in (1.0, 0.5):
        ref, ref_state, ref_ov = restate(y, scale)
        # the same stream in two host calls, the state carried between them
        st = np.zeros(8)
        b1, o1 = pkg.dsd_modulate(y[:20011], scale, st)
        b2, o2 = pkg.dsd_modulate(y[20011:], scale, st)
        np.testing.assert_array_equal(np.concatenate([b1, b2]), ref)
        assert st.tolist() == ref_state
        assert o1 + o2 == ref_ov == 0


def test_overload_resets_the_filter(pkg):
    # a state far outside what the loop reaches: the first output overloads, and then the recursion starts from zeros
    y = sine(997.0, 0.4, 4000)
    st = np.array([50.0] + [-30.0] * 7)
    bits, ov = pkg.dsd_modulate(y, 1.0, st.copy())
    ref, _, ref_ov = restate(y, 1.0, st.tolist())
    assert ov == ref_ov >= 1
    np.testing.assert_array_equal(bits, ref)
    clean, _ = pkg.dsd_modulate(y[1:], 1.0)
    np.testing.assert_array_equal(bits[1:], clean)


def band_spectrum(bits):
    """Power spectrum of the +-1 stream (a sine of amplitude A shows A^2 in its bins), 20 Hz .. 20 kHz mask."""
    x = bits.astype(np.float64) * 2.0 - 1.0
    w = windows.blackmanharris(len(x))
    X = np.abs(np.fft.rfft(x * w)) ** 2 / np.sum(w) ** 2 * 4.0
    f = np.arange(len(X)) * FS / len(x)
    return f, X, (f >= 20.0) & (f <= 20000.0)


def test_sine_snr(pkg):
    bits, ov = pkg.dsd_modulate(sine(997.0, 0.5, 2 * FS))
    f, X, band = band_spectrum(bits)
    sig = np.abs(f - 997.0) < 20.0
    snr = 10 * np.log10(X[sig].sum() / X[band & ~sig].sum())
    assert ov == 0
    assert snr >= 110.0, snr  # measured 115.4 dB


def test_silence_has_no_tones(pkg):
    ref_bits, _ = pkg.dsd_modulate(sine(997.0, 0.5, 2 * FS))
    f, X, band = band_spectrum(ref_bits)
    s = X[np.abs(f - 997.0) < 20.0].sum()
    bits, ov = pkg.dsd_modulate(np.zeros(2 * FS))
    _, Z, _ = band_spectrum(bits)
    worst = 10 * np.log10(Z[band].max() / s)
    assert ov == 0
    assert worst < -140.0, worst  # measured -154.5 dB


@pytest.mark.parametrize("kind", ["sine20", "sine997", "sine10k", "square", "noise", "clamped"])
def test_no_overloads(pkg, kind):
    n = FS + FS // 2
    rng = np.random.default_rng(3)
    y = {"sine20": lambda: sine(20.0, 0.5, n), "sine997": lambda: sine(997.0, 0.5, n),
         "sine10k": lambda: sine(10000.0, 0.5, n),
         "square": lambda: np.where(np.sin(2 * np.pi * 997.0 * np.arange(n) / FS) >= 0, 0.5, -0.5),
         "noise": lambda: rng.uniform(-0.5, 0.5, n),
         "clamped": lambda: np.concatenate([sine(997.0, 3.0, n // 2), np.where(rng.uniform(size=n - n // 2) < 0.5, 8.0, -8.0)])}[kind]()
    _, ov = pkg.dsd_modulate(y)
    assert ov == 0


def test_round_trip_through_the_reference(pkg, ref):
    """44100 sine -> reference CDSPResampler24 to 2822400 -> modulator (scale 0.5) -> bits as +-2 -> reference back to
    44100: the sine again, in band, away from the ends."""
    n = 44100 * 2
    x = sine(997.0, 0.9, n, 44100)
    up = ref.Resampler(44100.0, 2822400.0, n, 2.0, pkg.ATTEN_24).process(x)
    bits, ov = pkg.dsd_modulate(up, 0.5)
    assert ov == 0
    back = ref.Resampler(2822400.0, 44100.0, len(up), 2.0, pkg.ATTEN_24).process(bits.astype(np.float64) * 4.0 - 2.0)
    # both resamplers remove their own latency: the output lines up with the input
    seg = slice(22050, 44100)
    r = back[seg]
    snr = 10 * np.log10(np.dot(x[seg], x[seg]) / np.dot(r - x[seg], r - x[seg]))
    assert snr >= 100.0, snr  # measured 104.0 dB
