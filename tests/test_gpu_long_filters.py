"""GPU: low-pass kernels too long for one CTA's tile -- transition bands down to 0.5 % at every attenuation -- on the
large-tile BlockConvolver (k_bcl_gather / k_bcl_conv / k_bcl_scatter, 16384 .. 65536-point tiles), against the compiled
reference with the same call chunking."""
import numpy as np
import pytest

import oracle_util as ou

pytestmark = pytest.mark.gpu

LARGE = "k_bcl_gather+k_bcl_conv+k_bcl_scatter"
RAGGED = [4096, 0, 1, 65536, 3, 9000, 1, 0, 65536, 777, 30000]


def _oracle(ext):
    flavor = "e1" if ext else "e0"
    if not ou.have_ref(flavor):
        pytest.skip("oracle/_ref not built (needs /root/reference at build time)")
    return ou.RefOracle(flavor)


def _parity(pkg, src, dst, tb, atten, ext, n_ch, lens, max_in, seed=5, check=None, allow_empty=False):
    ref = _oracle(ext)
    rb = pkg.ResamplerBatch(n_ch, src, dst, max_in, tb, atten, device=0, extfft=ext)
    kernels = [k for k, _ in rb.batch.stage_kernels()]
    check = range(n_ch) if check is None else check
    rs = {c: ref.Resampler(src, dst, max_in, tb, atten) for c in check}
    x = ou.white_noise(n_ch, sum(lens), seed)
    got, want = {c: [] for c in check}, {c: [] for c in check}
    pos = 0
    for l in lens:
        y = rb.process(x[:, pos:pos + l])
        for c in check:
            r = rs[c].process(x[c, pos:pos + l])
            assert len(r) == y.shape[1], (src, dst, tb, atten, ext, l, len(r), y.shape[1])
            got[c].append(y[c])
            want[c].append(r)
        pos += l
    for c in check:
        a, b = np.concatenate(got[c]), np.concatenate(want[c])
        if allow_empty and (len(b) == 0 or not np.any(b)):  # a deep chain still inside its start-up latency
            assert not np.any(a)
            continue
        assert len(b) > 0 and np.any(b)
        m, r = ou.parity_metrics(a, b)
        assert m <= 32 * ou.EPS and r <= 4 * ou.EPS, (src, dst, tb, atten, ext, c, m / ou.EPS, r / ou.EPS)
    return kernels


@pytest.mark.parametrize("src,dst,tb,atten,ext", [
    (11025.0, 8000.0, 0.5, 218.0, 0),      # 2x on the zero-stuffed view -> whole-stepping interpolator
    (48000.0, 32000.0, 0.5, 180.15, 0),    # 2/3 on the zero-stuffed view
    (48000.0, 6003.0, 0.5, 218.0, 0),      # 1x, half support 6813
    (48000.0, 16000.0, 0.5, 180.15, 0),    # 1/3
    (96000.0, 48000.0, 0.5, 180.15, 1),    # reference-exact 1/2
    (64000.0, 48000.0, 0.5, 218.0, 1),     # reference-exact 3/4 on 65536-point blocks
    (8000.0, 96000.0, 0.5, 180.15, 0),     # 3x -> 2 x HBUp
    (44100.0, 8000.0, 0.5, 218.0, 0),      # HBDown -> long 1x -> interpolator
])
def test_long_filter_chains(pkg, src, dst, tb, atten, ext):
    kernels = _parity(pkg, src, dst, tb, atten, ext, 3, RAGGED, 65536)
    assert LARGE in kernels, kernels


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_narrow_transition_bands_are_never_refused(pkg, seed):
    rates = [8000.0, 11025.0, 16000.0, 22050.0, 32000.0, 44100.0, 48000.0, 64000.0, 88200.0, 96000.0, 176400.0,
             192000.0, 352800.0, 384000.0]
    rng = np.random.default_rng(1000 + seed)
    done = 0
    while done < 5:
        a, b = (float(v) for v in rng.choice(rates, 2, replace=False))
        if rng.random() < 0.25:
            b += float(rng.integers(1, 50))
        if a / b > 40 or b / a > 40:
            continue
        tb = float(rng.choice([0.5, 0.75, 1.0]))
        atten = float(rng.choice([pkg.ATTEN_16IR, pkg.ATTEN_16, pkg.ATTEN_24, 206.91]))
        ext = int(rng.integers(0, 2))
        max_in = int(rng.choice([512, 2048, 6000]))
        n_calls = 12 if a <= 4 * b else 40
        lens = [int(v) for v in rng.integers(0, max_in + 1, n_calls)] + [max_in, 1, 0, max_in]
        _parity(pkg, a, b, tb, atten, ext, 2, lens, max_in, seed=seed * 100 + done, allow_empty=True)
        done += 1


def test_channel_groups_share_the_scratch(pkg, monkeypatch):
    # a 1 MB scratch holds one channel's tile pair of 65536 points: the three kernels run once per channel
    monkeypatch.setenv("R8BGPU_BCL_SCRATCH_MB", "1")
    kernels = _parity(pkg, 48000.0, 16000.0, 0.5, 180.15, 0, 5, [65536, 1, 4000, 65536], 65536)
    assert LARGE in kernels


def test_int24_in_float32_out(pkg):
    src, dst, tb, atten, n_ch, l = 48000.0, 6003.0, 0.5, 218.0, 3, 65536
    rng = np.random.default_rng(21)
    a = pkg.ResamplerBatch(n_ch, src, dst, l, tb, atten, device=0)
    b = pkg.ResamplerBatch(n_ch, src, dst, l, tb, atten, device=0)
    for _ in range(2):
        v = rng.integers(-(1 << 23), 1 << 23, size=(n_ch, l), dtype=np.int32)
        raw = np.stack([v & 0xff, (v >> 8) & 0xff, (v >> 16) & 0xff], axis=-1).astype(np.uint8)
        y = a.batch.process_host_fmt(raw, fmt=pkg.S24, out_dtype=np.float32, in_scale=2.0 ** -23)
        want = b.process(v.astype(np.float64) * 2.0 ** -23).astype(np.float32)
        assert y.shape == want.shape
        assert np.array_equal(y, want)
