"""One-bit DSD input on the device: DSF (LSB-first) and DSDIFF (MSB-first) byte buffers resampled to PCM.

- Decoding is exact: every form of call fed DSD bytes gives, bit for bit, what the plain fp64 path gives when fed the
  bits as +-scale, on chains that start with k_hbdown, with k_hbdown_cascade, with a BlockConvolver (conversion launch),
  and on a passthrough plan.
- The in-kernel E/O split follows the absolute sample index (streams whose position is odd when DSD calls begin), and
  R8BGPU_NO_FORMAT_FUSION (a conversion launch instead) changes no bit.
- Planar lock-step calls on half-band-first chains make no extra launch.
- DSD_MSB on bit-reversed bytes is DSD_LSB; refusals change nothing; a sigma-delta-modulated tone comes out clean; one
  chain against the reference.
The layout itself is pinned to np.unpackbits in test_dsd_cpu.py.
"""
import numpy as np
import pytest

import oracle_util as ou

pytestmark = pytest.mark.gpu

F64, DSD_LSB, DSD_MSB = 0, 16, 17
CHAINS = [(2822400.0, 705600.0),    # k_hbdown first (one half-band stage, then a BlockConvolver)
          (2822400.0, 352800.0),    # a cascade of 2
          (2822400.0, 44100.0),     # cascade + BlockConvolver
          (2822400.0, 48000.0),     # third-band tables: cascade + BlockConvolver + interpolator
          (2822400.0, 1411200.0),   # BlockConvolver first: conversion launch
          (2822400.0, 2822400.0),   # passthrough
          (11289600.0, 44100.0)]    # cascade of 6 feeding k_hbdown
IDS = ["%g-%g" % c for c in CHAINS]


def pack(bits, msb=False):
    """bits [..., l] of 0/1 -> DSD bytes [..., l / 8] (np.packbits packs along the last axis)."""
    return np.packbits(np.asarray(bits, dtype=np.uint8), axis=-1, bitorder="big" if msb else "little")


def values(bits, scale):
    return np.where(np.asarray(bits) != 0, scale, -scale).astype(np.float64)


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(a):
    return a if isinstance(a, np.ndarray) else a.cpu().numpy()


def _plan(pkg, chain, M):
    return pkg.Plan(chain[0], chain[1], M, 2.0, pkg.ATTEN_24)


def _block(chain):
    """(MaxInLen, calls): enough input to get well past the latency (~109 K samples of DSD64 -> 44100)."""
    return (65536, 7) if chain[0] > 3e6 else (32768, 5)


def _lockstep(pkg, b, byt, fmt, l, scale, form):
    """One lock-step call on planar bytes [n_ch, l/8]; form: host, host_il, dev, dev_il.  Returns planar fp64."""
    il = form.endswith("_il")
    if form.startswith("host"):
        y = b.process_host_fmt(byt.T.copy() if il else byt, fmt=fmt, out_fmt=F64, in_scale=scale, interleaved=il)
        return y.T if il else y
    import torch
    n_ch = byt.shape[0]
    xin = _dev(byt.T.copy() if il else byt)
    cap = max(b.plan.max_out_len, 1)
    yo = torch.zeros((n_ch, cap), dtype=torch.float64, device="cuda")
    b.set_stream(torch.cuda.current_stream().cuda_stream)
    n = b.process_fmt(pkg.Buffer.make(xin.data_ptr(), fmt, il, n_ch if il else byt.shape[1], scale), l,
                      pkg.Buffer.make(yo.data_ptr(), F64, False, cap), cap, host=False)
    torch.cuda.synchronize()
    return yo[:, :n].cpu().numpy()


# ---- 1. bit-identity with the fp64 path ----------------------------------------------------------------------------

@pytest.mark.parametrize("scale", [1.0, 0.5])
@pytest.mark.parametrize("chain", CHAINS, ids=IDS)
def test_lockstep_matches_fp64(pkg, chain, scale):
    n_ch = 3
    M, calls = _block(chain)
    plan = _plan(pkg, chain, M)
    for form in ("host", "host_il", "dev", "dev_il"):
        rng = np.random.default_rng([CHAINS.index(chain), int(scale * 2), len(form)])
        b, twin = pkg.Batch(plan, n_ch), pkg.Batch(plan, n_ch)
        for k in range(calls):
            l = M if k % 3 != 1 else M // 2 + 8
            bits = rng.integers(0, 2, (n_ch, l))
            y = _lockstep(pkg, b, pack(bits), DSD_LSB, l, scale, form)
            yt = twin.process_host(values(bits, scale))
            np.testing.assert_array_equal(y, yt, err_msg=f"{form} call {k}")


@pytest.mark.parametrize("chain", CHAINS, ids=IDS)
def test_ragged_matches_fp64(pkg, chain):
    n_ch, scale = 4, 0.5
    M, calls = _block(chain)
    plan = _plan(pkg, chain, M)
    for form in ("host", "host_il", "dev", "dev_il"):
        rng = np.random.default_rng([7, CHAINS.index(chain), len(form)])
        b, twin = pkg.Batch(plan, n_ch), pkg.Batch(plan, n_ch)
        il = form.endswith("_il")
        for k in range(calls):
            lens = (rng.integers(0, M // 8 + 1, n_ch) * 8).astype(np.int32)
            lens[k % n_ch] = M
            bits = rng.integers(0, 2, (n_ch, M))
            byt = pack(bits)
            xin = byt.T.copy() if il else byt
            y, cnt = b.process_ragged_fmt(_dev(xin) if form.startswith("dev") else xin, lens, fmt=DSD_LSB, in_scale=scale,
                                          interleaved=il)
            yt, cnt_t = twin.process_ragged_fmt(values(bits, scale), lens)
            y = _np(y)
            np.testing.assert_array_equal(cnt, cnt_t)
            for c in range(n_ch):
                row = y[:cnt[c], c] if il else y[c, :cnt[c]]
                np.testing.assert_array_equal(row, yt[c, :cnt[c]], err_msg=f"{form} call {k} channel {c}")


@pytest.mark.parametrize("device", [False, True])
def test_mixed_dsd64_dsd128(pkg, device):
    M = 32768
    plans = [pkg.Plan(2822400.0, 44100.0, M, 2.0, pkg.ATTEN_24), pkg.Plan(5644800.0, 44100.0, M, 2.0, pkg.ATTEN_24)]
    plan_of = np.array([0, 1, 1, 0, 1], dtype=np.int32)
    mixed = pkg.Batch.mixed(plans, plan_of)
    rows = [np.nonzero(plan_of == p)[0] for p in range(2)]
    ords = [pkg.Batch(plans[p], len(rows[p])) for p in range(2)]
    rng = np.random.default_rng(41)
    for k in range(5):
        lens = (rng.integers(0, M // 8 + 1, len(plan_of)) * 8).astype(np.int32)
        lens[k % len(plan_of)] = M
        bits = rng.integers(0, 2, (len(plan_of), M))
        il = k == 1
        byt = pack(bits, msb=True)
        xin = byt.T.copy() if il else byt
        y, cnt = mixed.process_ragged_fmt(_dev(xin) if device else xin, lens, fmt=DSD_MSB, in_scale=0.5, interleaved=il)
        y = _np(y)
        for p in range(2):
            yo, co = ords[p].process_ragged_fmt(values(bits[rows[p]], 0.5), lens[rows[p]])
            np.testing.assert_array_equal(cnt[rows[p]], co)
            for i, c in enumerate(rows[p]):
                row = y[:cnt[c], c] if il else y[c, :cnt[c]]
                np.testing.assert_array_equal(row, yo[i, :co[i]], err_msg=f"call {k} channel {c}")


def test_device_all_matches_fp64(pkg, monkeypatch):
    monkeypatch.setenv("R8BGPU_FORCE_SHARDS", "2")
    n_ch, M = 5, 32768
    plan = pkg.Plan(2822400.0, 44100.0, M, 2.0, pkg.ATTEN_24)
    b, twin = pkg.Batch(plan, n_ch, pkg.DEVICE_ALL), pkg.Batch(plan, n_ch)
    assert len(b.shards()) == 2
    rng = np.random.default_rng(43)
    for k in range(5):
        bits = rng.integers(0, 2, (n_ch, M))
        il = k % 2 == 1
        byt = pack(bits)
        y = b.process_host_fmt(byt.T.copy() if il else byt, fmt=DSD_LSB, interleaved=il)
        np.testing.assert_array_equal(y.T if il else y, twin.process_host(values(bits, 1.0)), err_msg=f"call {k}")
    lens = (rng.integers(0, M // 8 + 1, n_ch) * 8).astype(np.int32)
    bits = rng.integers(0, 2, (n_ch, M))
    y, cnt = b.process_ragged_fmt(pack(bits).T.copy(), lens, fmt=DSD_LSB, interleaved=True)
    yt, cnt_t = twin.process_ragged_fmt(values(bits, 1.0), lens)
    np.testing.assert_array_equal(cnt, cnt_t)
    for c in range(n_ch):
        np.testing.assert_array_equal(y[:cnt[c], c], yt[c, :cnt[c]])


# ---- 2. absolute parity and the fusion knob -------------------------------------------------------------------------

@pytest.mark.parametrize("chain", [(2822400.0, 705600.0), (2822400.0, 44100.0), (11289600.0, 44100.0)],
                         ids=lambda c: "%g-%g" % c)
def test_odd_stream_position_and_fusion_knob(pkg, chain, monkeypatch):
    n_ch, scale = 3, 0.5
    M, calls = _block(chain)
    plan = _plan(pkg, chain, M)
    rng = np.random.default_rng(47)
    pre = [rng.uniform(-0.5, 0.5, (n_ch, l)) for l in (1001, 333, 7)]  # odd lengths: DSD calls start at odd positions
    blocks = [rng.integers(0, 2, (n_ch, M if k % 2 == 0 else 8 * 37)) for k in range(2 * calls)]
    outs = {}
    for mode in ("fused", "unfused", "fp64"):
        if mode == "unfused":
            monkeypatch.setenv("R8BGPU_NO_FORMAT_FUSION", "1")
        else:
            monkeypatch.delenv("R8BGPU_NO_FORMAT_FUSION", raising=False)
        b = pkg.Batch(plan, n_ch)
        ys = [b.process_host(x) for x in pre]
        for k, bits in enumerate(blocks):
            if mode == "fp64":
                ys.append(b.process_host(values(bits, scale)))
            else:
                ys.append(_lockstep(pkg, b, pack(bits), DSD_LSB, bits.shape[1], scale, "dev" if k % 2 else "host"))
        outs[mode] = np.concatenate(ys, axis=1)
    assert outs["fp64"].shape[1] > 50
    np.testing.assert_array_equal(outs["fused"], outs["fp64"])
    np.testing.assert_array_equal(outs["unfused"], outs["fp64"])


# ---- 3. launch counts ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("chain,extra", [((2822400.0, 705600.0), 0), ((2822400.0, 44100.0), 0), ((11289600.0, 44100.0), 0),
                                         ((2822400.0, 1411200.0), 1)], ids=lambda v: "%g-%g" % v if isinstance(v, tuple) else str(v))
@pytest.mark.parametrize("host", [True, False])
def test_launch_counts(pkg, chain, extra, host):
    n_ch = 4
    M, _ = _block(chain)
    plan = _plan(pkg, chain, M)
    rng = np.random.default_rng(53)
    bits = rng.integers(0, 2, (n_ch, M))
    bf, bd = pkg.Batch(plan, n_ch), pkg.Batch(plan, n_ch)
    bf.process_host(values(bits, 1.0))
    n0 = bd.kernel_launches
    _lockstep(pkg, bd, pack(bits), DSD_LSB, M, 1.0, "host" if host else "dev")
    assert bd.kernel_launches - n0 == bf.kernel_launches + extra, (bd.kernel_launches - n0, bf.kernel_launches)


# ---- 4. bit order --------------------------------------------------------------------------------------------------

def test_msb_on_reversed_bytes_is_lsb(pkg):
    n_ch, M = 3, 32768
    plan = pkg.Plan(2822400.0, 48000.0, M, 2.0, pkg.ATTEN_24)
    rng = np.random.default_rng(59)
    bl, bm = pkg.Batch(plan, n_ch), pkg.Batch(plan, n_ch)
    rev = pack(np.unpackbits(np.arange(256, dtype=np.uint8)[:, None], axis=1, bitorder="little"), msb=True)[:, 0]
    for k in range(4):
        byt = rng.integers(0, 256, (n_ch, M // 8)).astype(np.uint8)
        il = k == 2
        a = bl.process_host_fmt(byt.T.copy() if il else byt, fmt=DSD_LSB, interleaved=il)
        m = bm.process_host_fmt(rev[byt].T.copy() if il else rev[byt], fmt=DSD_MSB, interleaved=il)
        np.testing.assert_array_equal(m, a, err_msg=f"call {k}")


# ---- 5. refusals change nothing ------------------------------------------------------------------------------------

def test_refusals_change_nothing(pkg):
    import torch
    n_ch, M = 3, 32768
    plan = pkg.Plan(2822400.0, 44100.0, M, 2.0, pkg.ATTEN_24)
    b, twin = pkg.Batch(plan, n_ch), pkg.Batch(plan, n_ch)
    rng = np.random.default_rng(61)
    cap = max(plan.max_out_len, 1)
    yh = np.zeros((n_ch, cap), dtype=np.uint8)
    yd = torch.zeros((n_ch, cap), dtype=torch.uint8, device="cuda")

    def step():
        bits = rng.integers(0, 2, (n_ch, M))
        np.testing.assert_array_equal(b.process_host_fmt(pack(bits), fmt=DSD_LSB), twin.process_host(values(bits, 1.0)))

    step()
    byt = pack(rng.integers(0, 2, (n_ch, M)))
    xd = _dev(byt)
    lens = np.full(n_ch, M, np.int32)
    counts = np.zeros(n_ch, np.int32)
    for fo in (DSD_LSB, DSD_MSB):
        for host in (True, False):
            src = byt.ctypes.data if host else xd.data_ptr()
            dst = yh.ctypes.data if host else yd.data_ptr()
            with pytest.raises(pkg.R8bGpuError, match="DSD formats are input-only"):
                b.process_fmt(pkg.Buffer.make(src, DSD_LSB, False, M // 8), M, pkg.Buffer.make(dst, fo, False, cap), cap, host=host)
            step()
            with pytest.raises(pkg.R8bGpuError, match="DSD formats are input-only"):
                b.process_ragged_fmt(byt if host else xd, lens, fmt=DSD_LSB, out_fmt=fo)
            step()
            with pytest.raises(pkg.R8bGpuError, match="DSD formats are input-only"):
                b._flush_into(np.arange(n_ch, dtype=np.int32), None, yh if host else yd, fo, False, 1.0, counts)
            step()
        with pytest.raises(pkg.R8bGpuError, match="fmt must be"):
            pkg.dither_quantize(np.zeros(4), fo, 1)
    for host in (True, False):  # lengths that are not a multiple of 8
        with pytest.raises(pkg.R8bGpuError, match="multiples of 8"):
            b.process_fmt(pkg.Buffer.make(byt.ctypes.data if host else xd.data_ptr(), DSD_LSB, False, M // 8), M - 4,
                          pkg.Buffer.make(yh.ctypes.data if host else yd.data_ptr(), F64, False, cap // 8), cap // 8, host=host)
        step()
        bad = lens.copy()
        bad[1] = 1001
        with pytest.raises(pkg.R8bGpuError, match="multiples of 8"):
            b.process_ragged_fmt(byt if host else xd, bad, fmt=DSD_LSB)
        step()


# ---- 6. a real signal ----------------------------------------------------------------------------------------------

def sdm2(u):
    """A 2nd-order 1-bit sigma-delta modulator (two delay-free integrators fed back from the quantiser): bits of u."""
    bits = np.empty(len(u), dtype=np.uint8)
    i1 = i2 = 0.0
    y = -1.0
    for n, x in enumerate(u.tolist()):
        i1 += x - y
        i2 += i1 - y
        y = 1.0 if i2 >= 0.0 else -1.0
        bits[n] = y > 0.0
    return bits


def tone_metrics(y, fs, f0):
    """(amplitude of the least-squares fit at f0, in-band SINAD in dB up to 20 kHz)."""
    from scipy.signal import get_window
    t = np.arange(len(y)) / fs
    A = np.stack([np.sin(2 * np.pi * f0 * t), np.cos(2 * np.pi * f0 * t), np.ones_like(t)], axis=1)
    co = np.linalg.lstsq(A, y, rcond=None)[0]
    amp = float(np.hypot(co[0], co[1]))
    Y = np.abs(np.fft.rfft(y * get_window("blackmanharris", len(y)))) ** 2
    f = np.fft.rfftfreq(len(y), 1.0 / fs)
    sig = np.abs(f - f0) <= 8 * fs / len(y)
    band = (f > 20.0) & (f <= 20000.0)
    return amp, 10 * np.log10(Y[sig].sum() / Y[band & ~sig].sum())


def test_sigma_delta_tone(pkg):
    fs = 2822400.0
    n = int(0.25 * fs)
    u = 0.5 * np.sin(2 * np.pi * 1000.0 * np.arange(n) / fs)
    bits = sdm2(u)
    byt = pack(bits[None, :])
    b = pkg.Batch(pkg.Plan(fs, 44100.0, 65536, 2.0, pkg.ATTEN_24), 1)
    lens = np.array([n], dtype=np.int64)
    y, ol = b.oneshot_clips(byt, lens, fmt=DSD_LSB)
    y = y[0, 1000:-1000]
    amp, sinad = tone_metrics(y, 44100.0, 1000.0)
    assert abs(20 * np.log10(amp / 0.5)) < 0.05, amp
    assert sinad > 60.0, sinad
    yw, _ = b.oneshot_clips(byt, lens, fmt=DSD_MSB)  # the wrong bit order: the shaped noise folds into the band
    assert tone_metrics(yw[0, 1000:-1000], 44100.0, 1000.0)[1] < sinad - 30.0


# ---- 7. the reference ----------------------------------------------------------------------------------------------

def test_oracle_parity(pkg):
    src, dst, M, n_ch, scale = 2822400.0, 48000.0, 32768, 2, 0.5
    oracle = ou.best_oracle()
    rng = np.random.default_rng(67)
    b = pkg.Batch(pkg.Plan(src, dst, M, 2.0, pkg.ATTEN_24), n_ch)
    rs = [oracle.Resampler(src, dst, M, 2.0, pkg.ATTEN_24) for _ in range(n_ch)]
    ys, yr = [[] for _ in range(n_ch)], [[] for _ in range(n_ch)]
    for k in range(5):
        bits = rng.integers(0, 2, (n_ch, M))
        y = b.process_host_fmt(pack(bits), fmt=DSD_LSB, in_scale=scale)
        for c in range(n_ch):
            r = rs[c].process(values(bits[c], scale))
            assert len(r) == y.shape[1]
            ys[c].append(y[c])
            yr[c].append(r)
    for c in range(n_ch):
        a, r = np.concatenate(ys[c]), np.concatenate(yr[c])
        assert len(a) > 0
        m, rms = ou.parity_metrics(a, r)
        assert m <= 32 * ou.EPS and rms <= 4 * ou.EPS, (m / ou.EPS, rms / ou.EPS)
