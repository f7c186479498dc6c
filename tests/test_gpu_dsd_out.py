"""One-bit DSD output on the device (r8bgpu_batch_set_dsd_out): every call path against the host modulator
(r8bgpu_dsd_modulate_host) applied to the fp64 outputs of a twin batch fed the same blocks, packed by np.packbits, bit
for bit; byte counts and held-back bits; the state rules and the refusals.  The host modulator itself is pinned to a
restatement of the contract in test_dsd_out_cpu.py.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SCALE = 0.5
# (src, dst): PCM up to DSD64 / DSD64 at 48k / DSD128, DSD256 in to DSD64 out, and DSD64 passthrough
PLANS = [(44100.0, 2822400.0), (48000.0, 3072000.0), (44100.0, 5644800.0), (11289600.0, 2822400.0),
         (2822400.0, 2822400.0)]
N_CH = 6
MAX_IN = 4096


def _dsd_in(src):
    return src % 44100.0 == 0 and src >= 2822400.0


class Expect:
    """The host modulator per channel, with its state and its held-back bits carried between calls."""

    def __init__(self, pkg, n_ch, msb=False):
        self.pkg, self.msb = pkg, msb
        self.st = [np.zeros(8) for _ in range(n_ch)]
        self.held = [np.zeros(0, np.uint8) for _ in range(n_ch)]

    def __call__(self, c, y, zeros=0):
        bits, ov = self.pkg.dsd_modulate(np.concatenate([y, np.zeros(zeros)]), SCALE, self.st[c])
        assert ov == 0
        allb = np.concatenate([self.held[c], bits])
        n = len(allb) // 8 * 8
        self.held[c] = allb[n:]
        return np.packbits(allb[:n], bitorder="big" if self.msb else "little"), n

    def flush(self, c, y):
        out = self(c, y, (-(len(self.held[c]) + len(y))) % 8)
        self.clear([c])
        return out

    def clear(self, chans):
        for c in chans:
            self.st[c][:] = 0
            self.held[c] = np.zeros(0, np.uint8)


def _input(src, n_ch, l, seed):
    """Planar input of l samples per channel: DSD bytes for a DSD source, else a PCM mix of sines and noise."""
    rng = np.random.default_rng(seed)
    if _dsd_in(src):
        return rng.integers(0, 256, (n_ch, l // 8), dtype=np.uint8), 16
    t = np.arange(l) + 1000 * seed
    x = 0.8 * np.sin(2 * np.pi * 0.0226 * (t[None, :] + 37 * np.arange(n_ch)[:, None])) + 0.05 * rng.standard_normal((n_ch, l))
    return x, None


def _to_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(a):
    return a if isinstance(a, np.ndarray) else a.cpu().numpy()


def _pair(pkg, src, dst, n_ch=N_CH, device=-2):
    plan = pkg.Plan(src, dst, MAX_IN, 2.0, pkg.ATTEN_24)
    b, twin = pkg.Batch(plan, n_ch, device), pkg.Batch(plan, n_ch)
    b.set_dsd_out(True)
    return b, twin


def _row(y, c, nbytes, interleaved):
    return y[:nbytes, c] if interleaved else y[c, :nbytes]


def _ragged_round(pkg, b, twin, ex, x, fmt, lens, interleaved, device, out_fmt):
    xin = x.T.copy() if interleaved else x
    if device:
        xin = _to_dev(xin)
    y, cnt = b.process_ragged_fmt(xin, lens, out_fmt=out_fmt, interleaved=interleaved, out_scale=SCALE, fmt=fmt,
                                  in_scale=0.5 if fmt else 1.0)
    yt, cnt_t = twin.process_ragged_fmt(x, lens, out_fmt=pkg.F64, fmt=fmt, in_scale=0.5 if fmt else 1.0)
    y = _np(y)
    for c in range(len(lens)):
        want, n = ex(c, yt[c, :cnt_t[c]])
        assert cnt[c] == n and n % 8 == 0
        np.testing.assert_array_equal(_row(y, c, n // 8, interleaved), want, err_msg=f"channel {c}")
        # nothing past the count (the buffer starts zeroed; a byte the call wrote may be 0 too, so check the rest only)
        assert not np.any((y[n // 8:, c] if interleaved else y[c, n // 8:]))


def _flush_round(pkg, b, twin, ex, chans, targets, interleaved, device, out_fmt):
    y, cnt = b.flush(chans, targets, out_fmt=out_fmt, interleaved=interleaved, out_scale=SCALE,
                     device=("cuda" if device else None))
    yt, cnt_t = twin.flush(chans, targets)
    y = _np(y)
    for c in range(len(ex.st)):
        if c not in chans:
            assert cnt[c] == 0
            continue
        want, n = ex.flush(c, yt[c, :cnt_t[c]])
        assert cnt[c] == n and n % 8 == 0
        np.testing.assert_array_equal(_row(y, c, n // 8, interleaved), want, err_msg=f"flush channel {c}")


# ---- lock-step calls -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("src,dst", PLANS)
@pytest.mark.parametrize("host", [True, False])
@pytest.mark.parametrize("layout", ["lsb_planar", "msb_interleaved"])
def test_lockstep(pkg, src, dst, host, layout):
    msb, interleaved = layout == "msb_interleaved", layout == "msb_interleaved"
    out_fmt = pkg.DSD_MSB if msb else pkg.DSD_LSB
    b, twin = _pair(pkg, src, dst)
    ex = Expect(pkg, N_CH, msb)
    cap = b.max_out_len
    assert cap % 8 == 0
    for k, l in enumerate([4096, 1000, 24, 4096, 3000]):
        x, fmt = _input(src, N_CH, l, k)
        yt = twin.process_host_fmt(x, out_fmt=pkg.F64, fmt=fmt, in_scale=0.5 if fmt else 1.0)
        xin = x.T.copy() if interleaved else x
        if host:
            y = b.process_host_fmt(xin, out_fmt=out_fmt, interleaved=interleaved, out_scale=SCALE, fmt=fmt,
                                   in_scale=0.5 if fmt else 1.0)
        else:
            import torch
            xd = _to_dev(xin)
            yo = torch.zeros(((cap // 8, N_CH) if interleaved else (N_CH, cap // 8)), dtype=torch.uint8, device="cuda")
            b.set_stream(torch.cuda.current_stream().cuda_stream)
            w = xin.shape[0] if interleaved else xin.shape[1]
            n = b.process_fmt(pkg.Buffer.make(xd.data_ptr(), fmt or pkg.F64, interleaved, N_CH if interleaved else w,
                                              0.5 if fmt else 1.0), l,
                              pkg.Buffer.make(yo.data_ptr(), out_fmt, interleaved, N_CH if interleaved else cap // 8, SCALE),
                              cap, host=False)
            torch.cuda.synchronize()
            y = yo.cpu().numpy()
            y = y[:n // 8] if interleaved else y[:, :n // 8]
        for c in range(N_CH):
            want, n = ex(c, yt[c])
            np.testing.assert_array_equal(_row(y, c, n // 8, interleaved), want, err_msg=f"call {k} channel {c}")
            assert (y.shape[0] if interleaved else y.shape[1]) == n // 8
    _flush_round(pkg, b, twin, ex, list(range(N_CH)), None, interleaved, not host, out_fmt)
    # the channels restart after the flush
    x, fmt = _input(src, N_CH, 2000, 9)
    yt = twin.process_host_fmt(x, out_fmt=pkg.F64, fmt=fmt, in_scale=0.5 if fmt else 1.0)
    y = b.process_host_fmt(x, out_fmt=pkg.DSD_LSB, out_scale=SCALE, fmt=fmt, in_scale=0.5 if fmt else 1.0)
    ex.msb = False
    for c in range(N_CH):
        np.testing.assert_array_equal(y[c], ex(c, yt[c])[0])


# ---- ragged calls, flushes -------------------------------------------------------------------------------------------

RAGGED = ([(p, "lsb_planar") for p in PLANS] + [(p, "msb_interleaved") for p in PLANS] +
          [(PLANS[0], "msb_planar"), (PLANS[0], "lsb_interleaved")])


@pytest.mark.parametrize("rates,layout", RAGGED)
@pytest.mark.parametrize("device", [False, True])
def test_ragged_and_flush(pkg, rates, layout, device):
    src, dst = rates
    msb, interleaved = layout.startswith("msb"), layout.endswith("interleaved")
    out_fmt = pkg.DSD_MSB if msb else pkg.DSD_LSB
    b, twin = _pair(pkg, src, dst)
    ex = Expect(pkg, N_CH, msb)
    rng = np.random.default_rng(int(src + dst) % 1000)
    for k in range(5):
        lens = rng.integers(0, MAX_IN + 1, N_CH).astype(np.int32)
        lens[k % N_CH] = 0
        if _dsd_in(src):
            lens -= lens % 8
        x, fmt = _input(src, N_CH, MAX_IN, 20 + k)
        _ragged_round(pkg, b, twin, ex, x, fmt, lens, interleaved, device, out_fmt)
    # explicit targets (multiples of 8) on some channels, the rest keep their state
    n_out = twin.channel_totals()[1]
    chans = [1, 3, 4]
    targets = [int((n_out[c] + 100 + 7) // 8 * 8) for c in chans]
    _flush_round(pkg, b, twin, ex, chans, targets, interleaved, device, out_fmt)
    x, fmt = _input(src, N_CH, MAX_IN, 40)
    lens = np.full(N_CH, 1600, np.int32)
    _ragged_round(pkg, b, twin, ex, x, fmt, lens, interleaved, device, out_fmt)
    _flush_round(pkg, b, twin, ex, list(range(N_CH)), None, interleaved, device, out_fmt)
    np.testing.assert_array_equal(b.dsd_overloads(), np.zeros(N_CH))


def test_nothing_past_the_count(pkg):
    """Bytes past count / 8 keep what the caller's buffer held, on both forms and in both layouts."""
    b, twin = _pair(pkg, 44100.0, 2822400.0)
    lib = pkg.lib()
    lens = np.array([5, 0, 17, 4096, 333, 1], np.int32)
    x = np.random.default_rng(1).uniform(-0.5, 0.5, (N_CH, MAX_IN))
    cap = b.max_out_len
    for interleaved in (False, True):
        for host in (True, False):
            xin = x.T.copy() if interleaved else x
            y = np.full(((cap // 8, N_CH) if interleaved else (N_CH, cap // 8)), 0xA5, np.uint8)
            counts = np.zeros(N_CH, np.int32)
            bi = pkg.Buffer.make(xin.ctypes.data, pkg.F64, interleaved, N_CH if interleaved else MAX_IN)
            if host:
                bo = pkg.Buffer.make(y.ctypes.data, pkg.DSD_LSB, interleaved, N_CH if interleaved else cap // 8, SCALE)
                rc = lib.r8bgpu_batch_process_host_ragged_fmt(b._h, C.byref(bi), lens.ctypes.data, C.byref(bo), cap,
                                                              counts.ctypes.data)
            else:
                import torch
                xd, yd = _to_dev(xin), _to_dev(y)
                bi = pkg.Buffer.make(xd.data_ptr(), pkg.F64, interleaved, N_CH if interleaved else MAX_IN)
                bo = pkg.Buffer.make(yd.data_ptr(), pkg.DSD_LSB, interleaved, N_CH if interleaved else cap // 8, SCALE)
                b.set_stream(torch.cuda.current_stream().cuda_stream)
                rc = lib.r8bgpu_batch_process_ragged_fmt(b._h, C.byref(bi), lens.ctypes.data, C.byref(bo), cap,
                                                         counts.ctypes.data)
                torch.cuda.synchronize()
                y = yd.cpu().numpy()
            assert rc == 0
            assert np.all(counts % 8 == 0)
            for c in range(N_CH):
                rest = y[counts[c] // 8:, c] if interleaved else y[c, counts[c] // 8:]
                assert np.all(rest == 0xA5)


# ---- batch kinds -----------------------------------------------------------------------------------------------------

def test_device_all(pkg, monkeypatch):
    monkeypatch.setenv("R8BGPU_FORCE_SHARDS", "3")
    n_ch = 7
    b, twin = _pair(pkg, 44100.0, 2822400.0, n_ch, pkg.DEVICE_ALL)
    assert len(b.shards()) == 3
    ex = Expect(pkg, n_ch)
    for k in range(3):
        x, _ = _input(44100.0, n_ch, 2048, 50 + k)
        y = b.process_host_fmt(x, out_fmt=pkg.DSD_LSB, out_scale=SCALE)
        yt = twin.process_host(x)
        for c in range(n_ch):
            np.testing.assert_array_equal(y[c], ex(c, yt[c])[0], err_msg=f"call {k} channel {c}")
    rng = np.random.default_rng(4)
    for k in range(2):
        x, _ = _input(44100.0, n_ch, MAX_IN, 60 + k)
        _ragged_round(pkg, b, twin, ex, x, None, rng.integers(0, MAX_IN + 1, n_ch).astype(np.int32), False, False,
                      pkg.DSD_LSB)
    # a call one shard refuses (a length past MaxInLen in the last shard's channel) changes no shard
    x = np.zeros((n_ch, MAX_IN + 8))
    x[:, :MAX_IN] = _input(44100.0, n_ch, MAX_IN, 63)[0]
    bad = np.full(n_ch, 1000, np.int32)
    bad[n_ch - 1] = MAX_IN + 8
    with pytest.raises(pkg.R8bGpuError, match="outside"):
        b.process_ragged_fmt(x, bad, out_fmt=pkg.DSD_LSB, out_scale=SCALE)
    _ragged_round(pkg, b, twin, ex, x[:, :MAX_IN], None, np.full(n_ch, 1000, np.int32), False, False, pkg.DSD_LSB)
    _flush_round(pkg, b, twin, ex, [0, 2, 5, 6], None, False, False, pkg.DSD_LSB)
    assert len(b.dsd_overloads()) == n_ch


# ---- whole tiles: CTAs whose 32 lanes all walk a tile ----------------------------------------------------------------

@pytest.mark.parametrize("host", [True, False])
def test_whole_tiles(pkg, host):
    """40 channels: one CTA of 32 live lanes and one of 8.  Equal multi-tile lock-step calls (the first call's count is
    not a multiple of 8, so the later calls' interior tiles are walked whole after held-back bits), then ragged calls of
    long, different lengths (whole tiles until the CTA's shortest channel ends), then a flush."""
    n_ch = 40
    b, twin = _pair(pkg, 44100.0, 2822400.0, n_ch)
    ex = Expect(pkg, n_ch)
    cap = b.max_out_len
    held = []
    for k in range(3):
        x, _ = _input(44100.0, n_ch, MAX_IN, 100 + k)
        yt = twin.process_host(x)
        if host:
            y = b.process_host_fmt(x, out_fmt=pkg.DSD_LSB, out_scale=SCALE)
        else:
            import torch
            xd = _to_dev(x)
            yo = torch.zeros((n_ch, cap // 8), dtype=torch.uint8, device="cuda")
            b.set_stream(torch.cuda.current_stream().cuda_stream)
            nb = b.process_fmt(pkg.Buffer.make(xd.data_ptr(), pkg.F64, False, MAX_IN), MAX_IN,
                               pkg.Buffer.make(yo.data_ptr(), pkg.DSD_LSB, False, cap // 8, SCALE), cap, host=False)
            torch.cuda.synchronize()
            y = yo[:, :nb // 8].cpu().numpy()
        assert y.shape[1] * 8 >= 128 * 16  # many tiles per channel
        for c in range(n_ch):
            want, n = ex(c, yt[c])
            assert y.shape[1] == n // 8
            np.testing.assert_array_equal(y[c], want, err_msg=f"call {k} channel {c}")
        held.append(len(ex.held[0]))
    assert held[0] > 0  # the later calls start after held-back bits
    rng = np.random.default_rng(17)
    for k in range(2):
        x, _ = _input(44100.0, n_ch, MAX_IN, 110 + k)
        lens = rng.integers(2000, MAX_IN + 1, n_ch).astype(np.int32)
        _ragged_round(pkg, b, twin, ex, x, None, lens, False, not host, pkg.DSD_LSB)
    _flush_round(pkg, b, twin, ex, list(range(n_ch)), None, False, not host, pkg.DSD_LSB)


@pytest.mark.parametrize("device", [False, True])
def test_mixed_batch(pkg, device):
    plans = [pkg.Plan(44100.0, 2822400.0, MAX_IN, 2.0, pkg.ATTEN_24), pkg.Plan(48000.0, 3072000.0, MAX_IN, 2.0, pkg.ATTEN_24)]
    plan_of = [0, 1, 1, 0, 1, 0]
    b, twin = pkg.Batch.mixed(plans, plan_of), pkg.Batch.mixed(plans, plan_of)
    b.set_dsd_out(True)
    ex = Expect(pkg, len(plan_of))
    rng = np.random.default_rng(12)
    for k in range(4):
        lens = rng.integers(0, MAX_IN + 1, len(plan_of)).astype(np.int32)
        x, _ = _input(44100.0, len(plan_of), MAX_IN, 70 + k)
        _ragged_round(pkg, b, twin, ex, x, None, lens, k == 1, device, pkg.DSD_LSB)
    _flush_round(pkg, b, twin, ex, [0, 1, 2, 3, 4, 5], None, False, device, pkg.DSD_LSB)


def test_invariance_slot_width_layout(pkg):
    """One stream's bytes do not depend on the batch width, its slot or the layout.  (The same input blocks: a different
    chunking of the input gives the resampler's fp64 stream other roundings; the modulator's own chunking is covered by
    the comparisons with the host modulator above, which runs each stream in one piece.)"""
    plan = pkg.Plan(44100.0, 2822400.0, MAX_IN, 2.0, pkg.ATTEN_24)
    x1 = _input(44100.0, 1, 3 * MAX_IN, 3)[0][0]
    outs = []
    chunks = [7, 4089, 1, MAX_IN, MAX_IN - 1]
    for n_ch, slot, il in [(1, 0, False), (5, 3, False), (37, 36, True)]:
        b = pkg.Batch(plan, n_ch)
        b.set_dsd_out(True)
        rows, at = [], 0
        for l in chunks:
            x = np.zeros((n_ch, MAX_IN))
            x[slot, :l] = x1[at:at + l]
            at += l
            lens = np.zeros(n_ch, np.int32)
            lens[slot] = l
            y, cnt = b.process_ragged_fmt(x.T.copy() if il else x, lens, out_fmt=pkg.DSD_LSB, interleaved=il, out_scale=SCALE)
            rows.append(_row(y, slot, cnt[slot] // 8, il))
        y, cnt = b.flush([slot], out_fmt=pkg.DSD_LSB, out_scale=SCALE)
        rows.append(y[slot, :cnt[slot] // 8])
        assert at == 3 * MAX_IN
        outs.append(np.concatenate(rows))
    for o in outs[1:]:
        np.testing.assert_array_equal(o, outs[0])


# ---- state rules, refusals -------------------------------------------------------------------------------------------

def test_state_rules(pkg):
    b, twin = _pair(pkg, 44100.0, 2822400.0)
    ex = Expect(pkg, N_CH)
    lens = np.array([1001, 7, 4096, 0, 333, 2048], np.int32)
    xs = [_input(44100.0, N_CH, MAX_IN, 80 + k)[0] for k in range(3)]
    first = []
    for x in xs:
        _ragged_round(pkg, b, twin, ex, x, None, lens, False, False, pkg.DSD_LSB)
        first.append(b.dsd_overloads())
    b.clear()
    twin.clear()
    ex.clear(range(N_CH))
    for x in xs:
        _ragged_round(pkg, b, twin, ex, x, None, lens, False, False, pkg.DSD_LSB)
    b.clear_channels([2, 4])
    twin.clear_channels([2, 4])
    ex.clear([2, 4])
    _ragged_round(pkg, b, twin, ex, xs[0], None, lens, False, False, pkg.DSD_LSB)
    np.testing.assert_array_equal(b.dsd_overloads(), np.zeros(N_CH))
    # turning it on again restarts every modulator (the resampler keeps its state)
    b.set_dsd_out(True)
    ex.clear(range(N_CH))
    _ragged_round(pkg, b, twin, ex, xs[1], None, lens, False, False, pkg.DSD_LSB)


def test_refusals_change_nothing(pkg):
    # opt-in on a batch whose destination is not a DSD rate
    b48 = pkg.Batch(pkg.Plan(44100.0, 48000.0, MAX_IN, 2.0, pkg.ATTEN_24), 2)
    with pytest.raises(pkg.R8bGpuError, match="not a DSD rate"):
        b48.set_dsd_out(True)
    with pytest.raises(pkg.R8bGpuError, match="input-only"):
        b48.process_host_fmt(np.zeros((2, 64)), out_fmt=pkg.DSD_LSB)
    mixed = pkg.Batch.mixed([pkg.Plan(44100.0, 2822400.0, MAX_IN, 2.0, pkg.ATTEN_24),
                             pkg.Plan(44100.0, 96000.0, MAX_IN, 2.0, pkg.ATTEN_24)], [0, 1])
    with pytest.raises(pkg.R8bGpuError, match="not a DSD rate"):
        mixed.set_dsd_out(True)
    b, twin = _pair(pkg, 44100.0, 2822400.0)
    ex = Expect(pkg, N_CH)
    x = _input(44100.0, N_CH, MAX_IN, 90)[0]
    lens = np.array([1000, 8, 4096, 0, 5, 2000], np.int32)
    _ragged_round(pkg, b, twin, ex, x, None, lens, False, False, pkg.DSD_LSB)
    bad = [lambda: b.process_host_fmt(x, out_fmt=pkg.S16),
           lambda: b.process_ragged_fmt(x, lens, out_fmt=pkg.F32),
           lambda: b.process_host(x),
           lambda: b.process_ragged([x[c, :lens[c]] for c in range(N_CH)]),
           lambda: b.flush([0], [12345], out_fmt=pkg.DSD_LSB),
           lambda: b.flush([0], out_fmt=pkg.S16),
           lambda: b.clear_channels([9])]
    for f in bad:
        with pytest.raises(pkg.R8bGpuError):
            f()
    for f in (lambda: b.export_channels([0]), lambda: b.import_channels([0], [np.zeros(b.plan.state_bytes, np.uint8)])):
        with pytest.raises(pkg.R8bGpuError, match="DSD output is on"):
            f()
    _ragged_round(pkg, b, twin, ex, x, None, lens, False, False, pkg.DSD_LSB)
    _flush_round(pkg, b, twin, ex, [0, 3], [int((twin.channel_totals()[1][0] + 64) // 8 * 8), 0], False, False, pkg.DSD_LSB)
    # off again: exactly as before
    b.set_dsd_out(False)
    with pytest.raises(pkg.R8bGpuError, match="DSD formats are input-only"):
        b.process_ragged_fmt(x, lens, out_fmt=pkg.DSD_LSB)
    with pytest.raises(pkg.R8bGpuError, match="DSD output is off"):
        b.dsd_overloads()
    y, cnt = b.process_ragged_fmt(x, lens, out_fmt=pkg.F64)
    yt, cnt_t = twin.process_ragged_fmt(x, lens, out_fmt=pkg.F64)
    np.testing.assert_array_equal(cnt, cnt_t)
    np.testing.assert_array_equal(y, yt)
