"""Dithered integer output on the device (r8bgpu_batch_set_dither): every typed path against the host quantiser applied to
the fp64 outputs of a twin batch fed the same blocks, bit for bit; OFF channels against an untouched batch; the state
rules and the refusals.  The host quantiser itself is pinned to a numpy restatement of the contract in
test_dither_cpu.py.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SCALE = 32767.0
FSCALE = {2: SCALE, 3: SCALE * 256, 4: SCALE * 65536}  # full scale of S16, S24, S32
TAPS9 = [2.033, -2.165, 1.959, -1.590, 0.6149, -0.2, 0.1, -0.05, 0.01]
# per channel: (seed, taps) or None for OFF
SETTINGS = [None, (11, None), (12, TAPS9), (13, None), (14, [1.0]), None, (16, list(np.linspace(-0.3, 0.3, 16))), None]


def _apply(pkg, b, settings, offset=0):
    for c, s in enumerate(settings):
        if s is not None:
            b.set_dither([c + offset], s[0], s[1])


class Expect:
    """The host quantiser per channel, with each channel's output index and error history carried between calls."""

    def __init__(self, pkg, settings, fmt=None):
        self.pkg, self.settings, self.fmt = pkg, settings, fmt or pkg.S16
        self.n = np.zeros(len(settings), dtype=np.int64)
        self.st = [np.zeros(16) for _ in settings]

    def __call__(self, c, y, quantise=True):
        s = self.settings[c]
        if not quantise:  # a float-output call: the index advances, the history stays
            self.n[c] += len(y)
            return None
        sc = FSCALE[self.fmt]
        if s is None:
            q, _ = self.pkg.dither_quantize(y, self.fmt, 0, scale=sc, kind=self.pkg.DITHER_OFF)
        else:
            q, _ = self.pkg.dither_quantize(y, self.fmt, s[0], s[1], scale=sc, first_index=int(self.n[c]), state=self.st[c])
        self.n[c] += len(y)
        return q

    def clear(self, chans=None):
        for c in range(len(self.settings)) if chans is None else chans:
            self.n[c] = 0
            self.st[c][:] = 0


def _sig(n_ch, width, seed, amp=3e-4):
    rng = np.random.default_rng(seed)
    t = np.arange(width)
    return (amp * np.sin(2 * np.pi * 0.013 * (t[None, :] + 100 * np.arange(n_ch)[:, None]))
            + amp * 0.5 * rng.standard_normal((n_ch, width)))


def _to_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(a):
    return a if isinstance(a, np.ndarray) else a.cpu().numpy()


# ---- lock-step typed calls -------------------------------------------------------------------------------------------

# flat TPDF only: 44100->96000 narrows (and dithers) in the fused kernel's stores
FLAT = [None, (11, None), None, (13, None), None, (15, None), None, (17, None)]


@pytest.mark.parametrize("src,dst", [(44100.0, 96000.0), (48000.0, 44100.0)])
@pytest.mark.parametrize("host", [True, False])
@pytest.mark.parametrize("settings", ["mixed", "flat"])
def test_lockstep_fmt(pkg, src, dst, host, settings):
    SETTINGS = globals()["SETTINGS"] if settings == "mixed" else FLAT
    n_ch = len(SETTINGS)
    plan = pkg.Plan(src, dst, 4096, 2.0, pkg.ATTEN_24)
    b, twin, plain = pkg.Batch(plan, n_ch), pkg.Batch(plan, n_ch), pkg.Batch(plan, n_ch)
    _apply(pkg, b, SETTINGS)
    ex = Expect(pkg, SETTINGS)
    cap = plan.max_out_len
    for k, l in enumerate([4096, 1000, 4096, 17, 3000]):
        x = _sig(n_ch, l, k)
        yt = twin.process_host(x)
        if host:
            y = b.process_host_fmt(x, out_fmt=pkg.S16, out_scale=SCALE)
            yp = plain.process_host_fmt(x, out_fmt=pkg.S16, out_scale=SCALE)
        else:
            import torch
            outs = []
            for bb in (b, plain):
                xin = _to_dev(x)
                yo = torch.zeros((n_ch, cap), dtype=torch.int16, device="cuda")
                bb.set_stream(torch.cuda.current_stream().cuda_stream)
                n = bb.process_fmt(pkg.Buffer.make(xin.data_ptr(), pkg.F64, False, l), l,
                                   pkg.Buffer.make(yo.data_ptr(), pkg.S16, False, cap, SCALE), cap, host=False)
                torch.cuda.synchronize()
                outs.append(yo[:, :n].cpu().numpy())
            y, yp = outs
        assert y.shape == yt.shape == yp.shape
        for c in range(n_ch):
            np.testing.assert_array_equal(y[c], ex(c, yt[c]), err_msg=f"call {k} channel {c}")
            if SETTINGS[c] is None:
                np.testing.assert_array_equal(y[c], yp[c])  # OFF: today's bytes
    assert any(not np.array_equal(y[c], yp[c]) for c in range(n_ch) if SETTINGS[c] is not None)


# ---- ragged typed calls, flush, state rules ----------------------------------------------------------------------------

def _ragged_round(pkg, b, twin, ex, x, lens, interleaved, device, quantise=True):
    xin = x.T.copy() if interleaved else x
    if device:
        xin = _to_dev(xin)
    out_fmt = ex.fmt if quantise else pkg.F64
    y, cnt = b.process_ragged_fmt(xin, lens, out_fmt=out_fmt, interleaved=interleaved,
                                  out_scale=FSCALE[ex.fmt] if quantise else 1.0)
    yt, cnt_t = twin.process_ragged_fmt(x, lens, out_fmt=pkg.F64)
    y = _np(y)
    np.testing.assert_array_equal(cnt, cnt_t)
    for c in range(len(lens)):
        row = y[:cnt[c], c] if interleaved else y[c, :cnt[c]]
        q = ex(c, yt[c, :cnt[c]], quantise)
        if quantise:
            np.testing.assert_array_equal(row, q, err_msg=f"channel {c}")
    return y, cnt


def _flush_round(pkg, b, twin, ex, interleaved, device, chans=None):
    n_ch = len(ex.settings)
    chans = list(range(n_ch)) if chans is None else chans
    y, cnt = b.flush(chans, out_fmt=ex.fmt, interleaved=interleaved, out_scale=FSCALE[ex.fmt],
                     device=("cuda" if device else None))
    yt, cnt_t = twin.flush(chans)
    y = _np(y)
    np.testing.assert_array_equal(cnt, cnt_t)
    for c in chans:
        row = y[:cnt[c], c] if interleaved else y[c, :cnt[c]]
        np.testing.assert_array_equal(row, ex(c, yt[c, :cnt[c]]), err_msg=f"flush channel {c}")
    ex.clear(chans)


@pytest.mark.parametrize("interleaved", [False, True])
@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("fmt", [2, 3, 4])
def test_ragged_fmt_and_flush(pkg, interleaved, device, fmt):
    if fmt == 3 and device:
        pytest.skip("packed 24-bit device buffers are not offered by the torch front")
    n_ch = len(SETTINGS)
    plan = pkg.Plan(44100.0, 48000.0, 2048, 2.0, pkg.ATTEN_24)
    b, twin = pkg.Batch(plan, n_ch), pkg.Batch(plan, n_ch)
    _apply(pkg, b, SETTINGS)
    ex = Expect(pkg, SETTINGS, fmt)
    rng = np.random.default_rng(5)
    for k in range(4):
        lens = rng.integers(0, 2049, n_ch).astype(np.int32)
        _ragged_round(pkg, b, twin, ex, _sig(n_ch, 2048, 10 + k), lens, interleaved, device)
    _flush_round(pkg, b, twin, ex, interleaved, device)
    # settings survive the flush: the channels restart from index 0 with an empty history
    lens = np.full(n_ch, 1500, np.int32)
    _ragged_round(pkg, b, twin, ex, _sig(n_ch, 2048, 99), lens, interleaved, device)


def test_state_rules(pkg):
    n_ch = len(SETTINGS)
    plan = pkg.Plan(44100.0, 48000.0, 2048, 2.0, pkg.ATTEN_24)
    b, twin = pkg.Batch(plan, n_ch), pkg.Batch(plan, n_ch)
    _apply(pkg, b, SETTINGS)
    ex = Expect(pkg, SETTINGS)
    lens = np.full(n_ch, 2000, np.int32)
    xs = [_sig(n_ch, 2048, 40 + k) for k in range(3)]
    first = [_ragged_round(pkg, b, twin, ex, x, lens, False, False)[0] for x in xs]
    # clear(): the settings stay, the same input gives the same bytes
    b.clear()
    twin.clear()
    ex.clear()
    again = [_ragged_round(pkg, b, twin, ex, x, lens, False, False)[0] for x in xs]
    for a, z in zip(first, again):
        np.testing.assert_array_equal(a, z)
    # a float-output call in the middle keeps the shaper history; clear_channels restarts only the named channels
    _ragged_round(pkg, b, twin, ex, xs[0], lens, False, False, quantise=False)
    _ragged_round(pkg, b, twin, ex, xs[1], lens, False, False)
    b.clear_channels([2, 4])
    twin.clear_channels([2, 4])
    ex.clear([2, 4])
    _ragged_round(pkg, b, twin, ex, xs[2], lens, False, False)
    # setting a channel again keeps its history; new taps apply from its next output
    b.set_dither([2], 12, [0.5])
    ex.settings = list(ex.settings)
    ex.settings[2] = (12, [0.5])
    _ragged_round(pkg, b, twin, ex, xs[0], lens, False, False)


def test_invariance_slot_width_layout(pkg):
    plan = pkg.Plan(44100.0, 48000.0, 2048, 2.0, pkg.ATTEN_24)
    x1 = _sig(1, 2048, 3)
    outs = []
    for n_ch, slot, il in [(1, 0, False), (5, 3, False), (37, 36, True)]:
        b = pkg.Batch(plan, n_ch)
        b.set_dither([slot], 777, TAPS9)
        x = np.zeros((n_ch, 2048))
        x[slot] = x1[0]
        lens = np.full(n_ch, 2048, np.int32)
        rows = []
        for _ in range(3):
            y, cnt = b.process_ragged_fmt(x.T.copy() if il else x, lens, out_fmt=pkg.S16, interleaved=il, out_scale=SCALE)
            rows.append(y[:cnt[slot], slot] if il else y[slot, :cnt[slot]])
        outs.append(np.concatenate(rows))
    for o in outs[1:]:
        np.testing.assert_array_equal(o, outs[0])


def test_oneshot_clips(pkg):
    n_ch = len(SETTINGS)
    plan = pkg.Plan(48000.0, 44100.0, 2048, 2.0, pkg.ATTEN_24)
    b, twin = pkg.Batch(plan, n_ch), pkg.Batch(plan, n_ch)
    _apply(pkg, b, SETTINGS)
    lens = np.random.default_rng(1).integers(100, 5000, n_ch)
    x = _sig(n_ch, 5000, 8)
    y, op = b.oneshot_clips(x, lens, out_fmt=pkg.S16, out_scale=SCALE)
    yt, opt = twin.oneshot_clips(x, lens)
    np.testing.assert_array_equal(op, opt)
    ex = Expect(pkg, SETTINGS)
    for c in range(n_ch):
        np.testing.assert_array_equal(y[c, :op[c]], ex(c, yt[c, :op[c]]), err_msg=f"channel {c}")


@pytest.mark.parametrize("device", [False, True])
def test_mixed_batch(pkg, device):
    plans = [pkg.Plan(44100.0, 48000.0, 2048, 2.0, pkg.ATTEN_24), pkg.Plan(16000.0, 8000.0, 2048, 2.0, pkg.ATTEN_24),
             pkg.Plan(48000.0, 48000.0, 2048, 2.0, pkg.ATTEN_24)]
    plan_of = [0, 1, 2, 0, 1, 2, 0, 1]
    b, twin = pkg.Batch.mixed(plans, plan_of), pkg.Batch.mixed(plans, plan_of)
    _apply(pkg, b, SETTINGS)
    ex = Expect(pkg, SETTINGS)
    rng = np.random.default_rng(9)
    for k in range(3):
        lens = rng.integers(0, 2049, len(plan_of)).astype(np.int32)
        _ragged_round(pkg, b, twin, ex, _sig(len(plan_of), 2048, 60 + k), lens, k == 1, device)
    # flush every channel: a passthrough part's tail of zeros is dithered as in an ordinary batch
    _flush_round(pkg, b, twin, ex, False, device)


def test_trim_plan(pkg):
    n_ch = len(SETTINGS)
    plan = pkg.Plan.trim(44100.0, 48000.0, 2048, 2.0, pkg.ATTEN_24, 1e-3)
    b, twin = pkg.Batch(plan, n_ch), pkg.Batch(plan, n_ch)
    f = 1.0 + np.linspace(-5e-4, 5e-4, n_ch)
    for bb in (b, twin):
        bb.set_trim(range(n_ch), f)
    _apply(pkg, b, SETTINGS)
    ex = Expect(pkg, SETTINGS)
    for k in range(3):
        _ragged_round(pkg, b, twin, ex, _sig(n_ch, 2048, 70 + k), np.full(n_ch, 2048, np.int32), False, False)


def test_device_all_host_call(pkg, monkeypatch):
    monkeypatch.setenv("R8BGPU_FORCE_SHARDS", "3")
    n_ch = len(SETTINGS)
    plan = pkg.Plan(44100.0, 48000.0, 2048, 2.0, pkg.ATTEN_24)
    b, twin = pkg.Batch(plan, n_ch, pkg.DEVICE_ALL), pkg.Batch(plan, n_ch)
    assert len(b.shards()) == 3
    _apply(pkg, b, SETTINGS)
    ex = Expect(pkg, SETTINGS)
    for k in range(3):
        x = _sig(n_ch, 2048, 80 + k)
        y = b.process_host_fmt(x, out_fmt=pkg.S16, out_scale=SCALE)
        yt = twin.process_host(x)
        for c in range(n_ch):
            np.testing.assert_array_equal(y[c], ex(c, yt[c]), err_msg=f"call {k} channel {c}")


def test_off_is_today(pkg):
    n_ch = 6
    plan = pkg.Plan(44100.0, 96000.0, 2048, 2.0, pkg.ATTEN_24)
    untouched, off = pkg.Batch(plan, n_ch), pkg.Batch(plan, n_ch)
    off.set_dither(range(n_ch), 5, kind=pkg.DITHER_OFF)
    for k in range(3):
        x = _sig(n_ch, 2048, 90 + k)
        for fmt in (pkg.S16, pkg.S24, pkg.S32):
            np.testing.assert_array_equal(off.process_host_fmt(x, out_fmt=fmt, out_scale=SCALE * 256),
                                          untouched.process_host_fmt(x, out_fmt=fmt, out_scale=SCALE * 256))


def test_refusals_change_nothing(pkg):
    plan = pkg.Plan(44100.0, 48000.0, 2048, 2.0, pkg.ATTEN_24)
    b, ref = pkg.Batch(plan, 4), pkg.Batch(plan, 4)
    for bb in (b, ref):
        bb.set_dither([1], 3, TAPS9)
    bad = [dict(channels=[0], seeds=1, kind=9), dict(channels=[0], seeds=1, taps=[0.1] * 17),
           dict(channels=[0], seeds=1, taps=[0.5], kind=pkg.DITHER_OFF), dict(channels=[0], seeds=1, taps=[np.inf]),
           dict(channels=[4], seeds=1), dict(channels=[0, 0], seeds=1), dict(channels=[0, 1], seeds=1, taps=[[0.1], [np.nan]])]
    for kw in bad:
        with pytest.raises(pkg.R8bGpuError):
            b.set_dither(**kw)
    x = _sig(4, 2048, 1)
    np.testing.assert_array_equal(b.process_host_fmt(x, out_fmt=pkg.S16, out_scale=SCALE),
                                  ref.process_host_fmt(x, out_fmt=pkg.S16, out_scale=SCALE))


def test_cpp_front_set_dither(pkg, tmp_path):
    """r8b::CDSPResamplerBatch::setDither compiled against the library and run once: channel 1 (9 taps) against the
    host quantiser applied to a twin batch's fp64 output, channel 0 (OFF) against the cast."""
    import os
    import shutil
    import subprocess
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no g++")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib_dir = os.path.dirname(pkg.lib_path())
    exe = str(tmp_path / "dither_demo")
    subprocess.run([gxx, "-O1", "-std=c++11", "-I", os.path.join(root, "include"),
                    os.path.join(root, "tests", "cpp", "dither_demo.cpp"), "-o", exe, "-L", lib_dir, "-lr8bgpu",
                    "-Wl,-rpath," + lib_dir], check=True)
    frames = 3000
    _sig(2, frames, 4).tofile(str(tmp_path / "in.f64"))
    res = subprocess.run([exe, str(tmp_path / "in.f64"), str(tmp_path / "out.bin"), str(frames)], capture_output=True,
                         text=True)
    assert res.returncode == 0, (res.returncode, res.stderr)
    n = int(res.stdout)
    raw = open(str(tmp_path / "out.bin"), "rb").read()
    pos = 0
    for c in range(2):
        k = int(np.frombuffer(raw[pos:pos + 8], dtype=np.int64)[0])
        assert k == n
        y = np.frombuffer(raw[pos + 8:pos + 8 + 8 * k], dtype=np.float64)
        q = np.frombuffer(raw[pos + 8 + 8 * k:pos + 8 + 10 * k], dtype=np.int16)
        pos += 8 + 10 * k
        if c == 1:
            want, _ = pkg.dither_quantize(y, pkg.S16, 12345, TAPS9, scale=SCALE)
        else:
            want, _ = pkg.dither_quantize(y, pkg.S16, 0, scale=SCALE, kind=pkg.DITHER_OFF)
        np.testing.assert_array_equal(q, want)
