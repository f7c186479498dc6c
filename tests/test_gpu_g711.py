"""One-byte sample formats on the device: U8 and G.711 mu-law / A-law buffers on every typed path.

- Decoding: a typed call fed bytes gives, bit for bit, what the plain fp64 path gives when fed the decoded samples.
- The invariant: mu-law / A-law bytes are the G.711 encoding of the int16 bytes the same call writes as S16 (dither OFF
  and on); U8 bytes are the int8 value (cast or dither) + 128.
- The conversion of planar lock-step calls stays inside the resampling kernels (no extra launch).
- Silence is the encoding of zero; mixed and sharded batches agree with ordinary ones; mu-law round-trips.
The codec itself is pinned to a numpy restatement of G.711 in test_g711_cpu.py, which this file reuses.
"""
import numpy as np
import pytest

from test_g711_cpu import alaw_decode, alaw_encode, ulaw_decode, ulaw_encode

pytestmark = pytest.mark.gpu

U8, ULAW, ALAW, S16, F64 = 5, 6, 7, 2, 0
BYTE_FORMATS = [U8, ULAW, ALAW]
IN_SCALE = {U8: 1.0 / 128, ULAW: 1.0 / 32768, ALAW: 1.0 / 32768}
CHAINS = [(44100.0, 96000.0), (8000.0, 16000.0), (16000.0, 8000.0), (8000.0, 48000.0), (48000.0, 47999.0)]
TAPS9 = [2.033, -2.165, 1.959, -1.590, 0.6149, -0.2, 0.1, -0.05, 0.01]


def decode(fmt, b):
    b = np.asarray(b, dtype=np.int64)
    return {U8: lambda: b - 128, ULAW: lambda: ulaw_decode(b), ALAW: lambda: alaw_decode(b)}[fmt]()


def encode(fmt, s16):
    return (ulaw_encode if fmt == ULAW else alaw_encode)(s16)


def _bytes(rng, shape):
    return rng.integers(0, 256, shape).astype(np.uint8)


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(a):
    return a if isinstance(a, np.ndarray) else a.cpu().numpy()


def _lockstep_device(pkg, b, x, fmt, out_fmt, in_scale=1.0, out_scale=1.0):
    """Planar device-pointer lock-step call: x planar numpy of fmt's element type; returns planar numpy [n_ch, n]."""
    import torch
    n_ch, l = x.shape
    cap = b.plan.max_out_len
    xin = _dev(x)
    dt = {F64: torch.float64, S16: torch.int16}.get(out_fmt, torch.uint8)
    yo = torch.zeros((n_ch, max(cap, 1)), dtype=dt, device="cuda")
    b.set_stream(torch.cuda.current_stream().cuda_stream)
    n = b.process_fmt(pkg.Buffer.make(xin.data_ptr(), fmt, False, l, in_scale), l,
                      pkg.Buffer.make(yo.data_ptr(), out_fmt, False, max(cap, 1), out_scale), cap, host=False)
    torch.cuda.synchronize()
    return yo[:, :n].cpu().numpy()


# ---- 1. decoding ---------------------------------------------------------------------------------------------------

FORMS = ["host", "host_il", "device", "ragged_host", "ragged_host_il", "ragged_dev", "ragged_dev_il"]


@pytest.mark.parametrize("chain", CHAINS, ids=lambda c: "%g-%g" % c)
@pytest.mark.parametrize("fmt", BYTE_FORMATS)
def test_decoding_matches_fp64_path(pkg, chain, fmt):
    n_ch, M = 5, 2048
    plan = pkg.Plan(chain[0], chain[1], M, 2.0, pkg.ATTEN_24)
    sc = IN_SCALE[fmt]
    for form in FORMS:
        rng = np.random.default_rng(100 * CHAINS.index(chain) + 10 * fmt + FORMS.index(form))
        b, twin = pkg.Batch(plan, n_ch), pkg.Batch(plan, n_ch)
        il = form.endswith("_il")
        for k in range(3):
            if form.startswith("ragged"):
                lens = rng.integers(0, M + 1, n_ch).astype(np.int32)
                lens[k % n_ch] = M
                x = _bytes(rng, (n_ch, M))
                xf = decode(fmt, x).astype(np.float64) * sc
                xin = x.T.copy() if il else x
                if "dev" in form:
                    xin = _dev(xin)
                y, cnt = b.process_ragged_fmt(xin, lens, fmt=fmt, out_fmt=F64, in_scale=sc, interleaved=il)
                yt, cnt_t = twin.process_ragged_fmt(xf, lens, out_fmt=F64)
                y = _np(y)
                np.testing.assert_array_equal(cnt, cnt_t)
                for c in range(n_ch):
                    row = y[:cnt[c], c] if il else y[c, :cnt[c]]
                    np.testing.assert_array_equal(row, yt[c, :cnt[c]], err_msg=f"{form} call {k} channel {c}")
            else:
                l = [M, 1000, M][k]
                x = _bytes(rng, (n_ch, l))
                xf = decode(fmt, x).astype(np.float64) * sc
                yt = twin.process_host(xf)
                if form == "device":
                    y = _lockstep_device(pkg, b, x, fmt, F64, in_scale=sc)
                elif il:
                    y = b.process_host_fmt(x.T.copy(), fmt=fmt, out_fmt=F64, in_scale=sc, interleaved=True).T
                else:
                    y = b.process_host_fmt(x, fmt=fmt, out_fmt=F64, in_scale=sc)
                np.testing.assert_array_equal(y, yt, err_msg=f"{form} call {k}")


# ---- 2. the invariant ----------------------------------------------------------------------------------------------

# per channel: (seed, taps) or None for OFF.  "flat" keeps a flagship lock-step call dithering in the fused kernel's
# stores; a shaped channel sends the call through k_dither_shape.
SETTINGS = {"off": [None] * 6, "flat": [None, (11, None), None, (13, None), (15, None), None],
            "shaped": [None, (11, None), (12, TAPS9), None, (14, [1.0]), None]}


def _sig(rng, n_ch, width):
    t = np.arange(width)
    return 0.4 * np.sin(2 * np.pi * 0.011 * (t[None, :] + 50 * np.arange(n_ch)[:, None])) + 0.01 * rng.standard_normal((n_ch, width))


class U8Expect:
    """The host quantiser for U8 per channel, with each channel's output index and error history carried along."""

    def __init__(self, pkg, settings, scale):
        self.pkg, self.settings, self.scale = pkg, settings, scale
        self.n = np.zeros(len(settings), dtype=np.int64)
        self.st = [np.zeros(16) for _ in settings]

    def __call__(self, c, y):
        s = self.settings[c]
        if s is None:
            q, _ = self.pkg.dither_quantize(y, U8, 0, scale=self.scale, kind=self.pkg.DITHER_OFF)
        else:
            q, _ = self.pkg.dither_quantize(y, U8, s[0], s[1], scale=self.scale, first_index=int(self.n[c]), state=self.st[c])
        self.n[c] += len(y)
        return q


@pytest.mark.parametrize("chain", [(44100.0, 96000.0), (8000.0, 16000.0), (16000.0, 8000.0)], ids=lambda c: "%g-%g" % c)
@pytest.mark.parametrize("dither", ["off", "flat", "shaped"])
def test_companded_bytes_are_the_s16_bytes_encoded(pkg, chain, dither):
    settings = SETTINGS[dither]
    n_ch, M = len(settings), 2048
    plan = pkg.Plan(chain[0], chain[1], M, 2.0, pkg.ATTEN_24)
    fmts = [S16, ULAW, ALAW, U8]
    sc = {S16: 32767.0, ULAW: 32767.0, ALAW: 32767.0, U8: 127.0}
    bs = {f: pkg.Batch(plan, n_ch) for f in fmts}
    twin = pkg.Batch(plan, n_ch)
    for bb in bs.values():
        for c, s in enumerate(settings):
            if s is not None:
                bb.set_dither([c], s[0], s[1])
    ex = U8Expect(pkg, settings, sc[U8])
    rng = np.random.default_rng(5)

    def check(out, yt, cnt, il, what):
        for c in range(n_ch):
            row = {f: (out[f][:cnt[c], c] if il else out[f][c, :cnt[c]]) for f in fmts}
            for f in (ULAW, ALAW):
                np.testing.assert_array_equal(row[f], encode(f, row[S16].astype(np.int64)), err_msg=f"{what} {f} ch {c}")
            np.testing.assert_array_equal(row[U8], ex(c, yt[c, :cnt[c]]), err_msg=f"{what} U8 ch {c}")

    # lock-step: host planar (the flagship narrows in the fused kernel's stores), device planar, host interleaved
    for k, form in enumerate(["host", "device", "host_il"]):
        x = _sig(rng, n_ch, M)
        yt = twin.process_host(x)
        out = {}
        for f, bb in bs.items():
            if form == "device":
                out[f] = _lockstep_device(pkg, bb, x, F64, f, out_scale=sc[f])
            elif form == "host_il":
                out[f] = bb.process_host_fmt(x.T.copy(), interleaved=True, out_fmt=f, out_scale=sc[f]).T
            else:
                out[f] = bb.process_host_fmt(x, out_fmt=f, out_scale=sc[f])
        check(out, yt, np.full(n_ch, yt.shape[1]), False, form)
    # ragged (host interleaved, device planar), then a flush of every channel
    for k, (il, dev) in enumerate([(True, False), (False, True)]):
        lens = rng.integers(0, M + 1, n_ch).astype(np.int32)
        x = _sig(rng, n_ch, M)
        yt, cnt = twin.process_ragged_fmt(x, lens, out_fmt=F64)
        out = {}
        for f, bb in bs.items():
            xin = x.T.copy() if il else x
            y, c2 = bb.process_ragged_fmt(_dev(xin) if dev else xin, lens, out_fmt=f, out_scale=sc[f], interleaved=il)
            np.testing.assert_array_equal(c2, cnt)
            out[f] = _np(y)
        check(out, yt, cnt, il, "ragged")
    chans = list(range(n_ch))
    yt, cnt = twin.flush(chans)
    out = {}
    for f, bb in bs.items():
        y, c2 = bb.flush(chans, out_fmt=f, out_scale=sc[f], device="cuda")
        np.testing.assert_array_equal(c2, cnt)
        out[f] = _np(y)
    check(out, yt, cnt, False, "flush")


# ---- 3. launch count -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("chain", [(44100.0, 96000.0), (48000.0, 44100.0)], ids=lambda c: "%g-%g" % c)
@pytest.mark.parametrize("host", [True, False])
def test_planar_conversion_adds_no_launch(pkg, chain, host):
    n_ch, M = 8, 4096
    plan = pkg.Plan(chain[0], chain[1], M, 2.0, pkg.ATTEN_24)
    rng = np.random.default_rng(3)
    launches = {}
    for fmt in (S16, ULAW):
        b = pkg.Batch(plan, n_ch)
        for l in (M, 1000, M):
            x = (rng.integers(-3000, 3000, (n_ch, l)).astype(np.int16) if fmt == S16 else _bytes(rng, (n_ch, l)))
            if host:
                b.process_host_fmt(x, fmt=fmt, out_fmt=fmt)
            else:
                _lockstep_device(pkg, b, x, fmt, fmt)
        launches[fmt] = b.kernel_launches
    assert launches[S16] == launches[ULAW], launches


# ---- 4. silence ----------------------------------------------------------------------------------------------------

SILENCE = {U8: 128, ULAW: 0xFF, ALAW: 0xD5}


@pytest.mark.parametrize("fmt", BYTE_FORMATS)
@pytest.mark.parametrize("interleaved", [False, True])
@pytest.mark.parametrize("device", [False, True])
def test_passthrough_flush_writes_encoded_zero(pkg, fmt, interleaved, device):
    n_ch = 6
    plan = pkg.Plan(16000.0, 16000.0, 1024, 2.0, pkg.ATTEN_24)
    b = pkg.Batch(plan, n_ch)
    rng = np.random.default_rng(fmt)
    b.process_ragged_fmt(_bytes(rng, (n_ch, 1024)), np.full(n_ch, 700, np.int32), fmt=fmt, out_fmt=fmt)
    named = np.array([4, 1, 2], dtype=np.int32)
    extra = np.array([9, 33, 1], dtype=np.int64)
    targets = b.channel_totals()[1][named] + extra
    cap = 40
    shape = (cap, n_ch) if interleaved else (n_ch, cap)
    y = np.full(shape, 0x5A, dtype=np.uint8)
    if device:
        y = _dev(y)
    counts = np.zeros(n_ch, dtype=np.int32)
    b._flush_into(named, targets, y, fmt, interleaved, 1.0, counts)
    y = _np(y)
    if interleaved:
        y = y.T
    for c in range(n_ch):
        k = int(extra[list(named).index(c)]) if c in named else 0
        assert counts[c] == k
        assert (y[c, :k] == SILENCE[fmt]).all(), (c, y[c, :k])
        assert (y[c, k:] == 0x5A).all(), f"channel {c}: written past its count"


# ---- 5. other routes -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("fmt", BYTE_FORMATS)
@pytest.mark.parametrize("device", [False, True])
def test_mixed_batch_matches_ordinary(pkg, fmt, device):
    M = 2048
    plans = [pkg.Plan(8000.0, 16000.0, M, 2.0, pkg.ATTEN_24), pkg.Plan(16000.0, 8000.0, M, 2.0, pkg.ATTEN_24)]
    plan_of = np.array([0, 1, 1, 0, 1, 0, 0], dtype=np.int32)
    mixed = pkg.Batch.mixed(plans, plan_of)
    rows = [np.nonzero(plan_of == p)[0] for p in range(2)]
    ords = [pkg.Batch(plans[p], len(rows[p])) for p in range(2)]
    rng = np.random.default_rng(21 + fmt)
    sc = IN_SCALE[fmt]
    for k in range(3):
        lens = rng.integers(0, M + 1, len(plan_of)).astype(np.int32)
        x = _bytes(rng, (len(plan_of), M))
        il = k == 1
        xin = x.T.copy() if il else x
        y, cnt = mixed.process_ragged_fmt(_dev(xin) if device else xin, lens, fmt=fmt, out_fmt=fmt, in_scale=sc,
                                          out_scale=1.0 / sc, interleaved=il)
        y = _np(y)
        for p in range(2):
            yo, co = ords[p].process_ragged_fmt(x[rows[p]], lens[rows[p]], fmt=fmt, out_fmt=fmt, in_scale=sc, out_scale=1.0 / sc)
            np.testing.assert_array_equal(cnt[rows[p]], co)
            for i, c in enumerate(rows[p]):
                row = y[:cnt[c], c] if il else y[c, :cnt[c]]
                np.testing.assert_array_equal(row, yo[i, :co[i]], err_msg=f"call {k} channel {c}")
    tm, cm = mixed.flush(range(len(plan_of)), out_fmt=fmt, out_scale=1.0 / sc, device="cuda" if device else None)
    tm = _np(tm)
    for p in range(2):
        to, co = ords[p].flush(range(len(rows[p])), out_fmt=fmt, out_scale=1.0 / sc)
        np.testing.assert_array_equal(cm[rows[p]], co)
        for i, c in enumerate(rows[p]):
            np.testing.assert_array_equal(tm[c, :cm[c]], to[i, :co[i]], err_msg=f"flush channel {c}")


@pytest.mark.parametrize("fmt", BYTE_FORMATS)
def test_device_all_matches_ordinary(pkg, fmt, monkeypatch):
    monkeypatch.setenv("R8BGPU_FORCE_SHARDS", "3")
    n_ch, M = 7, 2048
    plan = pkg.Plan(8000.0, 16000.0, M, 2.0, pkg.ATTEN_24)
    b, twin = pkg.Batch(plan, n_ch, pkg.DEVICE_ALL), pkg.Batch(plan, n_ch)
    assert len(b.shards()) == 3
    for bb in (b, twin):
        bb.set_dither([1, 5], 9, TAPS9)
    rng = np.random.default_rng(31 + fmt)
    sc = IN_SCALE[fmt]
    for k in range(3):
        x = _bytes(rng, (n_ch, M))
        il = k == 1
        xin = x.T.copy() if il else x
        kw = dict(fmt=fmt, out_fmt=fmt, in_scale=sc, out_scale=1.0 / sc, interleaved=il)
        np.testing.assert_array_equal(b.process_host_fmt(xin, **kw), twin.process_host_fmt(xin, **kw), err_msg=f"call {k}")
    lens = rng.integers(0, M + 1, n_ch).astype(np.int32)
    x = _bytes(rng, (n_ch, M))
    y, cnt = b.process_ragged_fmt(x, lens, fmt=fmt, out_fmt=fmt, in_scale=sc, out_scale=1.0 / sc)
    yt, cnt_t = twin.process_ragged_fmt(x, lens, fmt=fmt, out_fmt=fmt, in_scale=sc, out_scale=1.0 / sc)
    np.testing.assert_array_equal(cnt, cnt_t)
    np.testing.assert_array_equal(y, yt)
    tf, cf = b.flush(range(n_ch), out_fmt=fmt, out_scale=1.0 / sc)
    tt, ct = twin.flush(range(n_ch), out_fmt=fmt, out_scale=1.0 / sc)
    np.testing.assert_array_equal(cf, ct)
    np.testing.assert_array_equal(tf, tt)


# ---- 6. mu-law round trip ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("device", [False, True])
def test_passthrough_ulaw_round_trip(pkg, device):
    n_ch = 3
    plan = pkg.Plan(8000.0, 8000.0, 512, 2.0, pkg.ATTEN_24)
    b = pkg.Batch(plan, n_ch)
    codes = np.arange(256, dtype=np.uint8)
    x = np.stack([codes, codes[::-1], np.roll(codes, 77)])
    y = _lockstep_device(pkg, b, x, ULAW, ULAW) if device else b.process_host_fmt(x, fmt=ULAW, out_fmt=ULAW)
    want = np.where(x == 0x7F, 0xFF, x)
    np.testing.assert_array_equal(y, want)


def test_format_8_refused(pkg):
    plan = pkg.Plan(8000.0, 16000.0, 512, 2.0, pkg.ATTEN_24)
    b = pkg.Batch(plan, 2)
    x = np.zeros((2, 512), dtype=np.uint8)
    y = np.zeros((2, b.plan.max_out_len), dtype=np.uint8)
    for fi, fo in ((8, U8), (U8, 8)):
        with pytest.raises(pkg.R8bGpuError, match="unknown sample format"):
            b.process_fmt(pkg.Buffer.make(x.ctypes.data, fi, False, 512), 512,
                          pkg.Buffer.make(y.ctypes.data, fo, False, y.shape[1]), y.shape[1], host=True)
