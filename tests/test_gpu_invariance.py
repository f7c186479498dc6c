"""GPU: results do not depend on the caller's buffer layout, the batch width, or which exact kernel path runs -- bit for bit.

None of these variations changes an output's arithmetic: tile geometry follows stream positions only (the parity of the
stream index, never the pointer), so any differing bit is a bug.  Every comparison is of bytes, against a baseline that
the parity tests already hold to the reference: a twin batch fed the same history through the host form (staging rows
the engine aligns itself), a narrow batch, or the default kernel path.

Caller buffers are built by `Region`: a device buffer larger than the block, filled with a sentinel bit pattern, with the
block at an element offset and a row stride inside it.  After a call the whole output buffer must equal the sentinel
image with exactly the returned samples written, and the input buffer must be unchanged.  Only legal layouts occur:
every pointer is aligned to its element size (any byte for packed 24-bit samples)."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from test_gpu_formats import pack24, unpack24
from test_gpu_ragged_formats import FORMATS, ragged_lens, samples

pytestmark = pytest.mark.gpu

F64, F32, S16, S24, S32 = 0, 1, 2, 3, 4
ESIZE = {F64: 8, F32: 4, S16: 2, S24: 3, S32: 4}
NPTYPE = {F64: np.float64, F32: np.float32, S16: np.int16, S24: np.int32, S32: np.int32}
SENTINEL = {F64: np.array([0x7FF4DEADBEEF1234], np.uint64), F32: np.array([0x7FA0BEEF], np.uint32),
            S16: np.array([0x5A5B], np.uint16), S32: np.array([0x13579BDF], np.uint32),
            S24: np.array([0xA5, 0x5A, 0xC3], np.uint8)}
LARGE = "k_bcl_gather+k_bcl_conv+k_bcl_scatter"

# name -> (src, dst, MaxInLen, TransBand, R8B_EXTFFT).  The fused kernels read a tile from the caller's block only when
# its whole 4096-sample FFT window lies in the block: MaxInLen 16384 gives every full call such tiles.
CHAINS = {
    "44100-96000": (44100.0, 96000.0, 16384, 2.0, 0),
    "48000-44100": (48000.0, 44100.0, 16384, 2.0, 0),
    "96000-44100": (96000.0, 44100.0, 16384, 2.0, 0),
    "44100-88200": (44100.0, 88200.0, 16384, 2.0, 0),
    "44100-176400": (44100.0, 176400.0, 16384, 2.0, 0),
    "48000-47999": (48000.0, 47999.0, 16384, 2.0, 0),
    "48000-48001": (48000.0, 48001.0, 16384, 2.0, 0),
    "48000-47990": (48000.0, 47990.0, 16384, 2.0, 0),
    "192000-44100": (192000.0, 44100.0, 16384, 2.0, 0),
    "2822400-44100": (2822400.0, 44100.0, 65536, 2.0, 0),
    "96000-48000": (96000.0, 48000.0, 4096, 2.0, 0),
    "48000-32000": (48000.0, 32000.0, 4096, 2.0, 0),
    "44100-132300": (44100.0, 132300.0, 4096, 2.0, 0),
    "44100-2822400-extfft": (44100.0, 2822400.0, 2048, 2.0, 1),
    "large-tile": (48000.0, 16000.0, 16384, 0.5, 0),
}


def make_plan(pkg, chain, max_in=None):
    src, dst, m, tb, ext = CHAINS[chain]
    return pkg.Plan(src, dst, m if max_in is None else max_in, tb, pkg.ATTEN_24, extfft=ext)


def kernels(batch):
    """(first, last) kernel of the chain as the batch runs it now."""
    names = [k for k, _ in batch.stage_kernels() if k != "(fused)"]
    return names[0], names[-1]


def out_step(plan):
    st = [s["out_step"] for s in plan.stages() if s["name"] == "frac_whole"]
    return st[0] if st else 0


class Region:
    """A device buffer holding n_ch x width samples of format fmt at byte `start`, rows `stride` samples apart (planar:
    one row per channel; interleaved: one row per sample index, the channels in its first n_ch columns); every other
    byte holds the sentinel."""

    def __init__(self, fmt, n_ch, width, start, stride, interleaved=False):
        import torch
        e = ESIZE[fmt]
        rows, cols = (width, n_ch) if interleaved else (n_ch, width)
        assert stride >= cols and start % (1 if fmt == S24 else e) == 0, "legal layouts only"
        self.fmt, self.e, self.n_ch, self.width, self.start, self.stride, self.inter = fmt, e, n_ch, width, start, stride, interleaved
        nbytes = start + (max(rows - 1, 0) * stride + cols) * e + 48
        self.image = np.resize(SENTINEL[fmt].view(np.uint8), nbytes)
        c, i, k = np.ogrid[:n_ch, :width, :e]
        self.idx = start + ((i * stride + c) if interleaved else (c * stride + i)) * e + k   # [n_ch, width, e]
        self.dev = torch.from_numpy(self.image).cuda()
        self.ptr = self.dev.data_ptr() + start

    def raw(self, v):
        """Bytes [n_ch, n, e] of planar values v (int32 values for S24)."""
        if self.fmt == S24:
            return pack24(v)
        return np.ascontiguousarray(v.astype(NPTYPE[self.fmt])).view(np.uint8).reshape(v.shape + (self.e,))

    def fill(self, v):
        """Write planar values [n_ch, width] into the block."""
        import torch
        self.image = self.image.copy()
        self.image[self.idx] = self.raw(v)
        self.dev = torch.from_numpy(self.image).cuda()
        self.ptr = self.dev.data_ptr() + self.start
        return self

    def row_phase(self, c):
        """Byte alignment mod 16 of channel c's first sample."""
        return (self.ptr + (c * self.e if self.inter else c * self.stride * self.e)) % 16

    def buffer(self, pkg, scale=1.0):
        return pkg.Buffer.make(self.ptr, self.fmt, self.inter, self.stride, scale)

    def got(self):
        return self.dev.cpu().numpy()

    def assert_untouched(self, what="the input"):
        assert np.array_equal(self.got(), self.image), what + " was written"

    def assert_holds(self, want, ctx=""):
        """want: per channel, the samples expected at [0, len) of the channel (planar values; int32 for S24).  Compares
        the samples bit for bit, then every other byte of the buffer against the sentinel."""
        got = self.got()
        for c, w in enumerate(want):
            n = len(w)
            g = got[self.idx[c, :n]]
            wb = self.raw(np.asarray(w).reshape(1, -1))[0]
            if not np.array_equal(g, wb):
                bad = np.nonzero(np.any(g != wb, axis=1))[0]
                i = int(bad[0])
                gv = unpack24(g[i]) if self.fmt == S24 else g[i].view(NPTYPE[self.fmt])[0]
                pytest.fail("%s: channel %d differs at %d of %d samples (first at %d, %d differ, got %r want %r, row phase %d)"
                            % (ctx, c, i, n, i, len(bad), gv, np.asarray(w)[i], self.row_phase(c)))
        expect = self.image.copy()
        for c, w in enumerate(want):
            if len(w):
                expect[self.idx[c, :len(w)]] = self.raw(np.asarray(w).reshape(1, -1))[0]
        diff = np.nonzero(got != expect)[0]
        assert len(diff) == 0, "%s: %d sentinel bytes overwritten, first at byte %d (block starts at %d)" % (
            ctx, len(diff), diff[0], self.start)


def fail_ctx(call, plan, total):
    return "call %d, output total before it %d, out_step %d" % (call, total, out_step(plan))


def sync():
    import torch
    torch.cuda.synchronize()


def use_torch_stream(batch):
    import torch
    batch.set_stream(torch.cuda.current_stream().cuda_stream)


# ---- A. lock-step fp64 device calls ------------------------------------------------------------------------------------

# chain -> (first kernel, last kernel, environment)
LOCKSTEP = {
    "44100-96000": ("k_up2_frac2", "k_up2_frac2", {}),
    "48000-44100": ("k_up2_frac2", "k_up2_frac2", {}),
    "96000-44100": ("k_up2_frac2", "k_up2_frac2", {}),               # the 1x pair reads the caller's block
    "44100-88200": ("k_up2_frac2<copy>", "k_up2_frac2<copy>", {}),
    "44100-176400": ("k_up2_frac2<copy>", "k_hbup", {}),
    "48000-47999": ("k_up2_frac", "k_up2_frac", {}),
    "192000-44100": ("k_hbdown", "k_up2_frac2", {}),                 # the 1x pair writes the caller's buffer
    "2822400-44100": ("k_hbdown_cascade", "k_blockconv", {}),
    "96000-48000": ("k_blockconv", "k_blockconv", {}),
    "48000-32000": ("k_blockconv", "k_blockconv", {}),
    "44100-132300": ("k_blockconv", "k_blockconv", {}),
    "44100-2822400-extfft": ("k_up2_frac2<copy>", "k_hbup_cascade", {}),
    "large-tile": (LARGE, LARGE, {}),
    "44100-96000-nofusion": ("k_blockconv", "k_frac<false>", {"R8BGPU_NO_FUSION": "1"}),
    "48000-47999-nofusion": ("k_blockconv", "k_frac<true>", {"R8BGPU_NO_FUSION": "1"}),
}

# up-factor of the fused pair (UP template parameter): the BlockConv stage in front of the interpolator
FUSED_UP = {"44100-96000": 2, "48000-44100": 2, "96000-44100": 1, "192000-44100": 1}


def lens_for(max_in):
    return [max_in, 0, 1, 7, max_in, 333, max_in - 1, max_in, 2 * (max_in // 3) + 1]


def test_the_1x_pair_is_first_for_some_rate_pair(pkg):
    """96000 -> 44100 plans BlockConv 1x -> whole-step interpolator: the 1x fused pair reads the caller's block."""
    st = make_plan(pkg, "96000-44100").stages()
    assert [(s["name"], s["up"], s["down"]) for s in st[:2]] == [("blockconv", 1, 1), ("frac_whole", 1, 1)]


@pytest.mark.parametrize("chain", list(LOCKSTEP))
def test_lockstep_device_layouts(pkg, chain, monkeypatch):
    first, last, env = LOCKSTEP[chain]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    base = chain.replace("-nofusion", "")
    plan = make_plan(pkg, base)
    n_ch, max_in, cap = 3, plan.max_in_len, plan.max_out_len
    a, b = pkg.Batch(plan, n_ch, 0), pkg.Batch(plan, n_ch, 0)
    assert kernels(a) == (first, last), a.stage_kernels()
    if base in FUSED_UP and not env:
        i = [k for k, _ in a.stage_kernels()].index("k_up2_frac2")
        assert plan.stages()[i]["up"] == FUSED_UP[base]
    use_torch_stream(a)
    rng = np.random.default_rng(len(chain))
    total = 0
    for call, l in enumerate(lens_for(max_in)):
        x = rng.uniform(-1.0, 1.0, size=(n_ch, l))
        in_stride = (max_in, max_in + 1, max_in + 3)[call % 3]
        out_stride = (cap, cap + 1, cap + 5)[(call + 1) % 3]
        xi = Region(F64, n_ch, l, 8 * (call % 4), in_stride).fill(x)
        yo = Region(F64, n_ch, cap, 8 * ((3 * call + 1) % 4), out_stride)
        n = a.process_ptr(xi.ptr, in_stride, l, yo.ptr, out_stride, cap)
        want = b.process_host(x)
        sync()
        assert n == want.shape[1]
        yo.assert_holds(list(want), fail_ctx(call, plan, total))
        xi.assert_untouched()
        total += n
    assert total > 0


# ---- B. ragged fp64 device calls ---------------------------------------------------------------------------------------

RAGGED = {
    "44100-96000": ("k_blockconv<ragged>", "k_frac<false,ragged>"),
    "192000-44100": ("k_hbdown<ragged>", "k_frac<false,ragged>"),
    "44100-176400": ("k_blockconv<ragged>", "k_hbup<ragged>"),
    "48000-47999": ("k_blockconv<ragged>", "k_frac<true,ragged>"),
    "large-tile": ("k_bcl_gather_ragged+k_bcl_conv+k_bcl_scatter_ragged",) * 2,
}


def ragged_raw(pkg, batch, xi, in_stride, lens, yo, out_stride, cap):
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    counts = np.full(batch.n_channels, -7, dtype=np.int32)
    use_torch_stream(batch)
    rc = pkg.lib().r8bgpu_batch_process_ragged(batch._h, C.c_void_p(xi.ptr), in_stride, lens.ctypes.data,
                                               C.c_void_p(yo.ptr), out_stride, cap, counts.ctypes.data)
    if rc < 0:
        raise pkg.R8bGpuError(pkg._err())
    return counts


@pytest.mark.parametrize("chain", list(RAGGED))
def test_ragged_device_layouts(pkg, chain):
    plan = make_plan(pkg, chain)
    n_ch, max_in, cap = 4, plan.max_in_len, plan.max_out_len
    a, b = pkg.Batch(plan, n_ch, 0), pkg.Batch(plan, n_ch, 0)
    use_torch_stream(a)
    rng = np.random.default_rng(100 + len(chain))
    # a lock-step call first: the ragged calls then refill the links the fused kernels kept in shared memory
    x = rng.uniform(-1.0, 1.0, size=(n_ch, max_in))
    xi = Region(F64, n_ch, max_in, 8, max_in + 1).fill(x)
    yo = Region(F64, n_ch, cap, 24, cap + 1)
    n = a.process_ptr(xi.ptr, max_in + 1, max_in, yo.ptr, cap + 1, cap)
    want = b.process_host(x)
    sync()
    yo.assert_holds(list(want), "lock-step call")
    totals = np.full(n_ch, n)
    diverged = 0
    for call, lens in enumerate(ragged_lens(rng, 5, n_ch, max_in)):
        width = max(int(lens.max()), 1)
        x = rng.uniform(-1.0, 1.0, size=(n_ch, width))
        in_stride = (width, width + 1, width + 3)[call % 3]
        out_stride = (cap, cap + 1, cap + 5)[(call + 2) % 3]
        xi = Region(F64, n_ch, width, 8 * (call % 4), in_stride).fill(x)
        yo = Region(F64, n_ch, cap, 8 * ((call + 3) % 4), out_stride)
        counts = ragged_raw(pkg, a, xi, in_stride, lens, yo, out_stride, cap)
        ys = b.process_ragged([x[c, :lens[c]].copy() for c in range(n_ch)])
        sync()
        assert list(counts) == [len(y) for y in ys]
        yo.assert_holds(ys, "ragged call %d, totals before it %s" % (call, list(totals)))
        xi.assert_untouched()
        totals += counts
        if a.channel_groups > 1:
            assert kernels(a) == RAGGED[chain], a.stage_kernels()
            diverged += 1
    assert diverged > 0


# ---- C. typed device buffers -------------------------------------------------------------------------------------------

def planar_values(fkey, raw, interleaved):
    v = unpack24(raw) if fkey == "s24" else raw
    return v.T if interleaved else v


def typed_starts(fkey, call, e):
    """Byte offset of the block: element offsets 0..3; packed 24-bit rows also at every byte phase."""
    return (7 * call) % 16 if fkey == "s24" else e * (call % 4)


TYPED_LOCKSTEP = ["44100-96000", "96000-44100", "192000-44100", "48000-47999"]


@pytest.mark.parametrize("interleaved", [False, True], ids=["planar", "interleaved"])
@pytest.mark.parametrize("fkey", list(FORMATS))
@pytest.mark.parametrize("chain", TYPED_LOCKSTEP)
def test_typed_lockstep_device_layouts(pkg, chain, fkey, interleaved):
    """process_fmt on caller buffers equals process_host_fmt (rows staged by the engine), bit for bit."""
    fmt, in_scale, out_scale = FORMATS[fkey]
    plan = make_plan(pkg, chain)
    n_ch, max_in, cap = 5, plan.max_in_len, plan.max_out_len
    a, b = pkg.Batch(plan, n_ch, 0), pkg.Batch(plan, n_ch, 0)
    use_torch_stream(a)
    rng = np.random.default_rng(7 * len(chain) + fmt)
    phases, total = set(), 0
    for call, l in enumerate([max_in, 1, 333, max_in, 0, max_in - 1, 2001, max_in]):
        v = samples(fkey, n_ch, l, rng)
        e = ESIZE[fmt]
        if interleaved:
            in_stride, out_stride = n_ch + 3, n_ch + 3
        else:
            in_stride, out_stride = (max_in + 1, max_in + 3)[call % 2], (cap + 1, cap + 3)[call % 2]
        xi = Region(fmt, n_ch, l, typed_starts(fkey, call, e), in_stride, interleaved).fill(v)
        yo = Region(fmt, n_ch, cap, typed_starts(fkey, call + 3, e), out_stride, interleaved)
        phases.update(xi.row_phase(c) for c in range(n_ch))
        n = a.process_fmt(xi.buffer(pkg, in_scale), l, yo.buffer(pkg, out_scale), cap, host=False)
        raw = v.T if interleaved else v
        raw = np.ascontiguousarray(pack24(raw) if fkey == "s24" else raw)
        want = planar_values(fkey, b.process_host_fmt(raw, interleaved=interleaved, in_scale=in_scale,
                                                      out_scale=out_scale, fmt=fmt, out_fmt=fmt), interleaved)
        sync()
        assert n == want.shape[1]
        yo.assert_holds(list(want), fail_ctx(call, plan, total))
        xi.assert_untouched()
        total += n
    if fkey == "s24" and not interleaved:
        assert phases == set(range(16)), sorted(phases)


@pytest.mark.parametrize("interleaved", [False, True], ids=["planar", "interleaved"])
@pytest.mark.parametrize("fkey", list(FORMATS))
@pytest.mark.parametrize("chain", ["44100-96000", "192000-44100"])
def test_typed_ragged_device_layouts(pkg, chain, fkey, interleaved):
    """The device form of the typed ragged call on caller buffers equals its host form, bit for bit."""
    fmt, in_scale, out_scale = FORMATS[fkey]
    plan = make_plan(pkg, chain)
    n_ch, max_in, cap = 5, plan.max_in_len, plan.max_out_len
    a, b = pkg.Batch(plan, n_ch, 0), pkg.Batch(plan, n_ch, 0)
    rng = np.random.default_rng(11 * len(chain) + fmt)
    x = rng.uniform(-0.9, 0.9, size=(n_ch, max_in))
    a.process_host(x)
    b.process_host(x)
    L = pkg.lib()
    for call, lens in enumerate(ragged_lens(rng, 4, n_ch, max_in)):
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        width = int(lens.max())
        v = samples(fkey, n_ch, width, rng)
        e = ESIZE[fmt]
        if interleaved:
            in_stride, out_stride = n_ch + 3, n_ch + 3
        else:
            in_stride, out_stride = width + 1 + 2 * (call % 2), cap + 1 + 2 * (call % 2)
        xi = Region(fmt, n_ch, width, typed_starts(fkey, call, e), in_stride, interleaved).fill(v)
        yo = Region(fmt, n_ch, cap, typed_starts(fkey, call + 2, e), out_stride, interleaved)
        counts = np.full(n_ch, -7, dtype=np.int32)
        use_torch_stream(a)
        rc = L.r8bgpu_batch_process_ragged_fmt(a._h, C.byref(xi.buffer(pkg, in_scale)), lens.ctypes.data,
                                               C.byref(yo.buffer(pkg, out_scale)), cap, counts.ctypes.data)
        assert rc >= 0, pkg._err()
        raw = v.T if interleaved else v
        raw = np.ascontiguousarray(pack24(raw) if fkey == "s24" else raw)
        y, cb = b.process_ragged_fmt(raw, lens, interleaved=interleaved, in_scale=in_scale, out_scale=out_scale,
                                     fmt=fmt, out_fmt=fmt)
        sync()
        assert np.array_equal(counts, cb)
        want = planar_values(fkey, y, interleaved)
        yo.assert_holds([want[c, :cb[c]] for c in range(n_ch)], "ragged call %d" % call)
        xi.assert_untouched()


@pytest.mark.parametrize("chain", ["44100-96000", "48000-44100", "96000-44100", "44100-88200"])
def test_float32_gather_equals_fp64_input(pkg, chain):
    """float32 samples at scale 1 (widened while the fused kernel gathers them, path 3) give the same fp64 output as
    fp64 input holding the same values (plain or bulk-copied loads, paths 1 and 2)."""
    plan = make_plan(pkg, chain)
    n_ch, max_in, cap = 4, plan.max_in_len, plan.max_out_len
    a, b = pkg.Batch(plan, n_ch, 0), pkg.Batch(plan, n_ch, 0)
    use_torch_stream(a)
    use_torch_stream(b)
    rng = np.random.default_rng(3 + len(chain))
    for call, l in enumerate([max_in, 777, max_in, 1, max_in - 1]):
        v = rng.uniform(-1.0, 1.0, size=(n_ch, l)).astype(np.float32)
        xf = Region(F32, n_ch, l, 4 * (call % 4), max_in + 1 + 2 * (call % 2)).fill(v)
        xd = Region(F64, n_ch, l, 8 * (call % 4), max_in + 1).fill(v.astype(np.float64))
        yf = Region(F64, n_ch, cap, 0, cap)
        yd = Region(F64, n_ch, cap, 8, cap + 1)
        n = a.process_fmt(xf.buffer(pkg), l, yf.buffer(pkg), cap, host=False)
        nd = b.process_ptr(xd.ptr, max_in + 1, l, yd.ptr, cap + 1, cap)
        sync()
        assert n == nd
        want = yd.got()[yd.idx[:, :nd]].reshape(-1).view(np.float64).reshape(n_ch, nd)
        yf.assert_holds(list(want), "call %d" % call)


# ---- D. batch width and the persistent loop ----------------------------------------------------------------------------

# chain -> (MaxInLen, typed (in fmt, out fmt, out scale) or None)
WIDE = {
    "44100-96000": (4096, None),
    "48000-44100": (4096, None),
    "192000-44100": (4096, None),
    "44100-88200": (4096, None),
    "48000-47999": (4096, None),
    "2822400-44100": (16384, None),
    "44100-2822400-extfft": (128, None),     # 8192 outputs per channel and call
    "44100-96000-f32-s16": (4096, (F32, S16, 20000.0)),
}


def wide_call(pkg, batch, x, typed, device):
    """One lock-step call of [n, l] samples: fp64, or the typed (planar) form; device tensors or host arrays."""
    import torch
    n_ch, l = x.shape
    cap = batch.plan.max_out_len
    if typed is None:
        if device:
            return batch.process(torch.from_numpy(x).cuda()).cpu().numpy()
        return batch.process_host(x)
    fi, fo, scale = typed
    xs = np.ascontiguousarray(x.astype(NPTYPE[fi]))
    if not device:
        return batch.process_host_fmt(xs, out_fmt=fo, out_scale=scale)
    dx = torch.from_numpy(xs).cuda()
    dy = torch.zeros((n_ch, cap), dtype=torch.int16, device="cuda")
    assert fo == S16
    use_torch_stream(batch)
    n = batch.process_fmt(pkg.Buffer.make(dx.data_ptr(), fi, False, l), l,
                          pkg.Buffer.make(dy.data_ptr(), fo, False, cap, scale), cap, host=False)
    return dy[:, :n].cpu().numpy()


@pytest.mark.parametrize("chain", list(WIDE))
def test_wide_batch_is_the_narrow_batch(pkg, chain, monkeypatch):
    """6 n_sm + 5 channels: every channel owns at least one tile per call, so each of the persistent kernel's 2 n_sm
    half-CTAs runs at least 3 tiles.  Channels {0, 1, n/2, n-2, n-1} get the rows a 5-channel batch gets; the host pipeline
    in 1, 3 and 8 channel groups gives the device form's bits."""
    import torch
    base = chain.replace("-f32-s16", "")
    max_in, typed = WIDE[chain]
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    n = 6 * n_sm + 5
    pick = [0, 1, n // 2, n - 2, n - 1]
    plan = make_plan(pkg, base, max_in)
    wide, narrow = pkg.Batch(plan, n, 0), pkg.Batch(plan, 5, 0)
    assert kernels(wide)[0] == LOCKSTEP[base][0], wide.stage_kernels()
    if kernels(wide)[0].startswith("k_up2_frac2"):
        assert n >= 6 * n_sm   # units >= channels >= 3 per half-CTA of the min(units / 2, n_sm)-CTA grid
    # full calls until the chain's first output (its latency), then the 4 calls that matter
    counts = plan.simulate([max_in] * 64)
    warm = next(i for i, v in enumerate(counts) if v)
    lens = [max_in] * warm + [max_in, max_in - 3, max_in, max_in // 2 + 1]

    def inputs():
        rng = np.random.default_rng(len(chain))
        for l in lens:
            x = rng.uniform(-0.9, 0.9, size=(n, l))
            yield x if typed is None else x.astype(np.float32).astype(np.float64)

    digests, produced = [], 0
    for x in inputs():
        yw = wide_call(pkg, wide, x, typed, True)
        yn = wide_call(pkg, narrow, np.ascontiguousarray(x[pick]), typed, False)
        assert yw.shape == (n, yn.shape[1])
        assert yw[pick].tobytes() == yn.tobytes()
        assert np.all(np.isfinite(yw.astype(np.float64)))
        digests.append((yw.shape, hashlib.sha256(yw.tobytes()).hexdigest()))
        produced += yw.shape[1]
    assert produced > 0
    del wide
    for groups in ("1", "3", "8"):    # 8 is the default; each group keeps >= 32 channels here, so none is merged
        monkeypatch.setenv("R8BGPU_HOST_GROUPS", groups)
        h = pkg.Batch(plan, n, 0)
        for x, d in zip(inputs(), digests):
            yh = wide_call(pkg, h, x, typed, False)
            assert (yh.shape, hashlib.sha256(yh.tobytes()).hexdigest()) == d, groups
        del h


# ---- E. exact alternative paths: knob against default ------------------------------------------------------------------

KNOBS = [
    ("no-bulk-copy", {"R8BGPU_F2_FLAGS": "4"}, ["44100-96000", "48000-44100", "192000-44100"]),
    ("ping-pong", {"R8BGPU_F2_FLAGS": "7"}, ["44100-96000", "48000-44100", "192000-44100"]),
    ("fma-glog0", {"R8BGPU_F2_FLAGS": "2", "R8BGPU_F2_GLOG": "0"}, ["44100-96000", "48000-44100"]),
    ("fma-glog1", {"R8BGPU_F2_FLAGS": "2", "R8BGPU_F2_GLOG": "1"}, ["44100-96000", "48000-44100"]),
    ("fma-glog2", {"R8BGPU_F2_FLAGS": "2", "R8BGPU_F2_GLOG": "2"}, ["44100-96000", "48000-44100"]),
    ("fma-no-stage", {"R8BGPU_F2_FLAGS": "2", "R8BGPU_NO_STAGE": "1"}, ["44100-96000", "48000-44100"]),
    ("no-stage", {"R8BGPU_NO_STAGE": "1"}, ["44100-96000", "48000-44100"]),
    ("mbu2", {"R8BGPU_F2_MBU": "2"}, ["44100-96000", "48000-44100", "192000-44100"]),
    ("mbu4", {"R8BGPU_F2_MBU": "4"}, ["44100-96000", "48000-44100", "192000-44100"]),
    ("mbu6", {"R8BGPU_F2_MBU": "6"}, ["44100-96000", "48000-44100", "192000-44100"]),
    ("no-align", {"R8BGPU_NO_ALIGN": "1"}, ["44100-96000"]),
    ("bank-global", {"R8BGPU_BANK_GLOBAL": "1"}, ["48000-47999", "48000-48001", "48000-47990"]),
    ("poly-single", {"R8BGPU_POLY_SINGLE": "1"}, ["48000-47999", "48000-48001", "48000-47990"]),
]
KNOB_CASES = [(name, env, chain) for name, env, chains in KNOBS for chain in chains]


def run_chain(pkg, chain, env, monkeypatch, n_ch=3, lens=None, device_layout=False):
    """Outputs of a fresh batch fed seeded lock-step calls with env set for its whole life; returns (y, kernels)."""
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, v)
        plan = make_plan(pkg, chain)
        b = pkg.Batch(plan, n_ch, 0)
        max_in = plan.max_in_len
        rng = np.random.default_rng(99)
        ys = []
        for call, l in enumerate(lens or lens_for(max_in)):
            x = rng.uniform(-1.0, 1.0, size=(n_ch, l))
            if device_layout:   # odd offsets and strides: the rows of the caller's buffer at every 8-byte phase
                use_torch_stream(b)
                cap = plan.max_out_len
                xi = Region(F64, n_ch, l, 8 * (call % 2), max_in + 1).fill(x)
                yo = Region(F64, n_ch, cap, 8 * ((call + 1) % 2), cap + 1)
                k = b.process_ptr(xi.ptr, max_in + 1, l, yo.ptr, cap + 1, cap)
                ys.append(yo.got()[yo.idx[:, :k]].reshape(-1).view(np.float64).reshape(n_ch, k))
            else:
                ys.append(b.process_host(x))
        return np.concatenate(ys, axis=1), b.stage_kernels()


@pytest.mark.parametrize("name,env,chain", KNOB_CASES, ids=["%s-%s" % (n, c) for n, _, c in KNOB_CASES])
def test_knob_is_bit_exact(pkg, name, env, chain, monkeypatch):
    want, k0 = run_chain(pkg, chain, {}, monkeypatch)
    got, k1 = run_chain(pkg, chain, env, monkeypatch)
    assert k1 == k0, (k0, k1)     # the same kernels run: the knob picks a variant inside them
    assert got.shape == want.shape and want.shape[1] > 0
    if got.tobytes() != want.tobytes():
        c, i = [int(v[0]) for v in np.nonzero(got.view(np.int64) != want.view(np.int64))]
        pytest.fail("%s: channel %d first differs at output %d (phase %d of out_step %d): %r vs %r"
                    % (name, c, i, i % max(out_step(make_plan(pkg, chain)), 1), out_step(make_plan(pkg, chain)),
                       got[c, i], want[c, i]))
    if name == "no-align":   # the phase shift also moves where rows fall in a caller's buffer
        g2, _ = run_chain(pkg, chain, env, monkeypatch, device_layout=True)
        w2, _ = run_chain(pkg, chain, {}, monkeypatch, device_layout=True)
        assert g2.tobytes() == w2.tobytes() == want.tobytes()


def hbup_tile_width(taps, budget, fuse_last2):
    """k_hbup_cascade's tile width for a shared-memory budget in doubles (the host's choice, restated)."""
    cl = len(taps)
    lo, hi = [0] * (cl + 1), [0] * (cl + 1)
    for k in range(cl - 1, -1, -1):
        lo[k] = (lo[k + 1] + 1) // 2 + taps[k] - 1
        hi[k] = ((hi[k + 1] - 1) // 2 if hi[k + 1] >= 1 else -1) + taps[k] + 1
    nbuf = cl - 1 if fuse_last2 else cl
    halo = sum(lo[k] + hi[k] + 8 for k in range(nbuf))
    w = max(((budget * 4) // 5 - halo) // ((1 << nbuf) - 1), 0) & ~31
    return min(max(w, 32), 1024)


def hbdown_tile_width(taps, budget):
    """k_hbdown_cascade's tile width for a shared-memory budget in doubles (the host's choice, restated)."""
    n = len(taps)
    back = [0] * (n + 1)
    for s in range(n - 1, -1, -1):
        back[s] = 2 * back[s + 1] + 2 * taps[s] - 1
    best = 0
    for w in (8, 16, 32, 64, 128, 256, 512, 1024):
        if sum(2 * ((((w - 1) << (n - s)) + 2 * back[s] + 1) // 2 + 2) for s in range(n)) <= budget:
            best = w
    return best


@pytest.mark.parametrize("chain,knob,budgets", [("44100-2822400-extfft", "R8BGPU_HB_SMEM_DOUBLES", (2000, 14000)),
                                                ("2822400-44100", "R8BGPU_HBD_SMEM_DOUBLES", (3200, 25000))])
def test_cascade_tile_width_is_bit_exact(pkg, chain, knob, budgets, monkeypatch):
    """Two shared-memory budgets that give the half-band cascade different tile widths.  Neither stage_kernels() nor
    the launch count shows a tile width (one launch per call whatever its grid), so the widths are restated from the
    host's rule on the plan's tap counts and checked to differ."""
    plan = make_plan(pkg, chain)
    taps = [s["kernel_len"] for s in plan.stages() if s["name"] in ("hbup", "hbdown")]
    if knob == "R8BGPU_HB_SMEM_DOUBLES":
        for fl2 in (False, True):
            assert hbup_tile_width(taps, budgets[0], fl2) != hbup_tile_width(taps, budgets[1], fl2)
        lens = [2048, 1, 777, 0, 2048, 2047, 2048]
    else:
        ws = [hbdown_tile_width(taps, b) for b in budgets]
        assert 0 < ws[0] < ws[1], ws
        lens = [65536, 1, 777, 0, 65536, 65535, 9999, 65536]
    want, k0 = run_chain(pkg, chain, {}, monkeypatch, lens=lens)
    kname = "k_hbup_cascade" if knob == "R8BGPU_HB_SMEM_DOUBLES" else "k_hbdown_cascade"
    assert kname in [k for k, _ in k0], k0
    for budget in budgets:
        got, k1 = run_chain(pkg, chain, {knob: str(budget)}, monkeypatch, lens=lens)
        assert k1 == k0
        assert got.shape == want.shape and got.tobytes() == want.tobytes(), budget
