"""GPU: independent streams with typed buffers -- r8bgpu_batch_process_ragged_fmt (device) and
r8bgpu_batch_process_host_ragged_fmt (host), through Batch.process_ragged_fmt and the raw C-ABI.

The typed calls must equal, bit for bit, "the fp64 ragged path on host-widened input + the C cast in numpy" (the
conversions of oneshot<Tin,Tout>(), CDSPResampler.h:592-651), write nothing past each channel's count, leave the input
alone, and refuse bad calls without changing the batch."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_formats import c_cast, pack24, unpack24

pytestmark = pytest.mark.gpu

LARGE = "k_bcl_gather+k_bcl_conv+k_bcl_scatter"
# (src, dst, MaxInLen, TransBand)
CHAINS = {
    "44100-96000": (44100.0, 96000.0, 4096, 2.0),     # fused 2x pair in lock-step: its link ring is refilled
    "48000-44100": (48000.0, 44100.0, 4096, 2.0),
    "192000-44100": (192000.0, 44100.0, 4096, 2.0),   # half-band decimator first
    "large-tile": (48000.0, 16000.0, 16384, 0.5),     # 0.5 % transition band: large-tile BlockConvolver
    "passthrough": (48000.0, 48000.0, 4096, 2.0),
}
# name -> (format, in_scale, out_scale)
FORMATS = {"s16": (2, 1.0, 1.0), "s24": (3, 2.0 ** -23, 2.0 ** 23), "s32": (4, 2.0 ** -31, 2.0 ** 31),
           "f32": (1, 1.0, 1.0), "f64": (0, 0.5, 3.0)}


def samples(fkey, n_ch, width, rng):
    """Values of format fkey, [n_ch, width] (int32 for s24: the values before packing)."""
    if fkey == "s16":
        return rng.integers(-20000, 20000, size=(n_ch, width), dtype=np.int16)
    if fkey == "s24":
        return rng.integers(-(1 << 22), 1 << 22, size=(n_ch, width), dtype=np.int32)
    if fkey == "s32":
        return rng.integers(-(1 << 30), 1 << 30, size=(n_ch, width), dtype=np.int32)
    x = rng.uniform(-0.9, 0.9, size=(n_ch, width))
    return x.astype(np.float32) if fkey == "f32" else x


def to_raw(fkey, v, interleaved):
    """The caller's buffer: planar [n_ch, width] or interleaved [width, n_ch] (packed [..., 3] for s24)."""
    v = v.T if interleaved else v
    return np.ascontiguousarray(pack24(v) if fkey == "s24" else v)


def from_raw(fkey, y, interleaved):
    """Planar values [n_ch, cap] of a returned buffer."""
    v = unpack24(y) if fkey == "s24" else y
    return v.T if interleaved else v


def narrow(fkey, y64, out_scale):
    y = y64 * out_scale
    if fkey == "s24":
        return np.clip(c_cast(y, np.int32), -(1 << 23), (1 << 23) - 1)
    return {"s16": lambda: c_cast(y, np.int16), "s32": lambda: c_cast(y, np.int32),
            "f32": lambda: c_cast(y, np.float32), "f64": lambda: y}[fkey]()


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def ragged_lens(rng, n_calls, n_ch, max_in):
    lens = rng.integers(0, max_in + 1, size=(n_calls, n_ch))
    for c in range(n_ch):
        rows = rng.choice(n_calls, 2, replace=False)
        lens[rows, c] = (0, max_in)
    return lens


class Twin:
    """A batch fed typed buffers next to a batch fed the same history as host-widened fp64 (process_ragged /
    process_host); every output of the first must be the C cast of the second's."""

    def __init__(self, pkg, chain, fkey, interleaved, device, n_ch=5, seed=1):
        src, dst, self.max_in, tb = CHAINS[chain]
        self.pkg, self.fkey, self.interleaved, self.device, self.n_ch = pkg, fkey, interleaved, device, n_ch
        self.fmt, self.in_scale, self.out_scale = FORMATS[fkey]
        self.plan = pkg.Plan(src, dst, self.max_in, tb, pkg.ATTEN_24)
        self.a = pkg.Batch(self.plan, n_ch, 0)
        self.b = pkg.Batch(self.plan, n_ch, 0)
        self.rng = np.random.default_rng(seed)
        self.total = np.zeros(n_ch, dtype=np.int64)   # input since each channel's last clear
        self.produced = 0

    def _input(self, width):
        v = samples(self.fkey, self.n_ch, width, self.rng)
        return to_raw(self.fkey, v, self.interleaved), v.astype(np.float64) * self.in_scale

    def _check(self, got, counts, ys):
        assert list(counts) == [len(y) for y in ys]
        for c in range(self.n_ch):
            want = narrow(self.fkey, ys[c], self.out_scale)
            assert same_bits(got[c, :counts[c]], want.astype(got.dtype)), (self.fkey, c)
            assert not np.any(got[c, counts[c]:]), "written past the count"
            self.produced += int(counts[c])

    def ragged(self, lens):
        lens = np.asarray(lens, dtype=np.int32)
        raw, wide = self._input(max(int(lens.max()), 1))
        kw = dict(interleaved=self.interleaved, in_scale=self.in_scale, out_scale=self.out_scale, fmt=self.fmt,
                  out_fmt=self.fmt)
        if self.device:
            import torch
            y, counts = self.a.process_ragged_fmt(torch.from_numpy(raw).cuda(), lens, **kw)
            y = y.cpu().numpy()
        else:
            y, counts = self.a.process_ragged_fmt(raw, lens, **kw)
        ys = self.b.process_ragged([wide[c, :lens[c]].copy() for c in range(self.n_ch)])
        self._check(from_raw(self.fkey, y, self.interleaved), counts, ys)
        self.total += lens

    def lockstep(self, l):
        """The same lock-step fp64 call on both batches (the links it keeps in shared memory are what the next ragged
        call has to refill)."""
        _, wide = self._input(l)
        ya, yb = self.a.process_host(wide), self.b.process_host(wide)
        assert same_bits(ya, yb)
        self.total += l

    def equalize(self):
        """Ragged calls that bring every channel to the same input total: one schedule again."""
        while np.any(self.total != self.total.max()):
            self.ragged(np.minimum(self.total.max() - self.total, self.max_in))

    def clear(self, channels):
        self.a.clear_channels(channels)
        self.b.clear_channels(channels)
        self.total[channels] = 0


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("interleaved", [False, True], ids=["planar", "interleaved"])
@pytest.mark.parametrize("fkey", list(FORMATS))
@pytest.mark.parametrize("chain", list(CHAINS))
def test_bit_exact_against_fp64_ragged(pkg, chain, fkey, interleaved, device):
    t = Twin(pkg, chain, fkey, interleaved, device, seed=len(chain) * 7 + len(fkey))
    if chain == "large-tile":
        assert LARGE in [k for k, _ in t.a.stage_kernels()]
    t.lockstep(t.max_in)
    for lens in ragged_lens(t.rng, 3, t.n_ch, t.max_in):
        t.ragged(lens)
    t.equalize()
    assert t.a.channel_groups == 1
    t.lockstep(t.max_in // 2 + 3)       # lock-step between ragged calls: the fused links run in shared memory
    t.clear([1])                         # mid-stream clear of one stream
    for lens in ragged_lens(t.rng, 3, t.n_ch, t.max_in):
        t.ragged(lens)
    assert t.produced > 0


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_plain_buffers_are_the_fp64_ragged_path(pkg, device):
    """Planar F64 with scale 1 runs exactly as process_ragged."""
    plan = pkg.Plan(44100.0, 96000.0, 4096, 2.0, pkg.ATTEN_24)
    a, b = pkg.Batch(plan, 4, 0), pkg.Batch(plan, 4, 0)
    rng = np.random.default_rng(5)
    for lens in ragged_lens(rng, 5, 4, 4096):
        x = rng.uniform(-1, 1, size=(4, 4096))
        if device:
            import torch
            y, counts = a.process_ragged_fmt(torch.from_numpy(x).cuda(), lens)
            y = y.cpu().numpy()
        else:
            y, counts = a.process_ragged_fmt(x, lens)
        ys = b.process_ragged([x[c, :lens[c]].copy() for c in range(4)])
        assert list(counts) == [len(v) for v in ys]
        for c in range(4):
            assert same_bits(y[c, :counts[c]], ys[c])


# ---- raw C-ABI calls: sentinels past the counts, untouched input, refusals -------------------------------------------

def raw_call(pkg, batch, x, lens, y, in_fmt, out_fmt, interleaved, device, out_cap=None, in_stride=None, in_scale=1.0,
             out_scale=1.0):
    """One typed ragged call on numpy (host form) or torch CUDA (device form) buffers, as the C-ABI takes them."""
    n_ch = batch.n_channels
    ptr = (lambda a: a.data_ptr()) if device else (lambda a: a.ctypes.data)
    if in_stride is None:
        in_stride = n_ch if interleaved else x.shape[1]
    bi = pkg.Buffer.make(ptr(x), in_fmt, interleaved, in_stride, in_scale)
    bo = pkg.Buffer.make(ptr(y), out_fmt, interleaved, n_ch if interleaved else y.shape[1], out_scale)
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    counts = np.full(n_ch, -7, dtype=np.int32)
    L = pkg.lib()
    fn = L.r8bgpu_batch_process_ragged_fmt if device else L.r8bgpu_batch_process_host_ragged_fmt
    if device:
        import torch
        batch.set_stream(torch.cuda.current_stream().cuda_stream)
    rc = fn(batch._h, C.byref(bi), lens.ctypes.data, C.byref(bo), int(batch.plan.max_out_len if out_cap is None else out_cap),
            counts.ctypes.data)
    if rc < 0:
        raise pkg.R8bGpuError(pkg._err())
    return counts


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("interleaved", [False, True], ids=["planar", "interleaved"])
def test_nothing_outside_the_extents_is_touched(pkg, interleaved, device):
    n_ch, max_in = 6, 4096
    plan = pkg.Plan(48000.0, 44100.0, max_in, 2.0, pkg.ATTEN_24)
    batch = pkg.Batch(plan, n_ch, 0)
    cap = plan.max_out_len
    rng = np.random.default_rng(11)
    for lens in ragged_lens(rng, 4, n_ch, max_in):
        x = rng.integers(-30000, 30000, size=(max_in, n_ch) if interleaved else (n_ch, max_in), dtype=np.int16)
        y = np.full((cap, n_ch) if interleaved else (n_ch, cap), 12345.0, dtype=np.float32)
        if device:
            import torch
            dx, dy = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
            counts = raw_call(pkg, batch, dx, lens, dy, pkg.S16, pkg.F32, interleaved, True)
            xa, ya = dx.cpu().numpy(), dy.cpu().numpy()
        else:
            xa, ya = x.copy(), y
            counts = raw_call(pkg, batch, xa, lens, ya, pkg.S16, pkg.F32, interleaved, False)
        assert np.array_equal(xa, x), "the input was written"
        yp = ya.T if interleaved else ya
        assert np.any(counts > 0)
        for c in range(n_ch):
            assert np.all(yp[c, counts[c]:] == 12345.0), ("written past the count", c, counts[c])
            assert not np.any(yp[c, :counts[c]] == 12345.0)


def test_forced_shards_interleaved_int16(pkg, monkeypatch):
    """Host form on a multi-device batch (two shards on one GPU): each shard takes its columns of the interleaved
    buffer; the result equals a single-device batch's bit for bit."""
    n_ch, max_in = 7, 4096
    one = pkg.Batch(pkg.Plan(44100.0, 96000.0, max_in, 2.0, pkg.ATTEN_24), n_ch, 0)
    monkeypatch.setenv("R8BGPU_FORCE_SHARDS", "2")
    plan = pkg.Plan(44100.0, 96000.0, max_in, 2.0, pkg.ATTEN_24)
    multi = pkg.Batch(plan, n_ch, pkg.DEVICE_ALL)
    assert len(multi.shards()) == 2
    rng = np.random.default_rng(17)
    all_lens = ragged_lens(rng, 6, n_ch, max_in)
    for i, lens in enumerate(all_lens):
        if i == 3:
            one.clear_channels([2, 5])
            multi.clear_channels([2, 5])
        x = rng.integers(-20000, 20000, size=(max_in, n_ch), dtype=np.int16)
        ya, ca = one.process_ragged_fmt(x, lens, interleaved=True)
        yb, cb = multi.process_ragged_fmt(x, lens, interleaved=True)
        assert np.array_equal(ca, cb)
        assert ya.dtype == np.int16 and same_bits(ya, yb)
        assert np.any(ca > 0)


@pytest.mark.parametrize("out_dtype", [np.int16, np.float32])
def test_against_compiled_reference(pkg, ref, out_dtype):
    """int16 in, one reference object per channel fed the widened input with the same chunking."""
    src, dst, n_ch, max_in = 48000.0, 44100.0, 4, 4096
    plan = pkg.Plan(src, dst, max_in, 2.0, 180.15)
    batch = pkg.Batch(plan, n_ch, 0)
    rs = [ref.Resampler(src, dst, max_in, 2.0, 180.15) for _ in range(n_ch)]
    rng = np.random.default_rng(23)
    got, want = [[] for _ in range(n_ch)], [[] for _ in range(n_ch)]
    for lens in ragged_lens(rng, 8, n_ch, max_in):
        x = rng.integers(-20000, 20000, size=(n_ch, max_in), dtype=np.int16)
        y, counts = batch.process_ragged_fmt(x, lens, out_dtype=out_dtype)
        for c in range(n_ch):
            r = rs[c].process(x[c, :lens[c]].astype(np.float64))
            assert len(r) == counts[c]
            got[c].append(y[c, :counts[c]])
            want[c].append(r)
    for c in range(n_ch):
        g, yr = np.concatenate(got[c]), np.concatenate(want[c])
        assert len(yr) > 0
        w = c_cast(yr, out_dtype)
        if out_dtype == np.float32:
            assert np.max(np.abs(g.astype(np.float64) - w.astype(np.float64)) / np.maximum(np.abs(yr), 1.0)) <= 2.0 ** -23
        else:
            assert np.max(np.abs(g.astype(np.int64) - w.astype(np.int64))) <= 1


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_refused_calls_change_nothing(pkg, device):
    n_ch, max_in = 4, 4096
    plan = pkg.Plan(44100.0, 96000.0, max_in, 2.0, pkg.ATTEN_24)
    a, b = pkg.Batch(plan, n_ch, 0), pkg.Batch(plan, n_ch, 0)
    cap = plan.max_out_len
    rng = np.random.default_rng(29)
    seq = ragged_lens(rng, 3, n_ch, max_in)
    xs = [rng.integers(-20000, 20000, size=(n_ch, max_in), dtype=np.int16) for _ in seq]

    def bufs(x):
        y = np.zeros((n_ch, cap), dtype=np.int16)
        if device:
            import torch
            return torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
        return x.copy(), y

    def run(batch, i):
        x, y = bufs(xs[i])
        counts = raw_call(pkg, batch, x, seq[i], y, pkg.S16, pkg.S16, False, device)
        return counts, (y.cpu().numpy() if device else y)

    run(a, 0)
    run(b, 0)
    bad = [
        dict(in_fmt=99),                                       # unknown format
        dict(interleaved=True, in_stride=n_ch - 1),            # interleaved stride below the channel count
        dict(in_scale=0.0),
        dict(out_scale=float("nan")),
        dict(lens=[0, -1, 5, 5]),
        dict(lens=[0, max_in + 1, 5, 5]),
        dict(out_cap=1),                                       # output capacity too small
    ]
    for kw in bad:
        x, y = bufs(xs[1])
        lens = kw.pop("lens", seq[1])
        args = dict(in_fmt=pkg.S16, interleaved=False)
        args.update(kw)
        before = a.kernel_launches
        with pytest.raises(pkg.R8bGpuError):
            raw_call(pkg, a, x, lens, y, args.pop("in_fmt"), pkg.S16, args.pop("interleaved"), device, **args)
        assert a.kernel_launches == before, kw
    for i in (1, 2):
        ca, ya = run(a, i)
        cb, yb = run(b, i)
        assert np.array_equal(ca, cb) and same_bits(ya, yb)


def test_fasttiming_and_multi_device_device_form_are_refused(pkg, monkeypatch):
    plan = pkg.Plan(48000.0, 47999.0, 1024, 2.0, pkg.ATTEN_24, fasttiming=1)
    b = pkg.Batch(plan, 2, 0)
    x = np.zeros((2, 64), dtype=np.int16)
    before = b.kernel_launches
    with pytest.raises(pkg.R8bGpuError, match="FASTTIMING"):
        b.process_ragged_fmt(x, [10, 20])
    assert b.kernel_launches == before
    monkeypatch.setenv("R8BGPU_FORCE_SHARDS", "2")
    m = pkg.Batch(pkg.Plan(44100.0, 96000.0, 1024, 2.0, pkg.ATTEN_24), 4, pkg.DEVICE_ALL)
    import torch
    with pytest.raises(pkg.R8bGpuError, match="shards"):
        m.process_ragged_fmt(torch.zeros((4, 64), dtype=torch.int16, device="cuda"), [64, 1, 0, 64])
    assert m.kernel_launches == 0
    y, counts = m.process_ragged_fmt(np.zeros((4, 64), dtype=np.int16), [64, 1, 0, 64])   # the host form runs
    assert not np.any(y)


@pytest.mark.parametrize("dtype", ["float32", "int16"])
def test_torch_tensors_match_numpy_host_form(pkg, dtype):
    import torch
    n_ch, max_in = 6, 4096
    plan = pkg.Plan(44100.0, 96000.0, max_in, 2.0, pkg.ATTEN_24)
    a, b = pkg.Batch(plan, n_ch, 0), pkg.Batch(plan, n_ch, 0)
    rng = np.random.default_rng(31)
    for i, lens in enumerate(ragged_lens(rng, 5, n_ch, max_in)):
        x = samples("f32" if dtype == "float32" else "s16", n_ch, max_in, rng)
        inter = bool(i & 1)
        xl = np.ascontiguousarray(x.T) if inter else x
        yt, ct = a.process_ragged_fmt(torch.from_numpy(xl).cuda(), lens, interleaved=inter)
        yn, cn = b.process_ragged_fmt(xl, lens, interleaved=inter)
        assert yt.is_cuda and str(yt.dtype) == "torch." + dtype
        assert np.array_equal(ct, cn) and same_bits(yt.cpu().numpy(), yn)
