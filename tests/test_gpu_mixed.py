"""GPU: mixed batches -- independent streams at different rates in one batch (r8bgpu_batch_create_mixed).

Channel c of a mixed batch runs plans[plan_of[c]] and must behave exactly like a reference object built with that plan's
parameters and fed the same chunking.  Two yardsticks:
  - parity: every channel against its own compiled reference object (counts equal, max|d| <= 32 eps, rms <= 4 eps);
  - bit-equality: for every plan a twin ordinary batch fed that plan's channels' blocks through the same entry point;
    the mixed batch runs each plan's chain on the same kernels, so its outputs, counts and channel totals must equal the
    twins' bit for bit.
Every plan set below has one MaxInLen (16384) and channels assigned in a shuffled order, so no plan's channels are
contiguous in the caller's buffers."""
import ctypes as C

import numpy as np
import pytest

import oracle_util as ou
from test_gpu_invariance import ESIZE, Region
from test_gpu_ragged import ragged_lens
from test_gpu_ragged_formats import samples

pytestmark = pytest.mark.gpu

MAX_IN = 16384
ATTEN = 180.15
# (src, dst, TransBand): every kind of part chain
PLANS = [
    (44100.0, 96000.0, 2.0),    # fused 2x pair in lock-step, the ragged chain once diverged
    (48000.0, 44100.0, 2.0),
    (96000.0, 44100.0, 2.0),    # 1x pair
    (48000.0, 47999.0, 2.0),    # order-2 interpolator
    (44100.0, 176400.0, 2.0),   # half-band upsamplers
    (192000.0, 44100.0, 2.0),   # half-band downsamplers
    (2822400.0, 44100.0, 2.0),  # half-band decimator cascade
    (96000.0, 48000.0, 2.0),    # block-exact decimation
    (48000.0, 16000.0, 0.5),    # large-tile BlockConvolver
    (16000.0, 16000.0, 2.0),    # passthrough
]
F64, F32, S16, S24, S32 = 0, 1, 2, 3, 4
FKEY = {S16: "s16", S24: "s24", F32: "f32", F64: "f64"}


def _oracle():
    if not ou.have_ref("e0"):
        pytest.skip("oracle/_ref not built (needs /root/reference at build time)")
    return ou.RefOracle("e0")


def shuffled_plan_of(n_plans, per_plan, seed):
    rng = np.random.default_rng(seed)
    while True:  # draw until no plan's channels are contiguous
        po = rng.permutation(np.repeat(np.arange(n_plans), per_plan)).astype(np.int32)
        if all(np.any(np.diff(np.nonzero(po == p)[0]) > 1) for p in range(n_plans)):
            return po


class Mixed:
    """A mixed batch next to one twin ordinary batch per plan, fed the same blocks."""

    def __init__(self, pkg, plans=PLANS, per_plan=2, seed=5, device=0):
        self.pkg = pkg
        self.specs = list(plans)
        self.plans = [pkg.Plan(s, d, MAX_IN, tb, ATTEN) for s, d, tb in self.specs]
        self.plan_of = shuffled_plan_of(len(self.plans), per_plan, seed) if len(self.plans) > 1 else \
            np.zeros(per_plan, np.int32)
        self.n_ch = len(self.plan_of)
        self.batch = pkg.Batch.mixed(self.plans, self.plan_of, device)
        self.rows = [np.nonzero(self.plan_of == p)[0] for p in range(len(self.plans))]
        self.twins = [pkg.Batch(pl, len(r), device) for pl, r in zip(self.plans, self.rows)]

    # -- fp64 ragged calls: list of blocks per channel (numpy: host form, CUDA tensors: device form)
    def ragged(self, xs):
        ys = self.batch.process_ragged(xs)
        for p, r in enumerate(self.rows):
            yt = self.twins[p].process_ragged([xs[c] for c in r])
            for k, c in enumerate(r):
                assert_bits(ys[c], yt[k], "fp64 ragged, channel %d (plan %d)" % (c, p))
        self.assert_totals()
        return ys

    # -- typed ragged calls: padded planar [n_ch, w] (interleaved: [w, n_ch]) numpy or CUDA tensor
    def ragged_fmt(self, x, lens, **kw):
        inter = kw.get("interleaved", False)
        y, counts = self.batch.process_ragged_fmt(x, lens, **kw)
        for p, r in enumerate(self.rows):
            xt = x[:, r] if inter else x[r]
            yt, ct = self.twins[p].process_ragged_fmt(xt, lens[r], **kw)
            assert np.array_equal(counts[r], ct)
            for k, c in enumerate(r):
                n = int(ct[k])
                a = y[:n, c] if inter else y[c, :n]
                b = yt[:n, k] if inter else yt[k, :n]
                assert_bits(a, b, "typed ragged %r, channel %d (plan %d)" % (kw, c, p))
        self.assert_totals()
        return y, counts

    def clear(self, channels):
        self.batch.clear_channels(channels)
        for p, r in enumerate(self.rows):
            loc = [k for k, c in enumerate(r) if c in set(channels)]
            if loc:
                self.twins[p].clear_channels(loc)

    def flush(self, channels, targets=None, **kw):
        y, counts = self.batch.flush(channels, targets, **kw)
        inter = kw.get("interleaved", False)
        chs = list(channels)
        for p, r in enumerate(self.rows):
            loc = [k for k, c in enumerate(r) if c in chs]
            if not loc:
                continue
            tg = None if targets is None else [targets[chs.index(r[k])] for k in loc]
            yt, ct = self.twins[p].flush(loc, tg, **kw)
            assert np.array_equal(counts[r], ct)
            for k in loc:
                n, c = int(ct[k]), r[k]
                a = y[:n, c] if inter else y[c, :n]
                b = yt[:n, k] if inter else yt[k, :n]
                assert_bits(a, b, "flush %r, channel %d (plan %d)" % (kw, c, p))
        self.assert_totals()
        return y, counts

    def assert_totals(self):
        n_in, n_out = self.batch.channel_totals()
        for p, r in enumerate(self.rows):
            ti, to = self.twins[p].channel_totals()
            assert np.array_equal(n_in[r], ti) and np.array_equal(n_out[r], to)


def _np(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)


def assert_bits(a, b, ctx):
    a, b = np.ascontiguousarray(_np(a)), np.ascontiguousarray(_np(b))
    assert a.shape == b.shape, (ctx, a.shape, b.shape)
    if not np.array_equal(a.view(np.uint8), b.view(np.uint8)):
        bad = np.nonzero(np.any((a.view(np.uint8) != b.view(np.uint8)).reshape(len(a), -1), axis=1))[0]
        pytest.fail("%s: %d of %d samples differ, the first at %d" % (ctx, len(bad), len(a), int(bad[0])))


def blocks(x, pos, lens):
    xs = [x[c, pos[c]:pos[c] + int(l)] for c, l in enumerate(lens)]
    pos += lens
    return xs


# ---- parity against one reference object per channel -------------------------------------------------------------

@pytest.mark.parametrize("device_form", [False, True])
def test_parity_per_channel(pkg, device_form):
    ref = _oracle()
    m = Mixed(pkg, seed=11)
    rs = [ref.Resampler(*(m.specs[p][:2]), MAX_IN, m.specs[p][2], ATTEN) for p in m.plan_of]
    rng = np.random.default_rng(21)
    n_calls = 6
    x = ou.white_noise(m.n_ch, MAX_IN * (n_calls + 1), 4)
    pos = np.zeros(m.n_ch, np.int64)
    got = [[[]] for _ in range(m.n_ch)]
    want = [[[]] for _ in range(m.n_ch)]
    cleared = [c for c in range(m.n_ch) if c % 3 == 1]  # channels of several plans
    for i, lens in enumerate(ragged_lens(rng, n_calls, m.n_ch, MAX_IN)):
        if i == 3:
            m.clear(cleared)
            for c in cleared:
                rs[c] = ref.Resampler(*(m.specs[m.plan_of[c]][:2]), MAX_IN, m.specs[m.plan_of[c]][2], ATTEN)
                got[c].append([])
                want[c].append([])
        xs = blocks(x, pos, lens)
        if device_form:
            import torch
            ys = [_np(y) for y in m.ragged([torch.from_numpy(v.copy()).cuda() for v in xs])]
        else:
            ys = m.ragged([v.copy() for v in xs])
        for c in range(m.n_ch):
            r = rs[c].process(xs[c])
            assert len(r) == len(ys[c]), (c, m.specs[m.plan_of[c]], len(r), len(ys[c]))
            got[c][-1].append(np.asarray(ys[c]))
            want[c][-1].append(r)
    n = 0
    for c in range(m.n_ch):
        for sg, sw in zip(got[c], want[c]):
            a, b = np.concatenate([np.zeros(0)] + sg), np.concatenate([np.zeros(0)] + sw)
            if len(b) == 0 or not np.any(b):
                assert not np.any(a)
                continue
            mx, rms = ou.parity_metrics(a, b)
            assert mx <= 32 * ou.EPS and rms <= 4 * ou.EPS, (c, m.specs[m.plan_of[c]], mx / ou.EPS, rms / ou.EPS)
            n += 1
    assert n >= m.n_ch


# ---- bit-equality with twin ordinary batches ---------------------------------------------------------------------

@pytest.mark.parametrize("fmt", [S16, S24, F32, F64])
@pytest.mark.parametrize("interleaved", [False, True])
@pytest.mark.parametrize("device_form", [False, True])
def test_twins_typed(pkg, fmt, interleaved, device_form):
    if device_form and fmt == S24:
        pytest.skip("packed 24-bit device buffers are covered by test_layouts")
    m = Mixed(pkg, seed=fmt + 3 * interleaved)
    rng = np.random.default_rng(7 + fmt)
    fkey = FKEY[fmt]
    for i, lens in enumerate(ragged_lens(rng, 4, m.n_ch, MAX_IN)):
        v = samples(fkey, m.n_ch, MAX_IN, rng)
        kw = {"interleaved": interleaved}
        if fmt == S24:
            from test_gpu_formats import pack24
            x = pack24(v)
            kw.update(fmt=S24, out_fmt=S24)
        else:
            x = v
        if fmt == F64:
            kw.update(in_scale=0.5, out_scale=3.0)
        if interleaved:
            x = np.ascontiguousarray(np.swapaxes(x, 0, 1))
        if device_form:
            import torch
            x = torch.from_numpy(x).cuda()
        if i == 2:
            m.clear([c for c in range(m.n_ch) if c % 4 == 0])
        m.ragged_fmt(x, lens.astype(np.int32), **kw)
    # end of stream: default targets on some channels, explicit ones on the others
    dev = 0 if device_form else None
    out_fmt = F64 if fmt == S24 else fmt
    m.flush([c for c in range(m.n_ch) if c % 2 == 0], device=dev, interleaved=interleaved, out_fmt=out_fmt)
    n_out = m.batch.channel_totals()[1]
    odd = [c for c in range(m.n_ch) if c % 2 == 1]
    m.flush(odd, [int(n_out[c]) + 1000 + 17 * c for c in odd], device=dev, interleaved=interleaved, out_fmt=out_fmt)


def test_one_plan_equals_ordinary(pkg):
    m = Mixed(pkg, plans=[PLANS[0]], per_plan=5)
    rng = np.random.default_rng(2)
    x = ou.white_noise(m.n_ch, MAX_IN * 5, 9)
    pos = np.zeros(m.n_ch, np.int64)
    for lens in ragged_lens(rng, 4, m.n_ch, MAX_IN):
        m.ragged(blocks(x, pos, lens))
    m.flush(list(range(m.n_ch)))


# ---- caller layouts: offsets, odd strides, padding columns, 24-bit byte phases -----------------------------------

LAYOUTS = [  # (fmt, interleaved, start element, stride slack)
    (F64, False, 1, 3), (S16, False, 3, 5), (F32, True, 2, 3), (S24, False, 1, 7), (S24, False, 2, 1),
    (S24, True, 5, 2), (S16, True, 0, 1),
]


@pytest.mark.parametrize("fmt,interleaved,start,slack", LAYOUTS)
def test_layouts(pkg, fmt, interleaved, start, slack):
    import torch
    m = Mixed(pkg, seed=31 + start)
    rng = np.random.default_rng(40 + start)
    fkey = FKEY[fmt]
    L = m.pkg.lib()
    e = ESIZE[fmt]
    cap = m.batch.max_out_len
    for i, lens in enumerate(ragged_lens(rng, 3, m.n_ch, MAX_IN)):
        lens = lens.astype(np.int32)
        v = samples(fkey, m.n_ch, MAX_IN, rng)
        w_in = MAX_IN
        rin = Region(fmt, m.n_ch, w_in, start * e, (m.n_ch if interleaved else w_in) + slack, interleaved).fill(v)
        rout = Region(fmt, m.n_ch, cap, start * e, (m.n_ch if interleaved else cap) + slack, interleaved)
        counts = np.zeros(m.n_ch, np.int32)
        m.batch.set_stream(torch.cuda.current_stream().cuda_stream)
        rc = L.r8bgpu_batch_process_ragged_fmt(m.batch._h, C.byref(rin.buffer(pkg)), lens.ctypes.data,
                                               C.byref(rout.buffer(pkg)), cap, counts.ctypes.data)
        assert rc == 0, pkg._err()
        torch.cuda.synchronize()
        want = [None] * m.n_ch
        for p, r in enumerate(m.rows):  # the twins, fed host-form planar buffers of the same values
            from test_gpu_formats import pack24
            xt = pack24(v[r]) if fmt == S24 else v[r]
            kw = {"fmt": S24, "out_fmt": S24} if fmt == S24 else {}
            yt, ct = m.twins[p].process_ragged_fmt(xt, lens[r], **kw)
            assert np.array_equal(counts[r], ct)
            for k, c in enumerate(r):
                want[c] = yt[k, :ct[k]]
                if fmt == S24:
                    from test_gpu_formats import unpack24
                    want[c] = unpack24(want[c])
        rout.assert_holds(want, "layout %r call %d" % ((fmt, interleaved, start, slack), i))
        rin.assert_untouched()


# ---- datasets: whole clips at many rates -------------------------------------------------------------------------

@pytest.mark.parametrize("device_form", [False, True])
def test_dataset_clips(pkg, device_form):
    ref = _oracle()
    rates = [8000.0, 16000.0, 22050.0, 32000.0, 44100.0, 48000.0]
    plans = [pkg.Plan(s, 16000.0, MAX_IN, 2.0, ATTEN) for s in rates]
    rng = np.random.default_rng(64)
    plan_of = rng.integers(0, len(rates), size=64).astype(np.int32)
    plan_of[:len(rates)] = np.arange(len(rates))
    b = pkg.Batch.mixed(plans, plan_of, 0)
    lens = rng.integers(0, 3 * MAX_IN, size=64)
    lens[[7, 8]] = (0, 1)
    x = ou.white_noise(64, int(lens.max()), 17)
    for c in range(64):
        x[c, lens[c]:] = 0.0
    if device_form:
        import torch
        y, oplens = b.oneshot_clips(torch.from_numpy(x).cuda(), lens)
        y = y.cpu().numpy()
    else:
        y, oplens = b.oneshot_clips(x, lens)
    for c in range(64):
        s = rates[plan_of[c]]
        assert oplens[c] == plans[plan_of[c]].default_target(lens[c])
        want = ref.Resampler(s, 16000.0, MAX_IN, 2.0, ATTEN).oneshot(x[c, :lens[c]], int(oplens[c]))
        got = y[c, :oplens[c]]
        if not np.any(want):
            assert not np.any(got)
            continue
        mx, rms = ou.parity_metrics(got, want)
        assert mx <= 32 * ou.EPS and rms <= 4 * ou.EPS, (c, s, mx / ou.EPS, rms / ou.EPS)


# ---- refusals change nothing -------------------------------------------------------------------------------------

def test_refusals(pkg):
    m = Mixed(pkg, seed=77)
    rng = np.random.default_rng(3)
    x = ou.white_noise(m.n_ch, MAX_IN * 12, 5)
    pos = np.zeros(m.n_ch, np.int64)
    step = iter(ragged_lens(rng, 10, m.n_ch, MAX_IN))
    m.ragged(blocks(x, pos, next(step)))
    L = pkg.lib()

    def refused(fn, words):
        with pytest.raises(pkg.R8bGpuError) as ei:
            fn()
        assert any(w in str(ei.value) for w in words), str(ei.value)
        m.ragged(blocks(x, pos, next(step)))  # the next call still equals the twins

    refused(lambda: m.batch.process_host(np.zeros((m.n_ch, 16))), ["ragged"])
    refused(lambda: m.batch.stage_kernels(), ["r8bgpu_batch_part"])
    refused(lambda: pkg.Batch.mixed(m.plans, m.plan_of, pkg.DEVICE_ALL), ["R8BGPU_DEVICE_ALL"])
    refused(lambda: pkg.Batch.mixed(m.plans + [pkg.Plan(48000.0, 47999.0, MAX_IN, 2.0, ATTEN, fasttiming=1)],
                                    np.append(m.plan_of, len(m.plans)), 0), ["FASTTIMING"])
    refused(lambda: pkg.Batch.mixed([m.plans[0], pkg.Plan(48000.0, 44100.0, 4096, 2.0, ATTEN)], [0, 1], 0), ["MaxInLen"])
    refused(lambda: pkg.Batch.mixed(m.plans, np.append(m.plan_of, 99), 0), ["plan_of"])

    def small_cap():
        lens = np.full(m.n_ch, 100, np.int32)
        xd = np.zeros((m.n_ch, 100))
        y = np.zeros((m.n_ch, m.batch.max_out_len))
        counts = np.zeros(m.n_ch, np.int32)
        if L.r8bgpu_batch_process_host_ragged(m.batch._h, xd.ctypes.data, 100, lens.ctypes.data, y.ctypes.data,
                                              m.batch.max_out_len, m.batch.max_out_len - 1, counts.ctypes.data) < 0:
            raise pkg.R8bGpuError(pkg._err())
    refused(small_cap, ["r8bgpu_batch_max_out_len"])
    refused(lambda: m.batch.flush([0, m.n_ch]), ["out of range"])
    refused(lambda: m.batch.flush([1, 1]), ["twice"])


# ---- launches and part introspection -----------------------------------------------------------------------------

def test_launches_and_parts(pkg):
    m = Mixed(pkg, seed=8)
    rng = np.random.default_rng(12)
    parts = [m.batch.part(i) for i in range(len(m.plans))]
    for i, lens in enumerate(ragged_lens(rng, 3, m.n_ch, MAX_IN)):
        lens = np.maximum(lens, 1000).astype(np.int32)
        v = samples("s16", m.n_ch, MAX_IN, rng)
        before, pb = m.batch.kernel_launches, [p.kernel_launches for p in parts]
        m.ragged_fmt(v, lens)
        d_parts = sum(p.kernel_launches - b for p, b in zip(parts, pb))
        assert m.batch.kernel_launches - before == d_parts + 2
        before, pb = m.batch.kernel_launches, [p.kernel_launches for p in parts]
        x = ou.white_noise(m.n_ch, MAX_IN, i)
        m.ragged([x[c, :lens[c]] for c in range(m.n_ch)])
        d_parts = sum(p.kernel_launches - b for p, b in zip(parts, pb))
        assert m.batch.kernel_launches - before == d_parts + 2
    for p, part in enumerate(parts):
        assert part.n_channels == len(m.rows[p])
        assert part.stage_kernels() == m.twins[p].stage_kernels()
    assert m.batch.channel_groups == sum(p.channel_groups for p in parts)
    assert m.batch.max_out_len == max(p.max_out_len for p in m.plans)
    assert m.batch.flush_max_out_len == max(p.flush_max_out_len for p in m.plans)
    assert m.batch.device_bytes > sum(p.device_bytes for p in parts)
    del parts


# ---- asynchrony: device calls queued back to back on a torch stream ----------------------------------------------

def test_async_device_calls(pkg):
    import torch
    rng = np.random.default_rng(99)
    dev_m = Mixed(pkg, seed=4)
    host_b = pkg.Batch.mixed(dev_m.plans, dev_m.plan_of, 0)
    all_lens = ragged_lens(rng, 5, dev_m.n_ch, MAX_IN).astype(np.int32)
    vs = [samples("f32", dev_m.n_ch, MAX_IN, rng) for _ in all_lens]
    s = torch.cuda.Stream()
    outs = []
    with torch.cuda.stream(s):
        xs = [torch.from_numpy(v).cuda() for v in vs]
        for x, lens in zip(xs, all_lens):
            outs.append(dev_m.batch.process_ragged_fmt(x, lens))
        tail = dev_m.batch.flush(list(range(dev_m.n_ch)), device=0, out_fmt=F32)
    s.synchronize()
    for (y, counts), v, lens in zip(outs, vs, all_lens):
        yh, ch = host_b.process_ragged_fmt(v, lens)
        assert np.array_equal(counts, ch)
        y = y.cpu().numpy()
        for c in range(dev_m.n_ch):
            assert_bits(y[c, :ch[c]], yh[c, :ch[c]], "async call, channel %d" % c)
    th, tc = host_b.flush(list(range(dev_m.n_ch)), out_fmt=F32)
    assert np.array_equal(tail[1], tc)
    yt = tail[0].cpu().numpy()
    for c in range(dev_m.n_ch):
        assert_bits(yt[c, :tc[c]], th[c, :tc[c]], "async flush, channel %d" % c)
