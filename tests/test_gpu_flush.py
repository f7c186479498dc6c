"""GPU: end of stream for independent streams (r8bgpu_batch_flush / _flush_host through Batch.flush, and
Batch.oneshot_clips).  Every flushed channel is compared with its own reference object fed the same chunking and then
blocks of silence until its output reaches the target (the tail of CDSPResampler::oneshot(), CDSPResampler.h:592-651):
equal counts, and per channel max|d| <= 32 eps, rms(d) <= 4 eps (the parity bar of test_gpu_parity.py).  Channels
that are not flushed keep running against their own, never-flushed reference objects."""
import numpy as np
import pytest

import oracle_util as ou
from test_gpu_formats import c_cast, pack24, unpack24
from test_gpu_parity import CHAINS
from test_gpu_ragged import Streams, ragged_lens

pytestmark = pytest.mark.gpu

SENTINEL = -7.25


class FlushStreams(Streams):
    """Streams plus flushes: a flushed channel's reference object is fed silence up to the target, then replaced by a
    fresh one (the reference's clear())."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.n_in = [0] * self.n_ch

    def _blocks(self, lens):
        for c, l in enumerate(lens):
            self.n_in[c] += int(l)
        return super()._blocks(lens)

    def _produced(self, c):
        n = 0
        for p in self.want[c]:
            n = 0 if p is None else n + len(p)
        return n

    def ref_tail(self, c, target):
        r, have, parts = self.rs[c], self._produced(c), []
        z = np.zeros(self.args[2])
        got = have
        while got < target:
            o = r.process(z)
            parts.append(o)
            got += len(o)
        return np.concatenate(parts)[:max(0, target - have)] if parts else np.zeros(0)

    def flush(self, channels, targets=None, device=False):
        n_in, n_out = self.batch.channel_totals()
        assert list(n_in) == self.n_in and list(n_out) == [self._produced(c) for c in range(self.n_ch)]
        y, counts = self.batch.flush(channels, targets, device=0 if device else None)
        y = y.cpu().numpy() if device else y
        for i, c in enumerate(channels):
            T = self.plan.default_target(self.n_in[c]) if targets is None else int(targets[i])
            want = self.ref_tail(c, T)
            assert counts[c] == len(want), (c, counts[c], len(want))
            self.got[c].append(y[c, :counts[c]].copy())
            self.want[c].append(want)
            self.rs[c] = self.ref.Resampler(*self.args)
            self.got[c].append(None)
            self.want[c].append(None)
            self.n_in[c] = 0
        assert all(counts[c] == 0 for c in range(self.n_ch) if c not in list(channels))
        return counts


@pytest.mark.parametrize("src,dst", CHAINS)
def test_chain_flush_parity(pkg, src, dst):
    s = FlushStreams(pkg, src, dst, 8192, 4)
    rng = np.random.default_rng(int(src * 3 + dst))
    for i, lens in enumerate(ragged_lens(rng, 3, 4, 8192)):
        s.ragged(list(lens), device=bool(i & 1))
    s.flush([2, 0])  # a subset mid-stream, host form
    for i, lens in enumerate(ragged_lens(rng, 3, 4, 8192)):
        s.ragged(list(lens), device=bool(i & 1))
    s.flush([0, 1, 2, 3], device=True)  # every channel, device form
    s.ragged([8192, 100, 0, 8192])  # fresh streams after the flush
    s.check()


def test_large_tile_chain(pkg):
    s = FlushStreams(pkg, 48000.0, 16000.0, 65536, 3, tb=0.5)
    for lens in ([65536, 0, 30000], [1, 65536, 65536]):
        s.ragged(lens)
    s.flush([0, 1], device=True)
    s.ragged([4000, 9000, 65536])
    s.flush([2, 1])
    s.check()


def test_hbdown_cascade(pkg):
    s = FlushStreams(pkg, 2822400.0, 44100.0, 65536, 3, total=65536 * 8)
    for lens in ([65536, 1000, 65536], [7, 65536, 0]):
        s.ragged(lens)
    s.flush([0, 2])
    s.ragged([65536, 65536, 33333])
    s.flush([0, 1, 2], device=True)
    s.check()


def test_hbup_cascade_64x(pkg):
    s = FlushStreams(pkg, 44100.0, 2822400.0, 2048, 3, ext=1)
    s.lockstep(2048)  # the links lock-step calls keep in shared memory are refilled by the flush
    s.ragged([2048, 100, 0])
    s.flush([1], device=True)
    s.ragged([1, 2048, 2048])
    s.flush([0, 1, 2])
    s.check()


@pytest.mark.parametrize("src,dst", [(44100.0, 96000.0), (48000.0, 47999.0), (192000.0, 44100.0)])
def test_several_sub_steps_and_explicit_targets(pkg, src, dst):
    """MaxInLen far below the chain's latency: the silence spans many sub-steps whose pieces land one after another;
    explicit targets below, at and above the default."""
    s = FlushStreams(pkg, src, dst, 256, 4)
    for lens in ([256, 17, 256, 0], [256, 256, 3, 256], [100, 256, 256, 256]):
        s.ragged(lens)
    n_out = s.batch.channel_totals()[1]
    T = [s.plan.default_target(v) for v in s.n_in]
    s.flush([0, 1, 2, 3], [int(n_out[0]) // 2, T[1], T[2] + 3000, T[3] + 1], device=True)
    s.ragged([256, 256, 256, 1])
    s.flush([3, 1])
    s.check()


def test_flush_on_lockstep_batch_and_right_after_clear(pkg):
    s = FlushStreams(pkg, 44100.0, 96000.0, 4096, 3)
    s.lockstep(4096)
    s.lockstep(1000)
    s.flush([1])
    assert s.batch.channel_groups == 2
    s.flush([1])  # N = 0: nothing to return
    s.flush([0, 2], device=True)
    assert s.batch.channel_groups == 1  # every channel fresh: lock-step again
    s.lockstep(4096)
    s.check()


def test_forced_two_shards_host_form(pkg, monkeypatch):
    monkeypatch.setenv("R8BGPU_FORCE_SHARDS", "2")
    s = FlushStreams(pkg, 48000.0, 44100.0, 8192, 5, device=pkg.DEVICE_ALL)
    assert len(s.batch.shards()) == 2
    rng = np.random.default_rng(5)
    for lens in ragged_lens(rng, 3, 5, 8192):
        s.ragged(list(lens))
    s.flush([4, 0, 2])
    s.ragged([8192] * 5)
    s.flush([1, 3, 4], [50000, 60000, 1])
    s.check()


def twin(pkg, n_ch=5, max_in=4096, src=44100.0, dst=96000.0):
    plan = pkg.Plan(src, dst, max_in, 2.0, pkg.ATTEN_24)
    a, b = pkg.Batch(plan, n_ch, 0), pkg.Batch(plan, n_ch, 0)
    rng = np.random.default_rng(3)
    x = ou.white_noise(n_ch, max_in, 7) * 20000.0
    for lens in ragged_lens(rng, 3, n_ch, max_in):
        xs = [x[c, :l].copy() for c, l in enumerate(lens)]
        a.process_ragged(xs)
        b.process_ragged(xs)
    return plan, a, b


@pytest.mark.parametrize("fkey,interleaved,device", [("s16", True, False), ("s16", True, True), ("s24", False, False),
                                                     ("s24", True, True), ("f32", False, True), ("s32", False, False)])
def test_typed_outputs(pkg, fkey, interleaved, device):
    """A typed flush is the C cast of the fp64 flush of a twin batch with the same history, bit for bit."""
    fmt, scale = {"s16": (2, 1.0), "s24": (3, 64.0), "f32": (1, 1.0), "s32": (4, 2.0 ** 12)}[fkey]
    plan, a, b = twin(pkg)
    ch = [3, 0, 4]
    y64, c64 = b.flush(ch)
    y, counts = a.flush(ch, interleaved=interleaved, device=0 if device else None, out_fmt=fmt, out_scale=scale)
    assert list(counts) == list(c64)
    y = y.cpu().numpy() if device else y
    v = unpack24(y) if fkey == "s24" else y
    v = v.T if interleaved else v
    for c in ch:
        z = y64[c, :counts[c]] * scale
        want = np.clip(c_cast(z, np.int32), -(1 << 23), (1 << 23) - 1) if fkey == "s24" else \
            c_cast(z, {"s16": np.int16, "f32": np.float32, "s32": np.int32}[fkey])
        assert np.array_equal(v[c, :counts[c]], want), c


# last stage: whole-step interpolator, half-band upsampler (3*2^k), half-band upsampler (2^k), large-tile BlockConv,
# BlockConv 1/2 after the half-band decimators, order-2 interpolator, BlockConv 2x alone
EDGE_CHAINS = [(44100.0, 96000.0, 4096, 2.0), (8000.0, 48000.0, 4096, 2.0), (44100.0, 176400.0, 4096, 2.0),
               (44100.0, 192000.0, 4096, 2.0), (48000.0, 16000.0, 16384, 0.5), (2822400.0, 44100.0, 65536, 2.0),
               (48000.0, 47999.0, 4096, 2.0), (44100.0, 88200.0, 4096, 2.0)]


@pytest.mark.parametrize("src,dst,max_in,tb", EDGE_CHAINS)
@pytest.mark.parametrize("odd,device,interleaved", [(True, True, False), (False, True, False), (True, False, False),
                                                    (True, True, True), (False, False, True)])
def test_write_bounds_at_target_cuts(pkg, src, dst, max_in, tb, odd, device, interleaved):
    """Sentinel-filled fp64 output exactly as wide as the largest count (out_cap == max count): only [0, counts[c]) of the
    named channels' rows (columns) change, every returned sample is written, and the tails match each channel's own
    reference object.  Odd explicit targets cut the last stage at odd counts, including counts whose half is a multiple
    of the half-band upsampler's block; the channels between the named ones are not flushed, so a write past a row's
    end shows in the next row."""
    import torch
    n_ch = 6
    s = FlushStreams(pkg, src, dst, max_in, n_ch, tb=tb, total=max_in * 8)
    s.ragged([max_in, max_in // 2 + 1, max_in, 3, max_in, max_in])
    s.ragged([max_in, 0, max_in // 3, max_in, 1, max_in])
    ch = [0, 2, 5]
    n_in, n_out = s.batch.channel_totals()
    if odd:
        targets = [int(n_out[0]) + 1, int(n_out[2]) + 513, int(n_out[5]) + 2 * 256 * 3 + 1]
    else:
        targets = [s.plan.default_target(int(n_in[c])) for c in ch]
    want = np.zeros(n_ch, dtype=np.int32)
    for c, T in zip(ch, targets):
        want[c] = max(0, T - int(n_out[c]))
    cap = max(int(want.max()), 1)
    shape = (cap, n_ch) if interleaved else (n_ch, cap)
    y = torch.full(shape, SENTINEL, dtype=torch.float64, device="cuda") if device else np.full(shape, SENTINEL)
    counts = np.zeros(n_ch, dtype=np.int32)
    s.batch._flush_into(np.array(ch, dtype=np.int32), np.array(targets, dtype=np.int64), y, pkg.F64, interleaved, 1.0,
                        counts)
    assert list(counts) == list(want)
    y = y.cpu().numpy() if device else y
    v = y.T if interleaved else y
    for c in range(n_ch):
        k = int(counts[c])
        assert np.all(v[c, k:] == SENTINEL), (c, k)
        assert not np.any(v[c, :k] == SENTINEL), (c, k)
    for c, T in zip(ch, targets):
        s.got[c].append(v[c, :counts[c]].copy())
        s.want[c].append(s.ref_tail(c, T))
        s.rs[c] = s.ref.Resampler(*s.args)
        s.got[c].append(None)
        s.want[c].append(None)
        s.n_in[c] = 0
    s.ragged([max_in] * n_ch)  # flushed channels start fresh, the others continue
    s.check()


@pytest.mark.parametrize("interleaved,device", [(False, True), (True, False), (False, False), (True, True)])
def test_nothing_written_past_counts(pkg, interleaved, device):
    """Sentinel-filled output: only [0, counts[c]) of the named channels' rows (columns) change."""
    import torch
    plan, a, _ = twin(pkg, n_ch=6)
    ch = np.array([1, 4, 5], dtype=np.int32)
    cap = plan.flush_max_out_len + 40
    shape = (cap, 6) if interleaved else (6, cap)
    y = np.full(shape, SENTINEL) if not device else torch.full(shape, SENTINEL, dtype=torch.float64, device="cuda")
    counts = np.zeros(6, dtype=np.int32)
    a._flush_into(ch, None, y, pkg.F64, interleaved, 1.0, counts)
    y = y.cpu().numpy() if device else y
    v = y.T if interleaved else y
    for c in range(6):
        k = int(counts[c])
        assert (k > 0) == (c in ch)
        assert np.all(v[c, k:] == SENTINEL) and not np.any(v[c, :k] == SENTINEL)


def test_passthrough(pkg):
    plan = pkg.Plan(48000.0, 48000.0, 1024)
    b = pkg.Batch(plan, 3, 0)
    b.process_ragged([np.ones(100), np.ones(7), np.ones(0)])
    assert list(b.channel_totals()[0]) == [100, 7, 0]
    y, counts = b.flush([0, 1], [150, 7])
    assert list(counts) == [50, 0, 0] and not np.any(y)
    y, counts = b.flush([2, 0], [5, 3], device=0, out_fmt=pkg.S16, interleaved=True)
    assert list(counts) == [3, 0, 5] and not torch_any(y)
    b.process_ragged([np.ones(0), np.ones(9), np.ones(4)])
    assert list(b.channel_totals()[0]) == [0, 9, 4]  # every named channel was cleared, even one with nothing to return


def torch_any(t):
    return bool(t.any().item())


@pytest.mark.parametrize("device", [False, True])
def test_oneshot_clips(pkg, ref, device):
    """Clips below, at and above MaxInLen against the reference's oneshot() per clip, default and explicit oplens."""
    import torch
    src, dst, max_in = 44100.0, 96000.0, 4096
    lens = np.array([100, 4096, 4097, 12000, 0, 9000])
    n = len(lens)
    x = ou.white_noise(n, int(lens.max()), 21)
    for c in range(n):
        x[c, lens[c]:] = 0.0
    plan = pkg.Plan(src, dst, max_in, 2.0, 180.15)
    b = pkg.Batch(plan, n, 0)
    for oplens in (None, [50, 9000, 9000, 1, 10, 30000]):
        xin = torch.from_numpy(x).cuda() if device else x
        y, ol = b.oneshot_clips(xin, lens, oplens)
        y = y.cpu().numpy() if device else y
        assert b.channel_groups == 1 and not np.any(b.channel_totals()[0])
        for c in range(n):
            want = ref.Resampler(src, dst, max_in, 2.0, 180.15).oneshot(x[c, :lens[c]], int(ol[c]))
            assert len(want) == ol[c]
            got = y[c, :ol[c]]
            assert not np.any(y[c, ol[c]:])
            if np.any(want):
                m, r = ou.parity_metrics(got, want)
                assert m <= 32 * ou.EPS and r <= 4 * ou.EPS, (c, m / ou.EPS, r / ou.EPS)
            else:
                assert not np.any(got)


def test_oneshot_clips_interleaved_int16(pkg):
    """Interleaved int16 clips: the C cast of the fp64 clips, bit for bit."""
    lens = np.array([3000, 8192, 100, 5000])
    rng = np.random.default_rng(2)
    x = rng.integers(-20000, 20000, size=(4, 8192), dtype=np.int16)
    plan = pkg.Plan(48000.0, 44100.0, 2048, 2.0, 180.15)
    b = pkg.Batch(plan, 4, 0)
    y64, ol = b.oneshot_clips(x.astype(np.float64), lens)
    y16, ol16 = b.oneshot_clips(np.ascontiguousarray(x.T), lens, interleaved=True)
    assert list(ol) == list(ol16)
    assert np.array_equal(y16.T, c_cast(y64, np.int16))


def test_refusals_change_nothing(pkg):
    s = FlushStreams(pkg, 44100.0, 96000.0, 4096, 3)
    s.ragged([4096, 100, 3000])
    before = s.batch.kernel_launches
    with pytest.raises(pkg.R8bGpuError, match="out of range"):
        s.batch.flush([0, 3])
    with pytest.raises(pkg.R8bGpuError, match="twice"):
        s.batch.flush([1, 1])
    with pytest.raises(pkg.R8bGpuError, match="negative"):
        s.batch.flush([1], [-1])
    counts = np.zeros(3, dtype=np.int32)
    with pytest.raises(pkg.R8bGpuError, match="capacity"):
        s.batch._flush_into(np.array([0, 2], dtype=np.int32), None, np.zeros((3, 10)), pkg.F64, False, 1.0, counts)
    assert s.batch.kernel_launches == before
    s.ragged([4096, 4096, 4096])  # the refused calls changed nothing: every channel continues its own stream
    s.flush([0, 1, 2])
    s.check()
    plan = pkg.Plan(48000.0, 47999.0, 1024, 2.0, pkg.ATTEN_24, fasttiming=1)
    b = pkg.Batch(plan, 2, 0)
    with pytest.raises(pkg.R8bGpuError, match="FASTTIMING"):
        b.flush([0])
    with pytest.raises(pkg.R8bGpuError, match="FASTTIMING"):
        b.flush([0, 1])
