"""GPU: moving streams -- export a channel's complete state and import it into another slot, batch or shard.

Yardstick: bit-identity.  A stream moved from slot a of batch A into slot b of batch B, and fed the same blocks from then
on, produces the same counts and the same fp64 (or dithered integer) bytes in B as it does in A; every other channel of
B is byte-identical to a twin of B that never imported; and an exporter is byte-identical to a twin that never exported.
A stream moved out of a lock-step fused batch into a ragged one changes kernel path (the fused kernel and the ragged chain
round differently, within the parity bar), so there the yardstick is the reference per channel at the parity bar."""
import pickle

import numpy as np
import pytest

import oracle_util as ou
from test_gpu_mixed import PLANS, assert_bits

pytestmark = pytest.mark.gpu

M = 16384
ATTEN = 180.15


def _blocks(rng, x, pos, lens):
    out = []
    for c, l in enumerate(lens):
        out.append(np.ascontiguousarray(x[c, pos[c]:pos[c] + l]))
        pos[c] += l
    return out


class Feed:
    """Random ragged blocks of white noise, one stream per channel."""

    def __init__(self, n_ch, seed, n=M * 12):
        self.rng = np.random.default_rng(seed)
        self.x = ou.white_noise(n_ch, n, seed=seed)
        self.pos = np.zeros(n_ch, dtype=np.int64)

    def lens(self, n_ch, lo=0, hi=M):
        return self.rng.integers(lo, hi + 1, size=n_ch)

    def next(self, lens):
        return _blocks(self.rng, self.x, self.pos, lens)


def _same_outputs(ya, yb, ctx):
    assert len(ya) == len(yb)
    for c, (a, b) in enumerate(zip(ya, yb)):
        assert_bits(a, b, "%s, channel %d" % (ctx, c))


# ---- 1. ragged to ragged, over one chain of each kind of part ------------------------------------------------------------

@pytest.mark.parametrize("src,dst,tb", PLANS)
def test_move_ragged_to_ragged_is_bit_exact(pkg, src, dst, tb):
    plan = pkg.Plan(src, dst, M, tb, ATTEN)
    A = pkg.Batch(plan, 5, 0)
    B, Bt = pkg.Batch(plan, 9, 0), pkg.Batch(plan, 9, 0)
    fa, fb = Feed(5, 11), Feed(9, 12)
    for _ in range(3):  # diverged streams in both batches
        A.process_ragged(fa.next(fa.lens(5)))
        xb = fb.next(fb.lens(9))
        _same_outputs(B.process_ragged(xb), Bt.process_ragged(xb), "B before the move")
    blob = A.export_channels([2])[0]
    assert len(blob) == plan.state_bytes
    B.import_channels([7], [blob])
    assert B.channel_totals()[0][7] == A.channel_totals()[0][2]
    assert B.channel_totals()[1][7] == A.channel_totals()[1][2]
    for _ in range(3):
        xa = fa.next(fa.lens(5))
        xb = fb.next(fb.lens(9))
        xb[7] = xa[2]
        ya, yb, yt = A.process_ragged(xa), B.process_ragged(xb), Bt.process_ragged(xb)
        assert_bits(yb[7], ya[2], "moved stream")
        for c in range(9):
            if c != 7:
                assert_bits(yb[c], yt[c], "B's channel %d next to the import" % c)


# ---- 2. out of a lock-step fused batch --------------------------------------------------------------------------------

@pytest.mark.parametrize("src,dst", [(44100.0, 96000.0), (48000.0, 44100.0)])
def test_move_from_lockstep_meets_the_reference(pkg, ref, src, dst):
    plan = pkg.Plan(src, dst, M, 2.0, ATTEN)
    A, At = pkg.Batch(plan, 4, 0), pkg.Batch(plan, 4, 0)
    x = ou.white_noise(4, M * 8, seed=3)
    L = 5000
    got = []
    for k in range(3):
        xa = x[:, k * L:(k + 1) * L]
        ya = A.process_host(xa)
        assert_bits(ya, At.process_host(xa), "lock-step before export")
        got.append(ya[1])
    blob = A.export_channels([1])[0]
    B = pkg.Batch(plan, 3, 0)
    B.import_channels([0], [blob])
    for k in range(3, 6):
        xa = x[:, k * L:(k + 1) * L]
        ya = A.process_host(xa)
        assert_bits(ya, At.process_host(xa), "the exporter after export")
        # (the moved stream runs the ragged chain, its source the fused kernel: the two paths round differently, within
        # the parity bar, so the yardstick here is the reference)
        yb = B.process_ragged([np.ascontiguousarray(xa[1]), np.zeros(0), np.zeros(0)])
        assert len(yb[0]) == len(ya[1])
        got.append(yb[0])
    r = ref.Resampler(src, dst, M, 2.0, ATTEN)
    want = np.concatenate([r.process(x[1, k * L:(k + 1) * L]) for k in range(6)])
    y = np.concatenate(got)
    assert len(y) == len(want)
    mx, rms = ou.parity_metrics(y, want)
    assert mx <= 32 * ou.EPS and rms <= 4 * ou.EPS, (mx / ou.EPS, rms / ou.EPS)


# ---- 3. host and device forms, and a pickled blob ------------------------------------------------------------------------

def test_host_and_device_blobs_are_the_same_bytes(pkg):
    import torch
    plan = pkg.Plan(44100.0, 96000.0, M, 2.0, ATTEN)
    A = pkg.Batch(plan, 4, 0)
    f = Feed(4, 21)
    for _ in range(3):
        A.process_ragged(f.next(f.lens(4)))
    host = A.export_channels([3, 0])
    dev = A.export_channels([3, 0], device=True)
    torch.cuda.synchronize()
    d = dev.cpu().numpy()
    for i in range(2):
        assert d[i, :plan.state_bytes].tobytes() == host[i]
    # device form in, host blob of the same stream out: the same bytes again
    B = pkg.Batch(plan, 2, 0)
    B.import_channels([1, 0], dev)
    assert B.export_channels([1, 0]) == host
    # a blob survives bytes -> pickle -> import
    C_ = pkg.Batch(plan, 3, 0)
    C_.import_channels([2], [pickle.loads(pickle.dumps(host[0]))])
    xa = f.next(f.lens(4))
    ya = A.process_ragged(xa)
    yc = C_.process_ragged([np.zeros(0), np.zeros(0), xa[3]])
    assert_bits(yc[2], ya[3], "pickled blob")


# ---- 4. across shards ---------------------------------------------------------------------------------------------------

def _shard_move(pkg, B):
    assert len(B.shards()) == 2
    f = Feed(6, 31)
    for _ in range(2):
        B.process_ragged(f.next(f.lens(6)))
    B.import_channels([4], B.export_channels([1]))  # shard 0 -> shard 1
    for _ in range(2):
        x = f.next(f.lens(6))
        x[4] = x[1]
        y = B.process_ragged(x)
        assert_bits(y[4], y[1], "stream moved between shards")


def test_move_between_shards(pkg, monkeypatch):
    monkeypatch.setenv("R8BGPU_FORCE_SHARDS", "2")
    _shard_move(pkg, pkg.Batch(pkg.Plan(48000.0, 44100.0, M, 2.0, ATTEN), 6, pkg.DEVICE_ALL))


def test_move_between_two_gpus(pkg, monkeypatch):
    if pkg.device_count() < 2:
        pytest.skip("needs two GPUs")
    monkeypatch.delenv("R8BGPU_FORCE_SHARDS", raising=False)
    B = pkg.Batch(pkg.Plan(48000.0, 44100.0, M, 2.0, ATTEN), 6, pkg.DEVICE_ALL)
    if len(B.shards()) != 2:
        pytest.skip("needs exactly two GPUs")
    _shard_move(pkg, B)


# ---- 5. ordinary -> mixed part -> ordinary --------------------------------------------------------------------------------

def test_ordinary_to_mixed_to_ordinary(pkg):
    specs = [(44100.0, 96000.0, 2.0), (48000.0, 47999.0, 2.0), (16000.0, 16000.0, 2.0)]
    plans = [pkg.Plan(s, d, M, tb, ATTEN) for s, d, tb in specs]
    plan_of = np.array([1, 0, 2, 0, 1], np.int32)
    Mx = pkg.Batch.mixed(plans, plan_of, 0)
    O, Ot, O2 = pkg.Batch(plans[0], 3, 0), pkg.Batch(plans[0], 3, 0), pkg.Batch(plans[0], 2, 0)
    f, fm = Feed(3, 41), Feed(5, 42)
    for _ in range(2):
        x = f.next(f.lens(3))
        _same_outputs(O.process_ragged(x), Ot.process_ragged(x), "twin")
        Mx.process_ragged(fm.next(fm.lens(5)))
    Mx.import_channels([3], O.export_channels([1]))
    for _ in range(2):
        x, xm = f.next(f.lens(3)), fm.next(fm.lens(5))
        xm[3] = x[1]
        yt, ym = Ot.process_ragged(x), Mx.process_ragged(xm)
        assert_bits(ym[3], yt[1], "ordinary -> mixed")
    with pytest.raises(pkg.R8bGpuError, match="another plan"):
        Mx.import_channels([0], O.export_channels([1]))  # channel 0 runs plans[1]
    O2.import_channels([0], Mx.export_channels([3]))
    for _ in range(2):
        x = f.next(f.lens(3))
        yt, y2 = Ot.process_ragged(x), O2.process_ragged([x[1], np.zeros(0)])
        assert_bits(y2[0], yt[1], "mixed -> ordinary")


# ---- 6. trim mid-drift and a shaped int16 stream ------------------------------------------------------------------------

def test_trim_stream_mid_drift(pkg):
    plan = pkg.Plan.trim(44100.0, 48000.0, M, 2.0, ATTEN, 0.01)
    A, B = pkg.Batch(plan, 3, 0), pkg.Batch(plan, 4, 0)
    A.set_trim([0, 1, 2], [1.001, 0.9995, 1.0002])
    B.set_trim([0, 1, 2, 3], [1.003, 1.0, 0.998, 1.0])
    f, fb = Feed(3, 51), Feed(4, 52)
    for k in range(3):
        A.set_trim([1], [0.9995 + 1e-5 * k])
        A.process_ragged(f.next(f.lens(3)))
        B.process_ragged(fb.next(fb.lens(4)))
    B.import_channels([2], A.export_channels([1]))
    assert B.trim()[2] == A.trim()[1]
    for k in range(3):
        fac = 0.9996 - 2e-5 * k
        A.set_trim([1], [fac])
        B.set_trim([2], [fac])
        x, xb = f.next(f.lens(3)), fb.next(fb.lens(4))
        xb[2] = x[1]
        assert_bits(B.process_ragged(xb)[2], A.process_ragged(x)[1], "trim stream, call %d" % k)


def test_shaped_int16_stream(pkg):
    plan = pkg.Plan(48000.0, 44100.0, M, 2.0, ATTEN)
    taps = [1.2, -0.9, 0.6, -0.4, 0.25, -0.15, 0.08, -0.04, 0.02]
    A, B = pkg.Batch(plan, 3, 0), pkg.Batch(plan, 2, 0)
    A.set_dither([1], 77, taps)
    f = Feed(3, 61)

    def call(batch, xs):
        w = max(max(len(v) for v in xs), 1)
        x = np.zeros((len(xs), w))
        for c, v in enumerate(xs):
            x[c, :len(v)] = v
        lens = np.array([len(v) for v in xs], np.int32)
        y, n = batch.process_ragged_fmt(x, lens, out_dtype=np.int16, out_scale=30000.0)
        return [y[c, :n[c]].copy() for c in range(len(xs))]

    for _ in range(3):
        call(A, f.next(f.lens(3)))
    B.import_channels([0], A.export_channels([1]))
    for _ in range(3):
        x = f.next(f.lens(3))
        assert_bits(call(B, [x[1], np.zeros(0)])[0], call(A, x)[1], "dithered int16 bytes")


# ---- 7. flush after a move -----------------------------------------------------------------------------------------------

def test_flush_after_a_move(pkg):
    plan = pkg.Plan(44100.0, 176400.0, M, 2.0, ATTEN)
    A, B = pkg.Batch(plan, 5, 0), pkg.Batch(plan, 9, 0)
    fa, fb = Feed(5, 71), Feed(9, 72)
    for _ in range(3):
        A.process_ragged(fa.next(fa.lens(5)))
        B.process_ragged(fb.next(fb.lens(9)))
    B.import_channels([7], A.export_channels([2]))
    ya, na = A.flush([2])
    yb, nb = B.flush([7])
    assert na[2] == nb[7] > 0
    assert_bits(yb[7, :nb[7]], ya[2, :na[2]], "flushed tail")


# ---- 8. edge streams ------------------------------------------------------------------------------------------------------

def test_fresh_and_short_streams(pkg):
    plan = pkg.Plan(44100.0, 96000.0, M, 2.0, ATTEN)
    A = pkg.Batch(plan, 2, 0)
    fresh = A.export_channels([0])[0]
    A.process_ragged([np.zeros(0), ou.white_noise(1, 10, seed=1)[0]])  # fewer inputs than any window
    short = A.export_channels([1])[0]
    B, Bt = pkg.Batch(plan, 3, 0), pkg.Batch(plan, 3, 0)
    f = Feed(3, 81)
    x = f.next(f.lens(3))
    _same_outputs(B.process_ragged(x), Bt.process_ragged(x), "twin")
    B.import_channels([0, 2], [fresh, short])
    Bt.clear_channels([0])
    for _ in range(2):
        x = f.next(f.lens(3))
        y, yt, ya = B.process_ragged(x), Bt.process_ragged(x), A.process_ragged([np.zeros(0), x[2]])
        assert_bits(y[0], yt[0], "fresh stream")
        assert_bits(y[1], yt[1], "untouched neighbour")
        assert_bits(y[2], ya[1], "short stream")


def test_one_blob_everywhere_runs_lockstep_again(pkg):
    plan = pkg.Plan(44100.0, 96000.0, M, 2.0, ATTEN)
    A = pkg.Batch(plan, 3, 0)
    f = Feed(3, 91)
    for _ in range(2):
        A.process_ragged(f.next(f.lens(3)))
    blob = A.export_channels([1])[0]
    B = pkg.Batch(plan, 4, 0)
    B.process_ragged(Feed(4, 92).next([100, 0, 3000, 7]))
    assert B.channel_groups > 1
    B.import_channels([0, 1, 2, 3], [blob] * 4)
    assert B.channel_groups == 1
    assert B.stage_kernels()[0][0] == "k_up2_frac2"
    x = f.next([4000] * 3)
    y = B.process_host(np.stack([x[1]] * 4))
    ya = A.process_ragged([np.zeros(0), x[1], np.zeros(0)])[1]
    assert y.shape[1] == len(ya)
    for c in range(1, 4):
        assert_bits(y[c], y[0], "lock-step after import, channel %d" % c)
    # the fused kernel against the ragged chain the source runs: equal counts, values within the parity bar
    mx, rms = ou.parity_metrics(y[0], ya)
    assert mx <= 32 * ou.EPS and rms <= 4 * ou.EPS, (mx / ou.EPS, rms / ou.EPS)


# ---- 9. refusals change nothing -------------------------------------------------------------------------------------------

def test_refusals_change_nothing(pkg):
    plan = pkg.Plan(48000.0, 44100.0, M, 2.0, ATTEN)
    other = pkg.Plan(48000.0, 44100.0, M, 2.0, ATTEN - 1.0)
    A, O = pkg.Batch(plan, 2, 0), pkg.Batch(other, 1, 0)
    B, Bt = pkg.Batch(plan, 3, 0), pkg.Batch(plan, 3, 0)
    f, fb = Feed(2, 101), Feed(3, 102)
    A.process_ragged(f.next(f.lens(2)))
    O.process_ragged([f.x[0, :500]])
    x = fb.next(fb.lens(3))
    _same_outputs(B.process_ragged(x), Bt.process_ragged(x), "twin")
    good = A.export_channels([0])[0]

    def flip(b, at):
        a = bytearray(b)
        a[at] ^= 0x40
        return bytes(a)

    cases = [
        ("different plan", [0], [O.export_channels([0])[0]]),
        ("format version", [0], [flip(good, 4)]),
        ("checksum", [0], [flip(good, len(good) - 3)]),
        ("truncated", [0], [good[:-8]]),
        ("out of range", [3], [good]),
        ("named twice", [1, 1], [good, good]),
    ]
    for why, ch, st in cases:
        with pytest.raises(pkg.R8bGpuError, match=why):
            B.import_channels(ch, st)
    fp = pkg.Plan(48000.0, 47999.0, M, 2.0, ATTEN, 0, 0, 1)  # an order-2 interpolator on R8B_FASTTIMING
    with pytest.raises(pkg.R8bGpuError, match="R8B_FASTTIMING"):
        pkg.Batch(fp, 2, 0).export_channels([0])
    for _ in range(2):
        x = fb.next(fb.lens(3))
        _same_outputs(B.process_ragged(x), Bt.process_ragged(x), "after the refusals")
