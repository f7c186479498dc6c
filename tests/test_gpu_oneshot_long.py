"""GPU: long clips on every lane of a batch (Batch.oneshot_long, r8bgpu_batch_oneshot / _oneshot_host).  Each clip's
output must be bit for bit (fp64) and byte for byte (typed outputs) what Batch.oneshot_clips returns for it on a
one-channel batch of the same plan -- the twin -- whatever the lane count, so that segments, warm starts and rounds are
invisible; and each clip meets the parity bar against the compiled reference's oneshot()."""
import numpy as np
import pytest

import oracle_util as ou
from __graft_entry__ import load_package

pkg = load_package()
pytestmark = pytest.mark.gpu

MAX_IN = 4096
CHAINS = [
    (44100.0, 96000.0, 2.0),    # whole stepping on the flagship chain
    (48000.0, 44100.0, 2.0),
    (48000.0, 47999.0, 2.0),    # order-2 bank
    (192000.0, 44100.0, 2.0),   # half-band down cascade
    (44100.0, 176400.0, 2.0),   # half-band up
    (48000.0, 16000.0, 2.0),    # 1/3 BlockConvolver
    (48000.0, 16000.0, 0.5),    # large-tile path
    (96000.0, 48000.0, 2.0),
    (48000.0, 48000.0, 2.0),    # passthrough
]


def clip_sets(rng):
    return {
        "long": [int(rng.integers(60, 90) * MAX_IN + rng.integers(0, MAX_IN))],
        "stereo": [40 * MAX_IN + 123] * 2,
        "short": [int(v) for v in rng.integers(0, 12 * MAX_IN, 19)] + [0, MAX_IN],
    }


def padded(lens, rng, dtype=np.float64):
    x = np.zeros((len(lens), max(max(lens), 1)), dtype=dtype)
    for r, n in enumerate(lens):
        x[r, :n] = rng.uniform(-0.9, 0.9, n)
    return x


def twin(plan, x, lens, oplens, **kw):
    """oneshot_clips of each clip on a one-channel batch: the run every lane layout must reproduce."""
    b = pkg.Batch(plan, 1, device=0)
    out = []
    for r, n in enumerate(lens):
        xr = x[:, r:r + 1] if kw.get("interleaved") else x[r:r + 1]
        y, _ = b.oneshot_clips(xr, [n], [oplens[r]], **kw)
        out.append(y[:oplens[r], 0] if kw.get("interleaved") else y[0, :oplens[r]])
    return out


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("src,dst,tb", CHAINS)
def test_bit_identity_fp64(src, dst, tb):
    import torch
    plan = pkg.Plan(src, dst, MAX_IN, tb, pkg.ATTEN_24)
    rng = np.random.default_rng(int(src + dst) % 1000)
    for name, lens in clip_sets(rng).items():
        x = padded(lens, rng)
        oplens = [plan.default_target(n) + (37 if r % 3 == 1 else 0) - (11 if r % 3 == 2 and n else 0) for r, n in enumerate(lens)]
        oplens = [max(0, v) for v in oplens]
        want = twin(plan, x, lens, oplens)
        for n_lanes in (1, 7, 256):
            b = pkg.Batch(plan, n_lanes, device=0)
            y, _ = b.oneshot_long(x, lens, oplens)
            yd, _ = b.oneshot_long(torch.from_numpy(x).cuda(), lens, oplens)
            yd = yd.cpu().numpy()
            for r in range(len(lens)):
                assert same_bits(y[r, :oplens[r]], want[r]), (name, n_lanes, r)
                assert same_bits(yd[r, :oplens[r]], want[r]), (name, n_lanes, r, "device")
                assert not np.any(y[r, oplens[r]:])
            assert b.channel_totals()[0].max() == 0  # left cleared


def kept_per_call(plan, segs, lens, B):
    """For each round and call: the outputs all lanes keep in it (from the twin's totals at each block boundary)."""
    out = {}
    for s in segs:
        n = int(lens[s["clip"]])
        blocks = [min(B, n - k * B) for k in range(-(-n // B))]
        E = np.concatenate([[0], np.cumsum(plan.simulate(blocks))]) if blocks else np.zeros(1, np.int64)
        k0 = int(s["start"]) // B
        for i in range(-(-(int(s["p1"]) - int(s["start"])) // B)):
            lo, hi = max(int(E[k0 + i]), int(s["e0"])), min(int(E[k0 + i + 1]), int(s["e1"]))
            out[(int(s["round"]), i)] = out.get((int(s["round"]), i), 0) + max(0, hi - lo)
    return out


def test_host_form_calls_that_keep_nothing():
    """Host form over a layout with calls in which no lane keeps an output (the large-tile chain's latency of about 7
    blocks, and the lanes' warm-up), in two rounds: the blocks of consecutive calls share one pinned staging block, so each
    must be uploaded before the next is staged."""
    plan = pkg.Plan(48000.0, 16000.0, MAX_IN, 0.5, pkg.ATTEN_24)
    rng = np.random.default_rng(21)
    lens = [100 * MAX_IN + 7, 90 * MAX_IN, 80 * MAX_IN + 1, 3 * MAX_IN, 2 * MAX_IN + 9]
    n_lanes = 4
    segs, _ = plan.simulate_oneshot(n_lanes, lens)
    assert plan.oneshot_warmup >= 2 * MAX_IN and segs["round"].max() >= 1
    assert 0 in kept_per_call(plan, segs, lens, MAX_IN).values()
    x = padded(lens, rng)
    oplens = [plan.default_target(n) for n in lens]
    want = twin(plan, x, lens, oplens)
    for il in (False, True):
        xi = np.ascontiguousarray(x.T) if il else x
        y, _ = pkg.Batch(plan, n_lanes, device=0).oneshot_long(xi, lens, interleaved=il)
        for r in range(len(lens)):
            assert same_bits(y[:oplens[r], r] if il else y[r, :oplens[r]], want[r]), (il, r)


@pytest.mark.parametrize("src,dst,tb", [c for c in CHAINS if c[0] != c[1]])
def test_parity_against_reference(src, dst, tb, ref):
    plan = pkg.Plan(src, dst, MAX_IN, tb, pkg.ATTEN_24)
    rng = np.random.default_rng(5)
    lens = [70 * MAX_IN + 99, 33 * MAX_IN]
    x = padded(lens, rng)
    y, oplens = pkg.Batch(plan, 64, device=0).oneshot_long(x, lens)
    for r, n in enumerate(lens):
        yr = ref.Resampler(src, dst, MAX_IN, tb, pkg.ATTEN_24).oneshot(x[r, :n], int(oplens[r]))
        mx, rm = ou.parity_metrics(y[r, :oplens[r]], yr)
        assert mx <= 32 * ou.EPS and rm <= 4 * ou.EPS, (r, mx, rm)


@pytest.mark.parametrize("fmt", ["lsb", "msb"])
@pytest.mark.parametrize("interleaved", [False, True])
def test_dsd_input(fmt, interleaved):
    f = pkg.DSD_LSB if fmt == "lsb" else pkg.DSD_MSB
    plan = pkg.Plan(2822400.0, 88200.0, 8 * MAX_IN, 2.0, pkg.ATTEN_24)
    rng = np.random.default_rng(7)
    lens = [8 * int(v) for v in rng.integers(1, 200000, 5)] + [8 * 300000]
    x = rng.integers(0, 256, (len(lens), max(lens) // 8), dtype=np.uint8)
    if interleaved:
        x = np.ascontiguousarray(x.T)
    oplens = [plan.default_target(n) for n in lens]
    want = twin(plan, x, lens, oplens, fmt=f, in_scale=0.5, interleaved=interleaved)
    for n_lanes in (7, 256):
        y, _ = pkg.Batch(plan, n_lanes, device=0).oneshot_long(x, lens, fmt=f, in_scale=0.5, interleaved=interleaved)
        for r in range(len(lens)):
            got = y[:oplens[r], r] if interleaved else y[r, :oplens[r]]
            assert same_bits(got, want[r]), (n_lanes, r)


TYPED = [(pkg.S16, 32767.0), (pkg.S24, 8388607.0), (pkg.S32, 2147483647.0), (pkg.F32, 1.0), (pkg.U8, 127.0),
         (pkg.ULAW, 32767.0), (pkg.ALAW, 32767.0)]


@pytest.mark.parametrize("out_fmt,scale", TYPED)
def test_typed_output_and_dither(out_fmt, scale):
    plan = pkg.Plan(48000.0, 44100.0, MAX_IN, 2.0, pkg.ATTEN_24)
    rng = np.random.default_rng(out_fmt)
    lens = [50 * MAX_IN + 5, 9 * MAX_IN, 1000]
    x = (padded(lens, rng) * 30000).astype(np.int16)
    oplens = [plan.default_target(n) for n in lens]
    want = twin(plan, x, lens, oplens, out_fmt=out_fmt, in_scale=1 / 32768.0, out_scale=scale)
    seeds = [11, 12, None]
    y64 = twin(plan, x, lens, oplens, out_fmt=pkg.F64, in_scale=1 / 32768.0)
    import torch
    for n_lanes, form, il in ((1, "host", False), (7, "host", True), (256, "host", False), (7, "device", False),
                              (256, "device", True)):
        b = pkg.Batch(plan, n_lanes, device=0)
        xi = np.ascontiguousarray(x.T) if il else x
        xi = torch.from_numpy(xi).cuda() if form == "device" else xi
        kw = dict(out_fmt=out_fmt, in_scale=1 / 32768.0, out_scale=scale, interleaved=il)
        y, _ = b.oneshot_long(xi, lens, **kw)
        yd, _ = b.oneshot_long(xi, lens, dither=seeds, **kw)
        if form == "device":
            y, yd = y.cpu().numpy(), yd.cpu().numpy()
        if il:
            y, yd = np.swapaxes(y, 0, 1), np.swapaxes(yd, 0, 1)
        for r in range(len(lens)):
            assert same_bits(y[r, :oplens[r]], want[r]), (n_lanes, form, il, r)
            if out_fmt == pkg.F32 or seeds[r] is None:
                assert same_bits(yd[r, :oplens[r]], want[r])
            else:
                q, _ = pkg.dither_quantize(y64[r], out_fmt, seeds[r], scale=scale, first_index=0)
                assert same_bits(yd[r, :oplens[r]], q), (n_lanes, form, il, r, "dither")


def test_long_dsd_clip_past_2_31():
    """One DSD64 clip of more than 2^31 samples on 1024 lanes: the segments of the dry run tile the output, and the whole
    output -- its last window included -- is bit for bit the one-channel run's (oneshot_clips, 32769 ragged calls)."""
    import torch
    plan = pkg.Plan(2822400.0, 88200.0, 65536, 2.0, pkg.ATTEN_24)
    n = 2 ** 31 + 8 * 65536 + 8 * 777
    x = np.random.default_rng(3).integers(0, 256, (1, n // 8), dtype=np.uint8)
    op = plan.default_target(n)
    segs, _ = plan.simulate_oneshot(1024, [n])
    segs = np.sort(segs, order="e0")
    assert segs["e0"][0] == 0 and segs["e1"][-1] == op and np.all(segs["e1"][:-1] == segs["e0"][1:])
    y, oplens = pkg.Batch(plan, 1024, device=0).oneshot_long(torch.from_numpy(x).cuda(), [n], fmt=pkg.DSD_LSB,
                                                             out_fmt=pkg.F32, in_scale=0.5)
    assert int(oplens[0]) == op and y.shape[1] == op
    y = y[0].cpu().numpy()
    want = twin(plan, x, [n], [op], fmt=pkg.DSD_LSB, out_fmt=pkg.F32, in_scale=0.5)[0]
    assert same_bits(y[-200000:], want[-200000:]) and np.any(want[-200000:] != 0)
    assert same_bits(y, want)


def test_refusals_change_nothing():
    plan = pkg.Plan(48000.0, 44100.0, MAX_IN, 2.0, pkg.ATTEN_24)
    rng = np.random.default_rng(9)
    lens = [20 * MAX_IN, 7 * MAX_IN]
    x = padded(lens, rng)
    fresh = pkg.Batch(plan, 16, device=0)
    b = pkg.Batch(plan, 16, device=0)
    blocks = [rng.uniform(-1, 1, int(v)) for v in rng.integers(0, MAX_IN, 16)]
    for bb in (fresh, b):  # both in the same mid-stream state
        bb.process_ragged(blocks)
    xs = (x * 1000).astype(np.int16)
    with pytest.raises(ValueError, match="clip lengths"):
        b.oneshot_long(x, [x.shape[1] + 1, 8])
    bad = [
        (dict(x=x, lens=[20 * MAX_IN, -1]), "negative length"),
        (dict(x=xs, lens=lens, dither=[pkg.Dither.make(1, taps=[0.5]), None], out_fmt=pkg.S16), "noise-shaped"),
        (dict(x=(x > 0).astype(np.uint8), lens=[13, 8], fmt=pkg.DSD_LSB), "multiples of 8"),
        (dict(x=x, lens=lens, out_fmt=pkg.DSD_LSB), "input-only"),
    ]
    for kw, msg in bad:
        if msg == "negative length":  # past the front-end's own length check: straight to the C-ABI
            lv = np.array(kw["lens"], dtype=np.int64)
            bi = pkg.Buffer.make(x.ctypes.data, pkg.F64, 0, x.shape[1])
            yo = np.zeros((2, 100000))
            bo = pkg.Buffer.make(yo.ctypes.data, pkg.F64, 0, yo.shape[1])
            assert pkg.lib().r8bgpu_batch_oneshot_host(b._h, pkg.C.byref(bi), 2, lv.ctypes.data, pkg.C.byref(bo), None,
                                                        None) < 0
            assert msg in pkg._err()
        else:
            with pytest.raises(pkg.R8bGpuError, match=msg):
                b.oneshot_long(**kw)
        nxt = [rng.uniform(-1, 1, int(v)) for v in rng.integers(0, MAX_IN, 16)]
        for c, (u, v) in enumerate(zip(b.process_ragged(nxt), fresh.process_ragged(nxt))):
            assert same_bits(u, v), (msg, c)
    dsd = pkg.Plan(48000.0, 2822400.0, MAX_IN, 2.0, pkg.ATTEN_24)
    bd = pkg.Batch(dsd, 4, device=0)
    bd.set_dsd_out(True)
    with pytest.raises(pkg.R8bGpuError, match="DSD output is on"):
        bd.oneshot_long(x, lens)
    tr = pkg.Batch(pkg.Plan.trim(48000.0, 44100.0, MAX_IN, 2.0, pkg.ATTEN_24, 0.001), 4, device=0)
    with pytest.raises(pkg.R8bGpuError, match="trim plans"):
        tr.oneshot_long(x, lens)
    mixed = pkg.Batch.mixed([plan, pkg.Plan(44100.0, 48000.0, MAX_IN, 2.0, pkg.ATTEN_24)], [0, 1], device=0)
    with pytest.raises(pkg.R8bGpuError, match="mixed and multi-device"):
        mixed.oneshot_long(x, lens)
    ft = pkg.Batch(pkg.Plan(48000.0, 47999.0, MAX_IN, 2.0, pkg.ATTEN_24, fasttiming=1), 4, device=0)
    with pytest.raises(pkg.R8bGpuError, match="R8B_FASTTIMING"):
        ft.oneshot_long(x, lens)
