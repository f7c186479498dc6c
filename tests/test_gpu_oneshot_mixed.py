"""GPU: long clips and their gradients at mixed rates (Batch.oneshot_long / oneshot_adjoint / resample_clips with
plan_of; r8bgpu_batch_oneshot_mixed / _mixed_host / _oneshot_adjoint_mixed).  Clip r runs plans[plan_of[r]] on that
part's lanes, and its output and gradient must be bit for bit (byte for byte when typed) what an ordinary batch of that
plan returns for it; the batch is left cleared, and refused calls change nothing."""
import numpy as np
import pytest

from __graft_entry__ import load_package

pkg = load_package()
pytestmark = pytest.mark.gpu

MAX_IN = 4096
# an upsampling 2x pair, a 1x pair with an interpolator, a half-band decimator, a passthrough part
RATES = [(22050.0, 48000.0), (44100.0, 16000.0), (192000.0, 44100.0), (16000.0, 16000.0)]
LANES = [7, 1, 3, 2]


def plans(max_in=MAX_IN, atten=pkg.ATTEN_24, rates=RATES):
    return [pkg.Plan(s, d, max_in, 2.0, atten) for s, d in rates]


def mixed(ps, lanes, seed=0):
    """A mixed batch with lanes[p] channels of plan p, in a shuffled channel order."""
    po = np.concatenate([np.full(n, p, np.int32) for p, n in enumerate(lanes)])
    np.random.default_rng(seed).shuffle(po)
    return pkg.Batch.mixed(ps, po, device=0)


def clip_set(rng, n_plans, long_blocks=60):
    """Lengths 0, below B, exactly B and long (60+ blocks) for every plan, in shuffled plan order."""
    lens, po = [], []
    for p in range(n_plans):
        for n in (0, int(rng.integers(1, MAX_IN)), MAX_IN, int(long_blocks * MAX_IN + rng.integers(0, MAX_IN))):
            lens.append(n)
            po.append(p)
    perm = rng.permutation(len(lens))
    return [lens[i] for i in perm], np.array([po[i] for i in perm], np.int32)


def padded(lens, rng, dtype=np.float64):
    x = np.zeros((len(lens), max(max(lens), 1)), dtype=dtype)
    for r, n in enumerate(lens):
        x[r, :n] = rng.uniform(-0.9, 0.9, n)
    return x


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def host(y):
    return y if isinstance(y, np.ndarray) else y.cpu().numpy()


def ordinary(ps, lanes, x, lens, po, oplens, interleaved=False, **kw):
    """Each clip through oneshot_long on an ordinary batch of its own plan: {clip: output}."""
    out = {}
    dither = kw.pop("dither", None)
    for p, plan in enumerate(ps):
        rows = [r for r in range(len(lens)) if po[r] == p]
        if not rows:
            continue
        xs = np.ascontiguousarray(x[:, rows] if interleaved else x[rows])
        dv = None if dither is None else [dither[r] for r in rows]
        y, _ = pkg.Batch(plan, lanes[p], device=0).oneshot_long(xs, [lens[r] for r in rows], [oplens[r] for r in rows],
                                                                interleaved=interleaved, dither=dv, **kw)
        y = host(y)
        for k, r in enumerate(rows):
            out[r] = y[:oplens[r], k] if interleaved else y[k, :oplens[r]]
    return out


def column(y, r, n, interleaved):
    y = host(y)
    return y[:n, r] if interleaved else y[r, :n]


@pytest.mark.parametrize("interleaved", [False, True])
def test_bit_identity_fp64(interleaved):
    import torch
    ps = plans()
    b = mixed(ps, LANES, 1)
    rng = np.random.default_rng(11)
    lens, po = clip_set(rng, len(ps))
    x = padded(lens, rng)
    oplens = [ps[po[r]].default_target(n) for r, n in enumerate(lens)]
    xi = np.ascontiguousarray(x.T) if interleaved else x
    want = ordinary(ps, LANES, xi, lens, po, oplens, interleaved)
    for form in ("host", "device"):
        xin = xi if form == "host" else torch.from_numpy(xi).cuda()
        y, op = b.oneshot_long(xin, lens, interleaved=interleaved, plan_of=po)
        assert list(op) == oplens  # the default targets are each clip's own plan's
        for r in range(len(lens)):
            assert same_bits(column(y, r, oplens[r], interleaved), want[r]), (form, r, po[r], lens[r])
            tail = host(y)[oplens[r]:, r] if interleaved else host(y)[r, oplens[r]:]
            assert not np.any(tail)
        assert b.channel_totals()[0].max() == 0  # left cleared
    # a few clips against the one-channel twin
    for r in [int(np.argmax(lens)), int(np.argmin(np.abs(np.array(lens) - MAX_IN)))]:
        yt, _ = pkg.Batch(ps[po[r]], 1, device=0).oneshot_clips(x[r:r + 1], [lens[r]], [oplens[r]])
        assert same_bits(yt[0, :oplens[r]], want[r]), r


def test_typed_output_per_clip_dither():
    import torch
    ps = plans()
    b = mixed(ps, LANES, 2)
    rng = np.random.default_rng(12)
    lens, po = clip_set(rng, len(ps), long_blocks=20)
    xs = (padded(lens, rng) * 20000).astype(np.int16)
    oplens = [ps[po[r]].default_target(n) for r, n in enumerate(lens)]
    dither = [None if r % 4 == 3 else 1000 + r for r in range(len(lens))]
    want = ordinary(ps, LANES, xs, lens, po, oplens, out_fmt=pkg.S16, out_scale=0.5, dither=dither)
    for xin in (xs, torch.from_numpy(xs).cuda()):
        y, _ = b.oneshot_long(xin, lens, out_fmt=pkg.S16, out_scale=0.5, dither=dither, plan_of=po)
        y = host(y)
        assert y.dtype == np.int16
        for r in range(len(lens)):
            assert same_bits(y[r, :oplens[r]], want[r]), r


def test_dsd_input():
    import torch
    ps = plans(rates=[(2822400.0, 88200.0), (5644800.0, 88200.0)])
    b = mixed(ps, [3, 2], 3)
    rng = np.random.default_rng(13)
    lens = [8 * 4096 * 30 + 64, 8 * 1000, 0, 8 * 4096 * 12, 8 * 4096 * 45 + 8]
    po = np.array([0, 1, 1, 0, 1], np.int32)
    nb = max(lens) // 8
    x = np.zeros((len(lens), nb), np.uint8)
    for r, n in enumerate(lens):
        x[r, :n // 8] = rng.integers(0, 256, n // 8)
    oplens = [ps[po[r]].default_target(n) for r, n in enumerate(lens)]
    want = ordinary(ps, [3, 2], x, lens, po, oplens, fmt=pkg.DSD_LSB)
    for xin in (x, torch.from_numpy(x).cuda()):
        y, _ = b.oneshot_long(xin, lens, fmt=pkg.DSD_LSB, plan_of=po)
        for r in range(len(lens)):
            assert same_bits(column(y, r, oplens[r], False), want[r]), r


def test_edge_cases():
    import torch
    ps = plans()
    b = mixed(ps, LANES, 4)
    rng = np.random.default_rng(14)
    y, op = b.oneshot_long(np.zeros((0, 8)), [], plan_of=np.zeros(0, np.int32))
    assert y.shape[0] == 0 and len(op) == 0
    lens = [5 * MAX_IN + 3, 0, 70 * MAX_IN, 999]
    x = padded(lens, rng)
    for p in (0, 3):  # every clip on one part (the others have none)
        po = np.full(len(lens), p, np.int32)
        op = [ps[p].default_target(n) for n in lens]
        want = ordinary(ps, LANES, x, lens, po, op)
        y, _ = b.oneshot_long(torch.from_numpy(x).cuda(), lens, plan_of=po)
        for r in range(len(lens)):
            assert same_bits(column(y, r, op[r], False), want[r]), (p, r)
    # an ordinary batch with every index 0 is r8bgpu_batch_oneshot
    plan = ps[1]
    ob = pkg.Batch(plan, 5, device=0)
    ya, _ = ob.oneshot_long(x, lens)
    yb, _ = ob.oneshot_long(x, lens, plan_of=np.zeros(len(lens), np.int32))
    assert same_bits(ya, yb)
    with pytest.raises(pkg.R8bGpuError, match="not a plan index"):
        ob.oneshot_long(x, lens, plan_of=[0, 1, 0, 0])


def test_stream_ordering():
    """The input is produced on a side stream just before the call: the parts must wait for it."""
    import torch
    ps = plans()
    b = mixed(ps, LANES, 5)
    rng = np.random.default_rng(15)
    lens, po = clip_set(rng, len(ps), long_blocks=30)
    x0 = torch.from_numpy(padded(lens, rng)).cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        a = torch.rand(3072, 3072, dtype=torch.float64, device="cuda")
        for _ in range(6):  # a few tens of milliseconds of work ahead of the input
            a = torch.tanh(a @ a)
        x = x0 * (a[0, 0] * 0.0 + 1.0)  # exactly x0, but only once the products are done
        y, _ = b.oneshot_long(x, lens, plan_of=po)
        y = y.cpu()
    s.synchronize()
    y2, _ = b.oneshot_long(x, lens, plan_of=po)
    assert torch.equal(x, x0)
    assert same_bits(y.numpy(), y2.cpu().numpy())


def fwd(b, x, lens, oplens, po):
    import torch
    y, _ = b.oneshot_long(torch.from_numpy(x).cuda(), lens, oplens, plan_of=po)
    return y.cpu().numpy()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_adjoint_bit_identity_and_dot_product(dtype):
    import torch
    ps = plans()
    b = mixed(ps, LANES, 6)
    rng = np.random.default_rng(16)
    lens, po = clip_set(rng, len(ps))
    oplens = [ps[po[r]].default_target(n) + (17 if r % 3 == 1 else 0) for r, n in enumerate(lens)]
    g = np.zeros((len(lens), max(max(oplens), 1)))
    for r in range(len(lens)):
        g[r, :oplens[r]] = rng.uniform(-1, 1, oplens[r])
    g = g.astype(dtype)
    gx = b.oneshot_adjoint(torch.from_numpy(g).cuda(), lens, oplens, plan_of=po).cpu().numpy()
    assert gx.dtype == dtype
    for p, plan in enumerate(ps):
        rows = [r for r in range(len(lens)) if po[r] == p]
        want = pkg.Batch(plan, LANES[p], device=0).oneshot_adjoint(
            torch.from_numpy(np.ascontiguousarray(g[rows])).cuda(), [lens[r] for r in rows], [oplens[r] for r in rows],
            width=gx.shape[1]).cpu().numpy()
        for k, r in enumerate(rows):
            assert same_bits(gx[r], want[k]), (p, r)
    if dtype != np.float64:
        return
    x = padded(lens, rng)
    y = fwd(b, x, lens, oplens, po)
    for r in range(len(lens)):
        lhs = float(np.dot(y[r, :oplens[r]], g[r, :oplens[r]]))
        rhs = float(np.dot(x[r, :lens[r]], gx[r, :lens[r]]))
        scale = np.linalg.norm(y[r, :oplens[r]]) * np.linalg.norm(g[r, :oplens[r]])
        if scale == 0.0:
            assert lhs == 0.0 and rhs == 0.0
        else:
            assert abs(lhs - rhs) <= 1e-13 * scale, r


def test_adjoint_interleaved_matches_planar():
    import torch
    ps = plans()
    b = mixed(ps, LANES, 7)
    rng = np.random.default_rng(17)
    lens, po = clip_set(rng, len(ps), long_blocks=10)
    oplens = [ps[po[r]].default_target(n) for r, n in enumerate(lens)]
    g = rng.uniform(-1, 1, (len(lens), max(oplens)))
    a = b.oneshot_adjoint(torch.from_numpy(g).cuda(), lens, oplens, plan_of=po).cpu().numpy()
    gi = torch.from_numpy(np.ascontiguousarray(g.T)).cuda()
    ai = b.oneshot_adjoint(gi, lens, oplens, interleaved=True, plan_of=po).cpu().numpy()
    assert same_bits(a, np.ascontiguousarray(ai.T))


def test_gradcheck():
    import torch
    ps = plans(64, pkg.ATTEN_16, RATES)
    b = mixed(ps, [2, 1, 1, 1], 8)
    x = torch.randn(4, 40, dtype=torch.float64, device="cuda", requires_grad=True)
    lens = np.array([40, 23, 31, 17])
    po = np.array([2, 0, 3, 1], np.int32)
    assert torch.autograd.gradcheck(lambda t: pkg.resample_clips(b, t, lens, plan_of=po), (x,), eps=1e-6, atol=1e-9,
                                    rtol=1e-7)
    x32 = x.detach().float().requires_grad_(True)
    y32 = pkg.resample_clips(b, x32, lens, plan_of=po)
    gy = torch.randn_like(y32)
    y32.backward(gy)
    x64 = x.detach().clone().requires_grad_(True)
    pkg.resample_clips(b, x64, lens, plan_of=po).backward(gy.double())
    assert torch.equal(x32.grad, x64.grad.float())


def _blocks(rng, n):
    return [rng.uniform(-1, 1, int(v)) for v in rng.integers(0, MAX_IN, n)]


def test_state_after_call():
    """A call leaves the whole mixed batch cleared, and the channels' dither settings as they were."""
    ps = plans()
    b, fresh = mixed(ps, LANES, 9), mixed(ps, LANES, 9)
    for bb in (b, fresh):
        bb.set_dither([0, 3, 5], [7, 8, 9])
    rng = np.random.default_rng(19)
    b.process_ragged(_blocks(rng, b.n_channels))  # mid-stream
    lens, po = clip_set(rng, len(ps), long_blocks=8)
    b.oneshot_long(padded(lens, rng), lens, plan_of=po)
    assert b.channel_totals()[0].max() == 0 and b.channel_totals()[1].max() == 0
    for _ in range(2):
        blk = _blocks(rng, b.n_channels)
        for c, (u, v) in enumerate(zip(b.process_ragged(blk), fresh.process_ragged(blk))):
            assert same_bits(u, v), c
        xs = (padded([len(v) for v in blk], rng) * 30000).astype(np.int16)
        ln = np.array([len(v) for v in blk], np.int32)
        yu, cu = b.process_ragged_fmt(xs, ln, out_fmt=pkg.S16, out_scale=0.5)
        yv, cv = fresh.process_ragged_fmt(xs, ln, out_fmt=pkg.S16, out_scale=0.5)
        assert same_bits(cu, cv) and same_bits(yu, yv)


def _c_call(b, x, lens, po, yo, stride_out=None, adjoint=False):
    """The C-ABI directly (past the front-end's own checks)."""
    lv = np.ascontiguousarray(lens, dtype=np.int64)
    pv = None if po is None else np.ascontiguousarray(po, dtype=np.int32)
    bi = pkg.Buffer.make(x.ctypes.data, pkg.F64, 0, x.shape[1])
    bo = pkg.Buffer.make(yo.ctypes.data, pkg.F64, 0, stride_out or yo.shape[1])
    pp = None if pv is None else pv.ctypes.data
    if adjoint:
        return pkg.lib().r8bgpu_batch_oneshot_adjoint_mixed(b._h, pkg.C.byref(bi), len(lens), pp, lv.ctypes.data, None,
                                                            pkg.C.byref(bo))
    return pkg.lib().r8bgpu_batch_oneshot_mixed_host(b._h, pkg.C.byref(bi), len(lens), pp, lv.ctypes.data,
                                                     pkg.C.byref(bo), None, None)


def test_refusals_change_nothing():
    import torch
    ps = plans()[:2] + [pkg.Plan.trim(48000.0, 44100.0, MAX_IN, 2.0, pkg.ATTEN_24, 0.001)]
    b, fresh = mixed(ps, [3, 2, 2], 10), mixed(ps, [3, 2, 2], 10)
    rng = np.random.default_rng(20)
    for bb in (b, fresh):
        bb.set_dither([1], [5])
    blk = _blocks(rng, b.n_channels)
    for bb in (b, fresh):  # both in the same mid-stream state
        bb.process_ragged(blk)
    lens = [9 * MAX_IN, 3 * MAX_IN]
    x = padded(lens, rng)
    xs = (x * 1000).astype(np.int16)
    yo = np.zeros((2, 100000))
    gd = torch.zeros((2, 100000), dtype=torch.float64, device="cuda")
    gh = torch.zeros((2, 100000), dtype=torch.int16, device="cuda")

    def continue_same(msg):
        nxt = _blocks(rng, b.n_channels)
        for c, (u, v) in enumerate(zip(b.process_ragged(nxt), fresh.process_ragged(nxt))):
            assert same_bits(u, v), (msg, c)

    cases = [
        (lambda: b.oneshot_long(x, lens, plan_of=[0, 2]), "plans\\[2\\]: trim plans"),
        (lambda: b.oneshot_long(x, lens, plan_of=[0, 3]), "not a plan index"),
        (lambda: b.oneshot_long(x, lens, plan_of=[-1, 0]), "not a plan index"),
        (lambda: b.oneshot_long(xs, lens, out_fmt=pkg.S16, plan_of=[0, 1],
                                dither=[pkg.Dither.make(1, taps=[0.5]), None]), "noise-shaped"),
        (lambda: b.oneshot_long(x, lens, out_fmt=pkg.DSD_LSB, plan_of=[0, 1]), "input-only"),
        (lambda: b.oneshot_adjoint(gd, lens, plan_of=[1, 2]), "plans\\[2\\]: trim plans"),
        (lambda: b.oneshot_adjoint(gd, lens, plan_of=[1, 5]), "not a plan index"),
        (lambda: b.oneshot_adjoint(gh, lens, plan_of=[1, 0]), "float64 or float32"),
    ]
    for f, msg in cases:
        with pytest.raises((pkg.R8bGpuError, TypeError), match=msg):
            f()
        continue_same(msg)
    raw = [
        (lambda: _c_call(b, x, [9 * MAX_IN, -1], [0, 1], yo), "negative length"),
        (lambda: _c_call(b, x, lens, None, yo), "null plan_of_clip"),
        (lambda: _c_call(b, x, lens, [0, 1], yo, stride_out=10), "output stride shorter than clip 0"),
        (lambda: _c_call(b, x, lens, None, yo, adjoint=True), "null plan_of_clip"),
    ]
    for f, msg in raw:
        assert f() < 0, msg
        assert msg in pkg._err(), (msg, pkg._err())
        continue_same(msg)
    # the trim part is fine when no clip names it
    ok = mixed(ps, [3, 2, 2], 10)
    want = ordinary(ps, [3, 2, 2], x, lens, [0, 1], [ps[0].default_target(lens[0]), ps[1].default_target(lens[1])])
    y, op = ok.oneshot_long(x, lens, plan_of=[0, 1])
    for r in range(2):
        assert same_bits(y[r, :op[r]], want[r])
    # R8B_FASTTIMING (ordinary batches only) and DSD output on
    fp = pkg.Batch(pkg.Plan(48000.0, 47999.0, MAX_IN, 2.0, pkg.ATTEN_24, fasttiming=1), 2, device=0)
    with pytest.raises(pkg.R8bGpuError, match="R8B_FASTTIMING"):
        fp.oneshot_long(x, lens, plan_of=[0, 0])
    dsd = pkg.Batch.mixed([pkg.Plan(44100.0, 2822400.0, MAX_IN, 2.0, pkg.ATTEN_24),
                           pkg.Plan(48000.0, 2822400.0, MAX_IN, 2.0, pkg.ATTEN_24)], [0, 1, 0], device=0)
    dsd.set_dsd_out(True)
    with pytest.raises(pkg.R8bGpuError, match="DSD output is on"):
        dsd.oneshot_long(x, lens, plan_of=[0, 1])
    with pytest.raises(pkg.R8bGpuError, match="DSD output is on"):
        dsd.oneshot_adjoint(gd, lens, [100, 100], plan_of=[0, 1])
    # the existing entry points keep refusing mixed batches
    with pytest.raises(pkg.R8bGpuError, match="mixed and multi-device"):
        b.oneshot_long(x, lens)
    continue_same("without plan_of")
    if pkg.device_count() > 1:
        front = pkg.Batch(ps[0], 4, device=-1)
        with pytest.raises(pkg.R8bGpuError, match="R8BGPU_DEVICE_ALL"):
            front.oneshot_long(x, lens, plan_of=[0, 0])
