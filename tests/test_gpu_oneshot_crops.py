"""GPU: crops of long clips and their gradients (Batch.oneshot_crops / oneshot_crops_adjoint / resample_crops;
r8bgpu_batch_oneshot_crops / _crops_host / _crops_adjoint).  Crop k's output must be bit for bit (byte for byte when
typed) elements [o0, o1) of the clip's oneshot_long output whatever else the call holds, and its gradient the whole-clip
adjoint of its zero-padded output gradient, equal as numbers, written over the hull of its input windows only."""
import numpy as np
import pytest

from __graft_entry__ import load_package

pkg = load_package()
pytestmark = pytest.mark.gpu

MAX_IN = 4096
CHAINS = [
    (44100.0, 96000.0, 2.0),    # 2x BlockConvolver -> whole stepping
    (48000.0, 47999.0, 2.0),    # order-2 bank
    (192000.0, 44100.0, 2.0),   # half-band down cascade
    (44100.0, 176400.0, 2.0),   # half-band up
    (48000.0, 16000.0, 0.5),    # large-tile path
    (96000.0, 48000.0, 2.0),    # block-exact
    (48000.0, 48000.0, 2.0),    # passthrough
]


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def host(y):
    return y if isinstance(y, np.ndarray) else y.cpu().numpy()


def padded(lens, rng, dtype=np.float64):
    x = np.zeros((len(lens), max(max(lens), 1)), dtype=dtype)
    for r, n in enumerate(lens):
        x[r, :n] = rng.uniform(-0.9, 0.9, n)
    return x


def crops_for(rng, oplens, per_clip=3):
    """Crops of every clip: o0 = 0, the flush tail, the whole clip, an empty one, random and overlapping ones."""
    cs = []
    for r, op in enumerate(oplens):
        op = int(op)
        cs += [(r, 0, min(op, 300)), (r, max(0, op - 500), op), (r, op // 2, op // 2)]
        for _ in range(per_clip):
            a = int(rng.integers(0, op + 1))
            cs.append((r, a, int(rng.integers(a, min(op, a + 20000) + 1))))
    cs.append((0, 0, int(oplens[0])))
    return np.array(cs, dtype=np.int64)


def check_slices(y, full, crops, interleaved=False):
    y, full = host(y), host(full)
    for k, (r, o0, o1) in enumerate(crops):
        got = y[:o1 - o0, k] if interleaved else y[k, :o1 - o0]
        want = full[o0:o1, r] if interleaved else full[r, o0:o1]
        assert same_bits(got, want), (k, r, o0, o1)
        rest = y[o1 - o0:, k] if interleaved else y[k, o1 - o0:]
        assert not np.any(np.ascontiguousarray(rest).view(np.uint8)), k


@pytest.mark.parametrize("src,dst,tb", CHAINS)
def test_forward_bit_identity_fp64(src, dst, tb):
    import torch
    plan = pkg.Plan(src, dst, MAX_IN, tb, pkg.ATTEN_24)
    rng = np.random.default_rng(int(src + dst) % 997)
    lens = [int(rng.integers(60, 90) * MAX_IN + rng.integers(0, MAX_IN)), 3 * MAX_IN + 17, 1000]
    x = padded(lens, rng)
    full, oplens = pkg.Batch(plan, 1, device=0).oneshot_long(x, lens)
    crops = crops_for(rng, oplens)
    for n_lanes in (1, 7, 256):
        b = pkg.Batch(plan, n_lanes, device=0)
        check_slices(b.oneshot_crops(x, crops, lens), full, crops)
        check_slices(b.oneshot_crops(torch.from_numpy(x).cuda(), crops, lens), full, crops)
        xi = np.ascontiguousarray(x.T)
        check_slices(b.oneshot_crops(xi, crops, lens, interleaved=True), np.ascontiguousarray(full.T), crops, True)
    # permuting the crops, or adding unrelated ones, changes no crop's bytes
    perm = rng.permutation(len(crops))
    extra = np.concatenate([crops[perm], [(1, 0, int(oplens[1])), (2, 5, 9)]])
    y = pkg.Batch(plan, 7, device=0).oneshot_crops(x, extra, lens)
    check_slices(y, full, extra)


TYPED = [(pkg.S16, 32767.0), (pkg.S24, 8388607.0), (pkg.S32, 2147483647.0), (pkg.F32, 1.0), (pkg.U8, 127.0),
         (pkg.ULAW, 32767.0), (pkg.ALAW, 32767.0)]


@pytest.mark.parametrize("out_fmt,scale", TYPED)
def test_typed_output_and_dither(out_fmt, scale):
    import torch
    plan = pkg.Plan(48000.0, 44100.0, MAX_IN, 2.0, pkg.ATTEN_24)
    rng = np.random.default_rng(out_fmt)
    lens = [50 * MAX_IN + 5, 9 * MAX_IN, 1000]
    x = (padded(lens, rng) * 30000).astype(np.int16)
    seeds = [11, 12, None]
    kw = dict(out_fmt=out_fmt, in_scale=1 / 32768.0, out_scale=scale)
    ref = pkg.Batch(plan, 3, device=0)
    full, oplens = ref.oneshot_long(x, lens, **kw)
    fulld, _ = ref.oneshot_long(x, lens, dither=seeds, **kw)
    crops = crops_for(rng, oplens, 2)
    for n_lanes, form, il in ((1, "host", False), (7, "host", True), (256, "device", False), (7, "device", True)):
        b = pkg.Batch(plan, n_lanes, device=0)
        xi = np.ascontiguousarray(x.T) if il else x
        xi = torch.from_numpy(xi).cuda() if form == "device" else xi
        fi = np.ascontiguousarray(np.swapaxes(full, 0, 1)) if il else full
        fd = np.ascontiguousarray(np.swapaxes(fulld, 0, 1)) if il else fulld
        check_slices(b.oneshot_crops(xi, crops, lens, interleaved=il, **kw), fi, crops, il)
        check_slices(b.oneshot_crops(xi, crops, lens, interleaved=il, dither=seeds, **kw), fd, crops, il)


def test_dsd_input():
    plan = pkg.Plan(2822400.0, 88200.0, 8 * MAX_IN, 2.0, pkg.ATTEN_24)
    rng = np.random.default_rng(7)
    lens = [8 * int(v) for v in rng.integers(1, 200000, 3)] + [8 * 300000]
    x = rng.integers(0, 256, (len(lens), max(lens) // 8), dtype=np.uint8)
    full, oplens = pkg.Batch(plan, 1, device=0).oneshot_long(x, lens, fmt=pkg.DSD_LSB, in_scale=0.5)
    crops = crops_for(rng, oplens)
    for n_lanes in (7, 256):
        y = pkg.Batch(plan, n_lanes, device=0).oneshot_crops(x, crops, lens, fmt=pkg.DSD_LSB, in_scale=0.5)
        check_slices(y, full, crops)


def test_large_tile_chain_long_clips():
    import torch
    plan = pkg.Plan(48000.0, 16000.0, 65536, 0.5, pkg.ATTEN_24)
    rng = np.random.default_rng(5)
    lens = [40 * 65536 + 1234, 12 * 65536]
    x = torch.from_numpy(padded(lens, rng, np.float32)).cuda()
    full, oplens = pkg.Batch(plan, 256, device=0).oneshot_long(x, lens)
    a = rng.integers(0, int(oplens[0]) - 64000, 16)
    crops = np.array([(k % 2, int(v) % (int(oplens[k % 2]) - 64000), int(v) % (int(oplens[k % 2]) - 64000) + 64000)
                      for k, v in enumerate(a)], dtype=np.int64)
    for n_lanes in (7, 256):
        check_slices(pkg.Batch(plan, n_lanes, device=0).oneshot_crops(x, crops, lens), full, crops)


def test_mixed_batch():
    rates = [(16000.0, 16000.0), (22050.0, 16000.0), (44100.0, 16000.0), (48000.0, 16000.0)]
    ps = [pkg.Plan(s, d, MAX_IN, 2.0, pkg.ATTEN_24) for s, d in rates]
    po = np.array([0, 1, 2, 3, 3, 2, 1, 0], np.int32)
    lanes = np.repeat(np.arange(4, dtype=np.int32), [2, 3, 5, 7])
    b = pkg.Batch.mixed(ps, lanes, device=0)
    rng = np.random.default_rng(11)
    lens = [int(rng.integers(5, 40) * MAX_IN + rng.integers(0, MAX_IN)) for _ in po]
    x = padded(lens, rng)
    oplens = [ps[p].default_target(n) for p, n in zip(po, lens)]
    crops = crops_for(rng, oplens, 2)
    y = host(b.oneshot_crops(x, crops, lens, plan_of=po))
    for p in range(4):
        rows = [r for r in range(len(po)) if po[r] == p]
        full, _ = pkg.Batch(ps[p], 3, device=0).oneshot_long(x[rows], [lens[r] for r in rows])
        for k, (r, o0, o1) in enumerate(crops):
            if po[r] == p:
                assert same_bits(y[k, :o1 - o0], full[rows.index(r), o0:o1]), (p, k)


def _torch_adjoint(b, g, lens, oplens, dtype):
    import torch
    return b.oneshot_adjoint(torch.from_numpy(g.astype(dtype)).cuda(), lens, oplens).cpu().numpy()


@pytest.mark.parametrize("src,dst,tb", CHAINS)
def test_adjoint_against_whole_clip(src, dst, tb):
    """One crop per clip: the whole-clip adjoint of g zero-padded to oplen, equal as numbers (a zero's sign may differ);
    the sentinel outside the hull stays; several crops of one clip sum in crop order."""
    import torch
    plan = pkg.Plan(src, dst, MAX_IN, tb, pkg.ATTEN_24)
    rng = np.random.default_rng(int(src * 3 + dst) % 991)
    lens = [int(rng.integers(30, 50) * MAX_IN + rng.integers(0, MAX_IN)), 5 * MAX_IN + 3, 700]
    oplens = [plan.default_target(n) for n in lens]
    crops = np.array([(0, oplens[0] // 3, oplens[0] // 3 + 9000), (1, 0, oplens[1]), (2, oplens[2] - 100, oplens[2])])
    n = len(crops)
    W = int((crops[:, 2] - crops[:, 1]).max())
    for n_lanes, dtype in ((1, np.float64), (7, np.float64), (256, np.float32)):
        b = pkg.Batch(plan, n_lanes, device=0)
        g = rng.standard_normal((n, W))
        gp = np.zeros((3, max(oplens)))
        for k, (r, o0, o1) in enumerate(crops):
            g[k, o1 - o0:] = 0
            gp[r, o0:o1] = g[k, :o1 - o0]
        want = _torch_adjoint(b, gp, lens, oplens, dtype)
        got = b.oneshot_crops_adjoint(torch.from_numpy(g.astype(dtype)).cuda(), crops, lens).cpu().numpy()
        assert got.dtype == dtype
        for k, (r, o0, o1) in enumerate(crops):
            lo, hi = plan.oneshot_crop_extents(lens[r], oplens[r], o0, o1) if plan.stages() else ([o0], [o1])
            lo0, hi0 = int(lo[0]), min(int(hi[0]), lens[r])
            assert np.array_equal(got[r, lo0:hi0], want[r, lo0:hi0]), (n_lanes, k)
            assert not np.any(want[r, :lo0]) and not np.any(want[r, hi0:lens[r]])
    # the sentinel outside the hull: straight to the C-ABI with a prefilled buffer
    b = pkg.Batch(plan, 7, device=0)
    g = torch.from_numpy(rng.standard_normal((n, W))).cuda()
    gx = torch.full((3, max(lens)), 7.5, dtype=torch.float64, device="cuda")
    cr = pkg._crops(crops)
    lv = np.array(lens, dtype=np.int64)
    bg = pkg.Buffer.make(g.data_ptr(), pkg.F64, 0, W)
    bx = pkg.Buffer.make(gx.data_ptr(), pkg.F64, 0, max(lens))
    b.set_stream(torch.cuda.current_stream().cuda_stream)
    assert pkg.lib().r8bgpu_batch_oneshot_crops_adjoint(b._h, pkg.C.byref(bg), 3, None, lv.ctypes.data, None, n,
                                                         cr.ctypes.data, pkg.C.byref(bx)) == 0, pkg._err()
    gx = gx.cpu().numpy()
    for k, (r, o0, o1) in enumerate(crops):
        lo, hi = plan.oneshot_crop_extents(lens[r], oplens[r], o0, o1) if plan.stages() else ([o0], [o1])
        lo0, hi0 = int(lo[0]), min(int(hi[0]), lens[r])
        assert np.all(gx[r, :lo0] == 7.5) and np.all(gx[r, hi0:] == 7.5)
    # several crops of one clip: the per-crop adjoints summed in crop order
    many = np.array([(0, 100, 5000), (0, 3000, 9000), (0, oplens[0] - 2000, oplens[0]), (0, 7, 7), (1, 0, 50)])
    Wm = int((many[:, 2] - many[:, 1]).max())
    gm = rng.standard_normal((len(many), Wm))
    for k, (r, o0, o1) in enumerate(many):
        gm[k, o1 - o0:] = 0
    got = b.oneshot_crops_adjoint(torch.from_numpy(gm).cuda(), many, lens).cpu().numpy()
    parts = [b.oneshot_crops_adjoint(torch.from_numpy(gm[k:k + 1]).cuda(), many[k:k + 1], lens).cpu().numpy()
             for k in range(len(many))]
    acc = {r: np.zeros(lens[r]) for r in (0, 1)}
    cov = {r: np.zeros(lens[r], bool) for r in (0, 1)}
    for k, (r, o0, o1) in enumerate(many):
        lo, hi = plan.oneshot_crop_extents(lens[r], oplens[r], o0, o1) if plan.stages() else ([o0], [o1])
        w = np.zeros(lens[r], bool)
        w[int(lo[0]):min(int(hi[0]), lens[r])] = True
        part = parts[k][r, :lens[r]]
        acc[r][w & cov[r]] += part[w & cov[r]]
        acc[r][w & ~cov[r]] = part[w & ~cov[r]]
        cov[r] |= w
    for r in (0, 1):
        assert np.array_equal(got[r, :lens[r]], acc[r]), r


@pytest.mark.parametrize("src,dst,tb", CHAINS)
def test_dot_product(src, dst, tb):
    """<C x, g> = <x, C^T g> with C x = oneshot_crops."""
    import torch
    plan = pkg.Plan(src, dst, MAX_IN, tb, pkg.ATTEN_24)
    rng = np.random.default_rng(int(src + 2 * dst) % 983)
    lens = [int(rng.integers(20, 40) * MAX_IN + rng.integers(0, MAX_IN)), 2 * MAX_IN + 9]
    oplens = [plan.default_target(n) for n in lens]
    crops = crops_for(rng, oplens, 2)
    W = int((crops[:, 2] - crops[:, 1]).max())
    for n_lanes in (1, 7, 256):
        b = pkg.Batch(plan, n_lanes, device=0)
        x = padded(lens, rng)
        g = rng.standard_normal((len(crops), max(W, 1)))
        for k, (r, o0, o1) in enumerate(crops):
            g[k, o1 - o0:] = 0
        y = b.oneshot_crops(torch.from_numpy(x).cuda(), crops, lens).cpu().numpy()
        gx = b.oneshot_crops_adjoint(torch.from_numpy(g).cuda(), crops, lens, width=x.shape[1]).cpu().numpy()
        lhs, rhs = float(np.sum(y * g)), float(np.sum(x * gx))
        assert abs(lhs - rhs) <= 1e-13 * max(1.0, np.abs(y * g).sum(), np.abs(x * gx).sum()), (n_lanes, lhs, rhs)


GRADCHECK = [
    (44100.0, 96000.0, 2.0),    # whole stepping
    (48000.0, 47999.0, 2.0),    # order-2 bank
    (192000.0, 44100.0, 2.0),   # half-band down
]


@pytest.mark.parametrize("src,dst,tb", GRADCHECK)
def test_gradcheck_and_sliced_loss(src, dst, tb):
    """The map is linear, so its Jacobian is exactly the forward of unit impulses: the adjoint must match it to rounding.
    gradcheck's central differences carry a rounding error of about ulp(|y|) / eps per entry and no truncation error
    (linear map): at eps = 1e-6 that is ~1e-9, gradcheck's own atol, so eps is 1e-3 here."""
    import torch
    plan = pkg.Plan(src, dst, 64, tb, pkg.ATTEN_16)
    b = pkg.Batch(plan, 3, device=0)
    gen = torch.Generator(device="cuda").manual_seed(int(src + dst) % 1009)
    x = torch.randn(2, 300, dtype=torch.float64, device="cuda", generator=gen).requires_grad_(True)
    lens = np.array([300, 170])
    op = [plan.default_target(int(n)) for n in lens]
    crops = np.array([(0, op[0] // 4, op[0] // 2), (1, 0, 9), (0, op[0] - 5, op[0]), (0, op[0] // 3, op[0] // 3 + 20)])
    W = int((crops[:, 2] - crops[:, 1]).max())
    f = lambda t: pkg.resample_crops(b, t, crops, lens)
    J = torch.zeros(len(crops) * W, x.numel(), dtype=torch.float64, device="cuda")
    for c in range(x.numel()):
        e = torch.zeros_like(x, requires_grad=False)
        e.view(-1)[c] = 1.0
        J[:, c] = f(e).reshape(-1)
    for _ in range(4):
        g = torch.randn(len(crops), W, dtype=torch.float64, device="cuda", generator=gen)
        gx = b.oneshot_crops_adjoint(g, crops, lens, width=300).reshape(-1)
        assert torch.allclose(gx, J.t() @ g.reshape(-1), rtol=0, atol=1e-13 * float(g.abs().sum()))
    assert torch.autograd.gradcheck(f, (x,), eps=1e-3, atol=1e-9, rtol=1e-7)
    gy = torch.randn(len(crops), W, dtype=torch.float64, device="cuda", generator=gen)
    xa = x.detach().clone().requires_grad_(True)
    y = pkg.resample_crops(b, xa, crops, lens)
    (y * gy).sum().backward()
    xb = x.detach().clone().requires_grad_(True)
    yc = pkg.resample_clips(b, xb, lens)
    loss = sum((yc[r, o0:o1] * gy[k, :o1 - o0]).sum() for k, (r, o0, o1) in enumerate(crops))
    loss.backward()
    assert torch.allclose(xa.grad, xb.grad, rtol=1e-12, atol=1e-14)
    assert torch.equal(y.detach(), torch.stack([torch.nn.functional.pad(yc[r, o0:o1], (0, y.shape[1] - (o1 - o0)))
                                                for r, o0, o1 in crops]).detach())


def test_refusals_change_nothing():
    plan = pkg.Plan(48000.0, 44100.0, MAX_IN, 2.0, pkg.ATTEN_24)
    rng = np.random.default_rng(9)
    lens = [20 * MAX_IN, 7 * MAX_IN]
    x = padded(lens, rng)
    op = plan.default_target(lens[0])
    fresh = pkg.Batch(plan, 16, device=0)
    b = pkg.Batch(plan, 16, device=0)
    blocks = [rng.uniform(-1, 1, int(v)) for v in rng.integers(0, MAX_IN, 16)]
    for bb in (fresh, b):
        bb.process_ragged(blocks)
    bad = [
        ([(2, 0, 5)], "crops\\[0\\].clip = 2 is not a clip"),
        ([(0, -1, 5)], "crops\\[0\\].o0 = -1 is negative"),
        ([(0, 9, 5)], "crops\\[0\\].o1 = 5 is before o0 = 9"),
        ([(0, 0, op + 1)], "is past oplens\\[0\\]"),
    ]
    import torch
    for crops, msg in bad:
        with pytest.raises(pkg.R8bGpuError, match=msg):
            b.oneshot_crops(x, crops, lens)
        with pytest.raises(pkg.R8bGpuError, match=msg):
            b.oneshot_crops_adjoint(torch.zeros(1, 10, dtype=torch.float64, device="cuda"), crops, lens)
    lv = np.array(lens, dtype=np.int64)
    bi = pkg.Buffer.make(x.ctypes.data, pkg.F64, 0, x.shape[1])
    yo = np.zeros((2, 100))
    bo = pkg.Buffer.make(yo.ctypes.data, pkg.F64, 0, 100)
    assert pkg.lib().r8bgpu_batch_oneshot_crops_host(b._h, pkg.C.byref(bi), 2, None, lv.ctypes.data, None, 1, None,
                                                      pkg.C.byref(bo), None) < 0
    assert "null crops" in pkg._err()
    cr = pkg._crops([(0, 0, 101)])
    assert pkg.lib().r8bgpu_batch_oneshot_crops_host(b._h, pkg.C.byref(bi), 2, None, lv.ctypes.data, None, 1,
                                                      cr.ctypes.data, pkg.C.byref(bo), None) < 0
    assert "output stride shorter than crop 0" in pkg._err()
    nxt = [rng.uniform(-1, 1, int(v)) for v in rng.integers(0, MAX_IN, 16)]
    for c, (u, v) in enumerate(zip(b.process_ragged(nxt), fresh.process_ragged(nxt))):
        assert same_bits(u, v), c
    dsd = pkg.Batch(pkg.Plan(48000.0, 2822400.0, MAX_IN, 2.0, pkg.ATTEN_24), 4, device=0)
    dsd.set_dsd_out(True)
    with pytest.raises(pkg.R8bGpuError, match="DSD output is on"):
        dsd.oneshot_crops(x, [(0, 0, 5)], lens)
    tr = pkg.Batch(pkg.Plan.trim(48000.0, 44100.0, MAX_IN, 2.0, pkg.ATTEN_24, 0.001), 4, device=0)
    with pytest.raises(pkg.R8bGpuError, match="trim plans"):
        tr.oneshot_crops(x, [(0, 0, 5)], lens)
    ft = pkg.Batch(pkg.Plan(48000.0, 47999.0, MAX_IN, 2.0, pkg.ATTEN_24, fasttiming=1), 4, device=0)
    with pytest.raises(pkg.R8bGpuError, match="R8B_FASTTIMING"):
        ft.oneshot_crops(x, [(0, 0, 5)], lens)
    xs = (x * 1000).astype(np.int16)
    with pytest.raises(pkg.R8bGpuError, match="noise-shaped"):
        b.oneshot_crops(xs, [(0, 0, 5)], lens, out_fmt=pkg.S16, dither=[pkg.Dither.make(1, taps=[0.5]), None])
