"""GPU: gradients through whole-clip resampling (Batch.oneshot_adjoint, r8bgpu_batch_oneshot_adjoint, resample_clips).
The adjoint must be the transpose of oneshot_long -- <A x, g> = <x, A^T g> for random pairs -- on every stage kind, and
its bytes must not depend on the lane count, the clip's position in the call, the buffer layout or repetition."""
import numpy as np
import pytest

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
    (96000.0, 48000.0, 2.0),    # block-exact 1/2
    (32000.0, 48000.0, 30.0),   # block-exact 3/2
    (64000.0, 48000.0, 0.5),    # block-exact 3/4 on the large-tile path
    (48000.0, 32000.0, 2.0),    # 2/3
    (48000.0, 48000.0, 2.0),    # passthrough
]


def _torch():
    import torch
    return torch


def forward(b, x, lens, oplens):
    torch = _torch()
    y, _ = b.oneshot_long(torch.from_numpy(x).cuda(), lens, oplens)
    return y.cpu().numpy()


def adjoint(b, g, lens, oplens, **kw):
    torch = _torch()
    return b.oneshot_adjoint(torch.from_numpy(np.ascontiguousarray(g)).cuda(), lens, oplens, **kw).cpu().numpy()


@pytest.mark.parametrize("src,dst,tb", CHAINS)
def test_dot_product(src, dst, tb):
    """<A x, g> = <x, A^T g>: A x is oneshot_long; long clips past the large-tile latency, and short ones."""
    plan = pkg.Plan(src, dst, MAX_IN, tb, pkg.ATTEN_24)
    rng = np.random.default_rng(int(src + dst + tb) % 1000)
    lens = [int(rng.integers(60, 90) * MAX_IN + rng.integers(0, MAX_IN)), 3 * MAX_IN + 17, 1, 0]
    oplens = [plan.default_target(n) for n in lens]
    oplens[1] += 41  # past the default target: more flush
    worst = 0.0
    for n_lanes in (1, 7, 256):
        b = pkg.Batch(plan, n_lanes, device=0)
        for trial in range(2):
            x = np.zeros((len(lens), max(lens)))
            g = np.zeros((len(lens), max(max(oplens), 1)))
            for r, n in enumerate(lens):
                x[r, :n] = rng.uniform(-1, 1, n)
                g[r, :oplens[r]] = rng.uniform(-1, 1, oplens[r])
            y = forward(b, x, lens, oplens)
            xt = adjoint(b, g, lens, oplens)
            for r in range(len(lens)):
                assert not np.any(xt[r, lens[r]:])
                lhs = float(np.dot(y[r, :oplens[r]], g[r, :oplens[r]]))
                rhs = float(np.dot(x[r, :lens[r]], xt[r, :lens[r]]))
                scale = np.linalg.norm(y[r, :oplens[r]]) * np.linalg.norm(g[r, :oplens[r]])
                if scale == 0.0:
                    assert lhs == 0.0 and rhs == 0.0
                    continue
                ratio = abs(lhs - rhs) / scale
                worst = max(worst, ratio)
                assert ratio <= 1e-13, (n_lanes, trial, r, ratio)
    print("dot-product ratio, worst: %.3g" % worst)


@pytest.mark.parametrize("src,dst,tb", [CHAINS[1], CHAINS[2], CHAINS[4], CHAINS[7], CHAINS[9]])
def test_bit_for_bit(src, dst, tb):
    """Same bytes whatever the lanes, the clip's index and neighbours, planar or interleaved, odd strides, repetition;
    float32 buffers equal float64 buffers of the same values, narrowed once."""
    torch = _torch()
    plan = pkg.Plan(src, dst, MAX_IN, tb, pkg.ATTEN_24)
    rng = np.random.default_rng(7)
    lens = [5 * MAX_IN + 3, 2 * MAX_IN, 11]
    oplens = [plan.default_target(n) for n in lens]
    g = np.zeros((3, max(oplens)))
    for r in range(3):
        g[r, :oplens[r]] = rng.uniform(-1, 1, oplens[r])
    ref = adjoint(pkg.Batch(plan, 1, device=0), g, lens, oplens)
    for n_lanes in (7, 256):
        b = pkg.Batch(plan, n_lanes, device=0)
        assert adjoint(b, g, lens, oplens).tobytes() == ref.tobytes()
        assert adjoint(b, g, lens, oplens).tobytes() == ref.tobytes()  # repeated
    b = pkg.Batch(plan, 3, device=0)
    perm = [2, 0, 1]
    got = adjoint(b, g[perm], [lens[i] for i in perm], [oplens[i] for i in perm])
    for k, i in enumerate(perm):
        assert got[k].tobytes() == ref[i].tobytes()
    one = adjoint(b, g[1:2], lens[1:2], oplens[1:2], width=ref.shape[1])
    assert one[0].tobytes() == ref[1].tobytes()
    gi = b.oneshot_adjoint(torch.from_numpy(np.ascontiguousarray(g.T)).cuda(), lens, oplens, interleaved=True).cpu().numpy()
    assert np.ascontiguousarray(gi.T).tobytes() == ref.tobytes()
    # odd strides: rows of a wider tensor through the C-ABI directly
    wide = torch.zeros((3, max(oplens) + 5), dtype=torch.float64, device="cuda")
    wide[:, :max(oplens)] = torch.from_numpy(g).cuda()
    out = torch.full((3, max(lens) + 3), float("nan"), dtype=torch.float64, device="cuda")
    bg = pkg.Buffer.make(wide.data_ptr(), pkg.F64, False, max(oplens) + 5, 1.0)
    bx = pkg.Buffer.make(out.data_ptr(), pkg.F64, False, max(lens) + 3, 1.0)
    L = np.array(lens, dtype=np.int64)
    O = np.array(oplens, dtype=np.int64)
    b.set_stream(torch.cuda.current_stream().cuda_stream)
    import ctypes as C
    assert pkg.lib().r8bgpu_batch_oneshot_adjoint(b._h, C.byref(bg), 3, L.ctypes.data, O.ctypes.data, C.byref(bx)) == 0
    o = out.cpu().numpy()
    for r in range(3):
        assert o[r, :lens[r]].tobytes() == ref[r, :lens[r]].tobytes()
        assert np.all(np.isnan(o[r, lens[r]:]))  # nothing written past lens
    g32 = g.astype(np.float32)
    r64 = adjoint(b, g32.astype(np.float64), lens, oplens).astype(np.float32)
    r32 = b.oneshot_adjoint(torch.from_numpy(g32).cuda(), lens, oplens).cpu().numpy()
    assert r32.dtype == np.float32 and r32.tobytes() == r64.tobytes()


GRADCHECK = [
    (44100.0, 96000.0, 2.0),    # BlockConv 2x + whole stepping
    (48000.0, 47999.0, 2.0),    # order-2 bank
    (192000.0, 44100.0, 2.0),   # half-band down
    (44100.0, 176400.0, 2.0),   # half-band up
    (96000.0, 48000.0, 2.0),    # block-exact
    (48000.0, 48000.0, 2.0),    # passthrough
]


@pytest.mark.parametrize("src,dst,tb", GRADCHECK)
def test_gradcheck(src, dst, tb):
    torch = _torch()
    plan = pkg.Plan(src, dst, 64, tb, pkg.ATTEN_16)
    b = pkg.Batch(plan, 3, device=0)
    x = torch.randn(2, 40, dtype=torch.float64, device="cuda", requires_grad=True)
    lens = np.array([40, 23])
    assert torch.autograd.gradcheck(lambda t: pkg.resample_clips(b, t, lens), (x,), eps=1e-6, atol=1e-9, rtol=1e-7)
    x32 = x.detach().float().requires_grad_(True)
    y32 = pkg.resample_clips(b, x32, lens)
    gy = torch.randn_like(y32)
    y32.backward(gy)
    assert x32.grad.dtype == torch.float32
    x64 = x.detach().clone().requires_grad_(True)
    pkg.resample_clips(b, x64, lens).backward(gy.double())
    assert not torch.any(x64.grad[1, 23:])
    # the float32 backward is the float64 one on the same (widened) values, narrowed once
    assert torch.equal(x32.grad, x64.grad.float())


def test_refusals(monkeypatch):
    torch = _torch()
    plan = pkg.Plan(44100.0, 48000.0, MAX_IN, 2.0, pkg.ATTEN_24)
    b = pkg.Batch(plan, 2, device=0)
    g = torch.zeros((1, 100), dtype=torch.float64, device="cuda")
    import ctypes as C
    L = np.array([80], dtype=np.int64)
    O = np.array([80], dtype=np.int64)
    out = torch.zeros((1, 80), dtype=torch.float64, device="cuda")

    def call(gfmt=pkg.F64, xfmt=pkg.F64, gscale=1.0, lens=L, oplens=O, xstride=80, gstride=100):
        bg = pkg.Buffer.make(g.data_ptr(), gfmt, False, gstride, gscale)
        bx = pkg.Buffer.make(out.data_ptr(), xfmt, False, xstride, 1.0)
        return pkg.lib().r8bgpu_batch_oneshot_adjoint(b._h, C.byref(bg), 1, lens.ctypes.data, oplens.ctypes.data, C.byref(bx))

    msgs = set()
    for kw in (dict(gfmt=pkg.S16), dict(xfmt=pkg.S32), dict(gscale=2.0), dict(lens=np.array([-1], dtype=np.int64)),
               dict(oplens=np.array([-3], dtype=np.int64)), dict(xstride=10), dict(gstride=10)):
        assert call(**kw) != 0, kw
        msgs.add(pkg._err())
    assert len(msgs) == 5  # format, scale, negative length and each short stride have their own message
    assert not torch.any(out)
    trim = pkg.Batch(pkg.Plan.trim(44100.0, 48000.0, MAX_IN, 2.0, pkg.ATTEN_24, 0.01), 1, device=0)
    with pytest.raises(pkg.R8bGpuError, match="trim"):
        trim.oneshot_adjoint(g, [80], [80])
    ft = pkg.Batch(pkg.Plan(48000.0, 47999.0, MAX_IN, 2.0, pkg.ATTEN_24, fasttiming=1), 4, device=0)
    with pytest.raises(pkg.R8bGpuError, match="R8B_FASTTIMING"):
        ft.oneshot_adjoint(g, [80], [80])
    mixed = pkg.Batch.mixed([plan, pkg.Plan(48000.0, 44100.0, MAX_IN, 2.0, pkg.ATTEN_24)], [0, 1], device=0)
    with pytest.raises(pkg.R8bGpuError, match="mixed and multi-device"):
        mixed.oneshot_adjoint(g, [80], [80])
    monkeypatch.setenv("R8BGPU_FORCE_SHARDS", "2")  # a front of two shards, also on a one-GPU box
    front = pkg.Batch(plan, 4, pkg.DEVICE_ALL)
    monkeypatch.delenv("R8BGPU_FORCE_SHARDS")
    with pytest.raises(pkg.R8bGpuError, match="mixed and multi-device"):
        front.oneshot_adjoint(g, [80], [80])
    dsd = pkg.Batch(pkg.Plan(48000.0, 2822400.0, MAX_IN, 2.0, pkg.ATTEN_24), 4, device=0)
    dsd.set_dsd_out(True)
    with pytest.raises(pkg.R8bGpuError, match="DSD output is on"):
        dsd.oneshot_adjoint(g, [80], [80])
    with pytest.raises(ValueError, match="input lengths"):
        b.oneshot_adjoint(g)
    # the batch still works
    x = torch.zeros((1, 80), dtype=torch.float64, device="cuda")
    b.oneshot_long(x, [80], [80])
    assert call() == 0


# ---- against the compiled reference: dense A from its oneshot() of unit impulses ---------------------------------------
DENSE = [c for c in CHAINS if c[0] != c[1]]
EPS = 2.0 ** -52


def reference_adjoint(src, dst, tb, n, oplen, g):
    """A^T g with column c of A the reference's oneshot() of a unit impulse at c (None without the compiled reference)."""
    import oracle_util as ou
    if not ou.have_ref("e0"):
        return None
    rs = ou.RefOracle("e0").Resampler(src, dst, MAX_IN, tb, pkg.ATTEN_24)
    out = np.empty(n)
    e = np.zeros(n)
    for c in range(n):
        e[c] = 1.0
        out[c] = float(np.dot(rs.oneshot(e, oplen), g))
        e[c] = 0.0
    return out


@pytest.mark.parametrize("src,dst,tb", DENSE)
def test_dense_against_reference(src, dst, tb):
    """The adjoint against A^T g of the reference's own matrix, first and last samples and the flush region included.
    Bars, relative to the result's max / rms: 32 eps max (the forward parity bar) and 12 eps rms, looser than the
    forward's 4 eps because every reference column carries its own FFT blocks' rounding over all of its outputs and A^T g
    sums thousands of them (measured: 9-28 eps max, 4.2-9.0 eps rms, DESIGN.md K9)."""
    plan = pkg.Plan(src, dst, MAX_IN, tb, pkg.ATTEN_24)
    n = 2 * MAX_IN + 57
    oplen = plan.default_target(n) + 41
    rng = np.random.default_rng(int(src - dst) % 997)
    g = rng.uniform(-1, 1, oplen)
    want = reference_adjoint(src, dst, tb, n, oplen, g)
    if want is None:
        pytest.skip("compiled reference (oracle/_ref) not built")
    got = adjoint(pkg.Batch(plan, 7, device=0), g[None, :], [n], [oplen])[0]
    d = got - want
    mx = float(np.max(np.abs(d))) / float(np.max(np.abs(want)))
    rms = float(np.sqrt(np.mean(d * d))) / float(np.sqrt(np.mean(want * want)))
    edge = max(float(np.max(np.abs(d[:64]))), float(np.max(np.abs(d[-64:])))) / float(np.max(np.abs(want)))
    print("dense %s->%s: max %.2f eps, rms %.2f eps, ends %.2f eps" % (src, dst, mx / EPS, rms / EPS, edge / EPS))
    assert mx <= 32 * EPS and rms <= 12 * EPS, (mx / EPS, rms / EPS)


def test_many_blocks_and_clips():
    """More block-exact blocks than gridDim.y holds (48-sample blocks over 3.4 M samples), and more clips than that."""
    plan = pkg.Plan(192000.0, 96000.0, MAX_IN, 45.0, 49.0)
    st = plan.stages()
    assert len(st) == 1 and st[0]["down"] == 2 and st[0]["ref_input_len"] == 48
    rng = np.random.default_rng(3)
    n = 70000 * 48 + 5
    b = pkg.Batch(plan, 256, device=0)
    x = rng.uniform(-1, 1, (1, n))
    op = plan.default_target(n)
    g = rng.uniform(-1, 1, (1, op))
    y = forward(b, x, [n], [op])
    xt = adjoint(b, g, [n], [op])
    ratio = abs(float(np.dot(y[0], g[0])) - float(np.dot(x[0], xt[0]))) / (np.linalg.norm(y[0]) * np.linalg.norm(g[0]))
    assert ratio <= 1e-13, ratio
    # 70000 clips through every new kernel kind and the conversions: 192000 -> 44100 (half-band, BlockConv, interpolator)
    plan = pkg.Plan(192000.0, 44100.0, MAX_IN, 2.0, pkg.ATTEN_24)
    k = 70000
    lens = rng.integers(1, 40, k)
    oplens = np.array([plan.default_target(int(v)) for v in lens])
    b = pkg.Batch(plan, 1024, device=0)
    x = rng.uniform(-1, 1, (k, 40)) * (np.arange(40)[None, :] < lens[:, None])
    g = rng.uniform(-1, 1, (k, int(oplens.max()))) * (np.arange(int(oplens.max()))[None, :] < oplens[:, None])
    y = forward(b, x, lens, oplens)
    xt = adjoint(b, g, lens, oplens, width=40)
    lhs, rhs = np.sum(y * g, axis=1), np.sum(x * xt, axis=1)
    # clips of a few samples: the two sums' own rounding, relative to both sides
    scale = np.linalg.norm(y, axis=1) * np.linalg.norm(g, axis=1) + np.linalg.norm(x, axis=1) * np.linalg.norm(xt, axis=1)
    assert np.all(np.abs(lhs - rhs) <= 1e-13 * scale)
    assert not np.any(xt * (np.arange(40)[None, :] >= lens[:, None]))
