"""CPU: crops of long clips with no GPU.  The span layout (Plan.simulate_oneshot_crops) over the long-clip chains and
seeded crop sets: each crop's kept ranges tile [o0, o1), its first segment starts W before P_lo, its span ends at the
first block boundary with E >= o1 or in the flush to oplens, and a whole-clip crop lays out exactly as
Plan.simulate_oneshot (P_lo is the first boundary whose E is the largest E <= o0, so that a crop from output 0 starts at
0 however many blocks the latency takes).  The crop extents (Plan.oneshot_crop_extents) against the compiled
reference's impulse columns, and every refusal of the crop calls."""
import numpy as np
import pytest

from __graft_entry__ import load_package
from test_oneshot_long_cpu import CHAINS, MAX_IN, plan_of, twin_totals

pkg = load_package()

LANES = [1, 7, 64]


def crop_set(seed, length, oplen, E):
    """(clip 0) crops covering the cases of the layout: o0 = 0, the latency ramp, block boundaries, empty crops, E(len)
    exactly, the flush tail, the whole clip and overlaps."""
    rng = np.random.default_rng(seed)
    Elen = int(E[-1])
    c = [(0, min(5, oplen)), (min(3, oplen), min(40, oplen)), (0, oplen), (oplen, oplen), (min(Elen, oplen), oplen)]
    c.append((max(0, min(Elen, oplen) - 30), min(Elen, oplen)))           # ends exactly at E(len)
    c.append((max(0, min(Elen, oplen) - 7), oplen))                       # reaches into the flush tail
    for b in E[1:-1][:3]:                                                 # straddle block boundaries
        c.append((max(0, int(b) - 11), min(oplen, int(b) + 13)))
    for _ in range(4):
        a = int(rng.integers(0, oplen + 1))
        c.append((a, int(rng.integers(a, oplen + 1))))
    a = int(rng.integers(0, oplen + 1))
    c.append((a, a))                                                      # empty
    if oplen > 50:
        c.append((oplen // 3, oplen // 2))
        c.append((oplen // 4, 2 * oplen // 3))                            # overlapping the one before
    return np.array([(0, a, b) for a, b in c], dtype=np.int64)


@pytest.mark.parametrize("src,dst,tb", CHAINS)
@pytest.mark.parametrize("lanes", LANES)
def test_crop_layout(src, dst, tb, lanes):
    plan = plan_of(src, dst, tb)
    B = MAX_IN
    W = plan.oneshot_warmup
    for seed, length in enumerate([1, B, 5 * B + 17, 23 * B + 1000]):
        oplen = plan.default_target(length)
        E = twin_totals(plan, length, B)
        nb = len(E) - 1
        crops = crop_set(seed, length, oplen, E)
        segs, n_calls = plan.simulate_oneshot_crops(lanes, [length], crops)
        assert n_calls >= 0
        for k, (_, o0, o1) in enumerate(crops):
            mine = np.sort(segs[segs["clip"] == k], order="e0")
            if o1 == o0:
                assert len(mine) == 0
                continue
            # the kept ranges tile [o0, o1)
            assert mine["e0"][0] == o0 and mine["e1"][-1] == o1
            assert np.all(mine["e0"][1:] == mine["e1"][:-1])
            assert np.all(mine["e1"] > mine["e0"])
            # the first segment starts W before P_lo
            e_lo = max(E[b] for b in range(max(nb, 1)) if E[b] <= o0)
            p_lo = min(b for b in range(max(nb, 1)) if E[b] == e_lo) * B
            # (segments of blocks with no output keep nothing and do not run: the first that runs starts past them)
            first = mine[np.argmin(mine["p0"])]
            assert first["p0"] >= p_lo and E[first["p0"] // B] == e_lo
            assert first["start"] == max(0, first["p0"] - W)
            # the span ends at the first boundary with E >= o1, or in the flush
            last = mine[np.argmax(mine["p1"])]
            ends = [b for b in range(nb + 1) if E[b] >= o1]
            if ends:
                assert last["p1"] == min(ends[0] * B, length)
            else:
                assert last["p1"] == length
            assert np.all(mine["p1"] - mine["p0"] >= 0)
        assert np.all(np.bincount(segs["round"] * lanes + segs["lane"]) <= 1)


@pytest.mark.parametrize("src,dst,tb", CHAINS)
@pytest.mark.parametrize("lanes", LANES)
def test_whole_clip_crop_is_the_long_clip_layout(src, dst, tb, lanes):
    plan = plan_of(src, dst, tb)
    lens = np.array([1, MAX_IN - 1, 3 * MAX_IN, 5 * MAX_IN + 17, 40 * MAX_IN + 3], dtype=np.int64)
    op = np.array([plan.default_target(int(v)) for v in lens], dtype=np.int64)
    crops = np.stack([np.arange(len(lens)), np.zeros(len(lens), np.int64), op], axis=1)
    a, na = plan.simulate_oneshot(lanes, lens, op)
    b, nb_ = plan.simulate_oneshot_crops(lanes, lens, crops, op)
    assert np.array_equal(a, b)
    # the same calls, but for the whole clips' flushes that add nothing (oplen == E(len): passthrough)
    assert nb_ == na or (plan.passthrough and nb_ < na)


def test_crops_of_one_clip_share_the_clip_and_spread_over_lanes():
    """Many short crops of one long clip still fill the lanes: segments of the fewest blocks that fit."""
    plan = plan_of(48000.0, 16000.0, 2.0)
    length = 400 * MAX_IN
    op = plan.default_target(length)
    rng = np.random.default_rng(3)
    a = rng.integers(0, op - 5000, 32)
    crops = np.stack([np.zeros(32, np.int64), a, a + 4000], axis=1)
    segs, n_calls = plan.simulate_oneshot_crops(64, [length], crops)
    assert len(np.unique(segs["clip"])) == 32
    assert segs["round"].max() == 0          # one round
    W = plan.oneshot_warmup
    assert n_calls <= (W + 4000 * 3 + 2 * MAX_IN) // MAX_IN + 1


def test_refusals():
    plan = plan_of(44100.0, 48000.0, 2.0)
    lens = [10000]
    op = plan.default_target(10000)
    cases = [
        ([(1, 0, 5)], "crops\\[0\\].clip = 1 is not a clip of the call"),
        ([(-1, 0, 5)], "crops\\[0\\].clip = -1 is not a clip"),
        ([(0, 0, 5), (0, -1, 5)], "crops\\[1\\].o0 = -1 is negative"),
        ([(0, 7, 5)], "crops\\[0\\].o1 = 5 is before o0 = 7"),
        ([(0, 0, op + 1)], "crops\\[0\\].o1 = %d is past oplens\\[0\\] = %d" % (op + 1, op)),
    ]
    for crops, msg in cases:
        with pytest.raises(pkg.R8bGpuError, match=msg):
            plan.simulate_oneshot_crops(4, lens, crops)
    assert plan.simulate_oneshot_crops(4, lens, np.zeros((0, 3), np.int64))[0].size == 0
    t = pkg.Plan.trim(44100.0, 48000.0, MAX_IN, 2.0, pkg.ATTEN_24, 0.01)
    with pytest.raises(pkg.R8bGpuError, match="trim plans"):
        t.simulate_oneshot_crops(4, lens, [(0, 0, 5)])
    with pytest.raises(pkg.R8bGpuError, match="trim plans"):
        t.oneshot_crop_extents(100, 100, 0, 5)
    with pytest.raises(pkg.R8bGpuError, match="within"):
        plan.oneshot_crop_extents(100, 100, 5, 4)
    with pytest.raises(pkg.R8bGpuError, match="within"):
        plan.oneshot_crop_extents(100, 100, 0, 101)


def test_refusals_without_a_device_change_nothing():
    """The batch calls check everything before they touch a device: with no batch there is nothing to change, and the
    crop checks' messages come first for the host form too."""
    L = pkg.lib()
    import ctypes as C
    cr = pkg._crops([(0, 0, 5)])
    lens = np.array([100], dtype=np.int64)
    assert L.r8bgpu_batch_oneshot_crops(None, None, 1, None, lens.ctypes.data, None, 1, cr.ctypes.data, None, None) == -1
    assert "batch_oneshot_crops: bad arguments" in pkg._err()
    assert L.r8bgpu_batch_oneshot_crops_adjoint(None, None, 1, None, lens.ctypes.data, None, 1, cr.ctypes.data, None) == -1
    assert "batch_oneshot_crops_adjoint: bad arguments" in pkg._err()


@pytest.mark.parametrize("src,dst,tb", CHAINS)
def test_extents_nest_and_match_the_whole_clip(src, dst, tb):
    plan = plan_of(src, dst, tb)
    n = 7 * MAX_IN + 33
    op = plan.default_target(n)
    lo, hi = plan.oneshot_crop_extents(n, op, 0, op)
    assert np.array_equal(hi, plan.oneshot_adjoint_extents(n, op))
    for o0, o1 in [(0, 10), (op // 3, op // 2), (op - 20, op), (op // 2, op // 2)]:
        lo, hi = plan.oneshot_crop_extents(n, op, o0, o1)
        if o1 == o0:
            assert np.all(lo == 0) and np.all(hi == 0)
            continue
        assert np.all(lo <= hi) and np.all(lo >= 0)
        assert np.array_equal(hi, plan.oneshot_adjoint_extents(n, o1))
        lo2, hi2 = plan.oneshot_crop_extents(n, op, max(0, o0 - 5), o1)
        assert np.all(lo2 <= lo)
        for j, st in enumerate(plan.stages()):
            if st["kind"] == 4:
                assert lo[j] % 2 == 0


# ---- extents against the compiled reference --------------------------------------------------------------------------
THR = 1e-12

ou = pytest.importorskip("oracle_util")
needs_ref = pytest.mark.skipif(not ou.have_ref("e0"), reason="compiled reference (oracle/_ref) not built")

REF_CHAINS = [
    (44100.0, 96000.0, MAX_IN, 2.0, pkg.ATTEN_24),
    (48000.0, 44100.0, MAX_IN, 2.0, pkg.ATTEN_24),
    (48000.0, 47999.0, MAX_IN, 2.0, pkg.ATTEN_24),
    (192000.0, 44100.0, MAX_IN, 2.0, pkg.ATTEN_24),
    (44100.0, 176400.0, MAX_IN, 2.0, pkg.ATTEN_24),
    (48000.0, 16000.0, MAX_IN, 2.0, pkg.ATTEN_24),
    (16000.0, 8000.0, 16384, 10.0, 80.0),      # 1/2 block-exact
]


def _columns(run, cols):
    return [c for c in cols if np.any(np.abs(run(c)) > THR)]


def _reach(st):
    if st["kind"] == 0:
        if st["down"] in (2, 4) and st["ref_input_len"] > 0:
            return (st["ref_input_len"] + st["kernel_len"]) // max(st["up"], 1) + 2
        return (st["kernel_len"] // 2) // max(st["up"], 1) + 2
    return 128


@needs_ref
@pytest.mark.parametrize("src,dst,max_in,tb,atten", REF_CHAINS)
def test_chain_crop_extents_against_reference(src, dst, max_in, tb, atten):
    """No input outside [lo_0, hi_0) reaches a kept output of the reference's oneshot(), and the first and last that do
    lie within the first stage's tap reach of lo_0 and hi_0."""
    plan = pkg.Plan(src, dst, max_in, tb, atten)
    rs = ou.RefOracle("e0").Resampler(src, dst, max_in, tb, atten)
    n = 3 * max_in + 57
    oplen = plan.default_target(n)
    o0, o1 = oplen // 3, oplen // 3 + 200
    lo, hi = plan.oneshot_crop_extents(n, oplen, o0, o1)
    lo0, hi0 = int(lo[0]), int(hi[0])
    assert 0 < lo0 < hi0 < n

    def run(c):
        e = np.zeros(n)
        e[c] = 1.0
        return rs.oneshot(e, oplen)[o0:o1]
    reach = _reach(plan.stages()[0])
    outside = list(range(max(0, lo0 - reach - 64), lo0)) + list(range(hi0, min(n, hi0 + 64)))
    assert _columns(run, outside) == []
    first = _columns(run, range(lo0, min(hi0, lo0 + reach + 1)))
    assert first and first[0] - lo0 <= reach
    last = _columns(run, range(hi0 - 1, max(lo0, hi0 - reach - 2), -1))
    assert last and hi0 - 1 - last[0] <= reach


SINGLE = [
    (0, [0.5, 10.0, 80.0, 1.0, 1, 1], ("blockconv", 0.5, 10.0, 80.0, 1.0, 1, 1)),
    (0, [0.5, 10.0, 80.0, 2.0, 2, 1], ("blockconv", 0.5, 10.0, 80.0, 2.0, 2, 1)),
    (0, [0.25, 10.0, 80.0, 1.0, 1, 2], ("blockconv", 0.25, 10.0, 80.0, 1.0, 1, 2)),   # block-exact 1/2
    (0, [1.0 / 3, 10.0, 80.0, 2.0, 2, 3], ("blockconv", 1.0 / 3, 10.0, 80.0, 2.0, 2, 3)),
    (1, [48000.0, 44100.0, 80.0, 0], ("frac", 48000.0, 44100.0, 80.0, False)),
    (3, [80.0, 2, 0], ("hbup", 80.0, 2, False)),
    (4, [80.0, 2, 0], ("hbdown", 80.0, 2, False)),
]


@needs_ref
@pytest.mark.parametrize("kind,params,refargs", SINGLE)
def test_single_stage_crop_extents_against_reference(kind, params, refargs):
    max_in = 1024
    p = pkg.Plan.single_stage(kind, params, max_in)
    ref = ou.RefOracle("e0")
    mk = lambda: getattr(ref, "stage_" + refargs[0])(*refargs[1:])
    n, oplen = 3000, 1500
    o0, o1 = 400, 600
    lo, hi = p.oneshot_crop_extents(n, oplen, o0, o1)
    lo0, hi0 = int(lo[0]), int(hi[0])
    assert 0 < lo0 < hi0 < n

    def run(c):
        st = mk()
        x = np.zeros(n + max_in * 64)
        x[c] = 1.0
        out, pos = [], 0
        while sum(len(o) for o in out) < o1:
            out.append(st.process(x[pos:pos + max_in]))
            pos += max_in
        return np.concatenate(out)[o0:o1]
    st = p.stages()[0]
    slack = {0: 2 + 2 * st["down"], 1: 2, 2: 2, 3: 1, 4: 1}[kind]
    if kind == 0 and st["down"] in (2, 4) and st["ref_input_len"] > 0:
        slack = (st["ref_input_len"] + st["kernel_len"]) // max(st["up"], 1) + 2
    outside = list(range(max(0, lo0 - 64), lo0)) + list(range(hi0, min(n, hi0 + 64)))
    assert _columns(run, outside) == []
    first = _columns(run, range(lo0, min(hi0, lo0 + slack + 1)))
    assert first and first[0] - lo0 <= slack, (lo0, first[:1], slack)
    last = _columns(run, range(hi0 - 1, max(lo0, hi0 - slack - 2), -1))
    assert last and hi0 - 1 - last[0] <= slack
