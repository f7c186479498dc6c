"""CPU: the extents of the transposed chain (Plan.oneshot_adjoint_extents, r8bgpu_plan_oneshot_adjoint_extents) and the
scratch a call needs (Plan.oneshot_adjoint_bytes), with no GPU.  Extents are restated in closed form on single-stage plans
and followed through whole chains: R_j of stage j is what stage j reads for the outputs stage j + 1 needs."""
import numpy as np
import pytest

from __graft_entry__ import load_package

pkg = load_package()

MAX_IN = 4096
CHAINS = [
    (44100.0, 96000.0, 2.0),
    (48000.0, 44100.0, 2.0),
    (48000.0, 47999.0, 2.0),
    (192000.0, 44100.0, 2.0),
    (44100.0, 176400.0, 2.0),
    (48000.0, 16000.0, 2.0),
    (48000.0, 16000.0, 0.5),
    (96000.0, 48000.0, 2.0),
    (32000.0, 48000.0, 30.0),
    (64000.0, 48000.0, 0.5),
]


def _chain_ok(plan, n, op):
    ext = plan.oneshot_adjoint_extents(n, op)
    assert len(ext) == len(plan.stages())
    return ext


@pytest.mark.parametrize("src,dst,tb", CHAINS)
def test_extents_monotone_and_bounded(src, dst, tb):
    plan = pkg.Plan(src, dst, MAX_IN, tb, pkg.ATTEN_24)
    prev = None
    for n in (1, 17, MAX_IN, 3 * MAX_IN + 5):
        op = plan.default_target(n)
        ext = _chain_ok(plan, n, op)
        assert np.all(ext >= 1)
        if prev is not None:
            assert np.all(ext >= prev)
        prev = ext
        # the first stage reads the clip and at most a filter's reach of the flush's zeros past it
        assert ext[0] >= min(n, 1)
    assert np.all(plan.oneshot_adjoint_extents(5000, 0) == 0)


@pytest.mark.parametrize("up,down", [(1, 1), (2, 1), (2, 3), (1, 3), (3, 1)])
def test_single_blockconv_closed_form(up, down):
    """Output q of BlockConv (U, D) reads the zero-stuffed stream at D q - L .. D q + L: R = (D (q_last) + L) // U + 1."""
    p = pkg.Plan.single_stage(0, [0.5 / max(up, down), 10.0, 80.0, float(up), up, down], MAX_IN)
    st = p.stages()[0]
    L = (st["kernel_len"] - 1) // 2
    for op in (1, 2, 101, 5000):
        assert list(p.oneshot_adjoint_extents(4 * MAX_IN, op)) == [(down * (op - 1) + L) // up + 1]


def test_passthrough_and_bytes():
    p = pkg.Plan(48000.0, 48000.0, MAX_IN, 2.0, pkg.ATTEN_24)
    assert len(p.oneshot_adjoint_extents(1000, 1200)) == 0
    assert p.oneshot_adjoint_bytes([1000, 10], [1200, 0]) >= 2 * 2 * 1202 * 8
    q = pkg.Plan(44100.0, 48000.0, MAX_IN, 2.0, pkg.ATTEN_24)
    small = q.oneshot_adjoint_bytes([MAX_IN])
    big = q.oneshot_adjoint_bytes([10 * MAX_IN, 10 * MAX_IN])
    assert big > 2 * small
    with pytest.raises(pkg.R8bGpuError, match="negative length"):
        q.oneshot_adjoint_bytes([-1])


def test_refused_plans():
    t = pkg.Plan.trim(44100.0, 48000.0, MAX_IN, 2.0, pkg.ATTEN_24, 0.01)
    with pytest.raises(pkg.R8bGpuError, match="trim"):
        t.oneshot_adjoint_extents(100, 100)


# ---- extents against the compiled reference --------------------------------------------------------------------------
# Column c of A is the reference's output for a unit impulse at input c.  An entry counts as nonzero above THR (the
# chains' gain is about 1): the reference's FFT rounding (about 1e-16) stays below it.
THR = 1e-12

ou = pytest.importorskip("oracle_util")
needs_ref = pytest.mark.skipif(not ou.have_ref("e0"), reason="compiled reference (oracle/_ref) not built")


def _last_significant_column(run, n):
    """The largest input index below n whose impulse reaches a kept output."""
    last = -1
    for c in range(n - 1, -1, -1):
        y = run(c)
        if y.size and np.any(np.abs(y) > THR):
            return c
    return last


def _chain_run(rs, n, oplen):
    def run(c):
        e = np.zeros(n)
        e[c] = 1.0
        return rs.oneshot(e, oplen)
    return run


def _stage_run(mk, n, oplen, max_in):
    def run(c):
        st = mk()
        x = np.zeros(n + max_in * 64)
        x[c] = 1.0
        out, pos = [], 0
        while sum(len(o) for o in out) < oplen:
            out.append(st.process(x[pos:pos + max_in]))
            pos += max_in
        return np.concatenate(out)[:oplen]
    return run


# CHAINS at MaxInLen 4096, and BlockConvolver geometries of tests/test_blockconv_geometry_cpu.py (BLOCKCONVS)
REF_CHAINS = [(s, d, MAX_IN, tb, pkg.ATTEN_24) for s, d, tb in CHAINS[:6] + CHAINS[7:9]] + [
    (32000.0, 48000.0, 16384, 45.0, 49.0),     # 3/2 block-exact, M 64
    (64000.0, 48000.0, 16384, 45.0, 49.0),     # 3/4 block-exact, M 128
    (16000.0, 8000.0, 16384, 10.0, 80.0),      # 1/2 block-exact, M 512
    (48000.0, 32000.0, 16384, 45.0, 49.0),     # 2/3, UP 2
    (8000.0, 48000.0, 16384, 0.5, pkg.ATTEN_24),  # 3x on the large-tile path
    (47999.0, 8000.0, 16384, 0.5, pkg.ATTEN_24),  # 1x on the large-tile path, then the order-2 bank
]


@needs_ref
@pytest.mark.parametrize("src,dst,max_in,tb,atten", REF_CHAINS)
def test_chain_extent_against_reference(src, dst, max_in, tb, atten):
    """Stage 0's extent covers every input the kept outputs of the reference's oneshot() reach, and is tight within the
    first stage's tap reach.  oplen is cut so that the extent ends inside the clip."""
    plan = pkg.Plan(src, dst, max_in, tb, atten)
    rs = ou.RefOracle("e0").Resampler(src, dst, max_in, tb, atten)
    n = 2 * max_in + 57
    oplen = plan.default_target(n) // 2
    R = int(plan.oneshot_adjoint_extents(n, oplen)[0])
    assert R < n
    run = _chain_run(rs, n, oplen)
    c_last = _last_significant_column(run, R + 64)
    assert c_last < R                         # covers the support
    st = plan.stages()[0]
    reach = {0: (st["kernel_len"] // 2) // max(st["up"], 1) + 2,
             1: 128, 2: 128, 3: 128, 4: 128}[st["kind"]]  # plus the later stages' outermost taps, which fall below THR
    if st["kind"] == 0 and st["down"] in (2, 4) and st["ref_input_len"] > 0:
        reach = (st["ref_input_len"] + st["kernel_len"]) // max(st["up"], 1) + 2  # block-exact: one block's window
    assert R - 1 - c_last <= reach, (R, c_last, reach)


SINGLE = [
    # (kind, params, reference stage factory args)
    (0, [0.5, 10.0, 80.0, 1.0, 1, 1], ("blockconv", 0.5, 10.0, 80.0, 1.0, 1, 1)),
    (0, [0.5, 10.0, 80.0, 2.0, 2, 1], ("blockconv", 0.5, 10.0, 80.0, 2.0, 2, 1)),
    (0, [0.25, 10.0, 80.0, 1.0, 1, 2], ("blockconv", 0.25, 10.0, 80.0, 1.0, 1, 2)),   # block-exact 1/2
    (0, [1.0 / 3, 10.0, 80.0, 2.0, 2, 3], ("blockconv", 1.0 / 3, 10.0, 80.0, 2.0, 2, 3)),
    (0, [1.0 / 3, 10.0, 80.0, 3.0, 3, 1], ("blockconv", 1.0 / 3, 10.0, 80.0, 3.0, 3, 1)),
    (1, [48000.0, 44100.0, 80.0, 0], ("frac", 48000.0, 44100.0, 80.0, False)),
    (3, [80.0, 2, 0], ("hbup", 80.0, 2, False)),
    (4, [80.0, 2, 0], ("hbdown", 80.0, 2, False)),
]


@needs_ref
@pytest.mark.parametrize("kind,params,refargs", SINGLE)
def test_single_stage_extent_against_reference(kind, params, refargs):
    """Each stage kind on its own (Plan.single_stage against the reference's stage class): R covers the support of the
    outputs [0, oplen) and is tight within the stage's tap reach."""
    max_in = 1024
    p = pkg.Plan.single_stage(kind, params, max_in)
    ref = ou.RefOracle("e0")
    mk = lambda: getattr(ref, "stage_" + refargs[0])(*refargs[1:])
    n, oplen = 3000, 1500
    while int(p.oneshot_adjoint_extents(n, oplen)[0]) > n - 100:  # the extent ends inside the clip
        oplen //= 2
    R = int(p.oneshot_adjoint_extents(n, oplen)[0])
    run = _stage_run(mk, n, oplen, max_in)
    c_last = _last_significant_column(run, min(R + 64, n))
    assert c_last < R
    st = p.stages()[0]
    slack = {0: 2 + 2 * st["down"], 1: 2, 2: 2, 3: 1, 4: 1}[kind]
    assert R - 1 - c_last <= slack, (R, c_last, slack)
