"""Per-channel rate trim on the host (no GPU): trim plans, their refusals, and the order-2 timing they schedule.

A trim plan is the chain of (src, dst) with its interpolator always the order-2 bank; each channel's interpolator then
runs at dsr = fl(dst * f) times the chain's power-of-two factor, and a new factor re-bases the position the way the
reference re-bases it every 1000 outputs (CDSPFracInterpolator.h:907-919).  These tests hold the host scheduler to:
  - the compiled reference at (src, fl(dst * f)) for a constant factor (its counts);
  - an ordinary plan's schedule at f = 1;
  - a float64 restatement of the timing for factors that change every call (counts and read positions, bit for bit).
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import oracle_util  # noqa: E402


def _pkg():
    import __graft_entry__
    return __graft_entry__.load_package()


A16, A24 = 136.45, 180.15


def _err(fn):
    with pytest.raises(_pkg().R8bGpuError) as ei:
        fn()
    return str(ei.value)


# ---- refusals ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mt", [0.0, -1e-4, 0.0100001, 0.5, float("nan")])
def test_max_trim_out_of_range(mt):
    m = _err(lambda: _pkg().Plan.trim(44100.0, 48000.0, 1024, 2.0, A24, mt))
    assert "max_trim must lie in (0, 0.01]" in m, m


def test_passthrough_refused():
    m = _err(lambda: _pkg().Plan.trim(48000.0, 48000.0, 1024, 2.0, A24, 1e-3))
    assert "passthrough" in m, m


@pytest.mark.parametrize("src,dst", [(44100.0, 88200.0), (44100.0, 352800.0), (48000.0, 16000.0), (96000.0, 48000.0)])
def test_chain_without_interpolator_refused(src, dst):
    P = _pkg()
    assert all(s["name"] not in ("frac_poly", "frac_whole") for s in P.Plan(src, dst, 1024, 2.0, A24).stages())
    m = _err(lambda: P.Plan.trim(src, dst, 1024, 2.0, A24, 1e-3))
    assert "no fractional interpolator" in m, m


def test_whole_stepping_pair_gets_the_order2_bank():
    P = _pkg()
    nominal = [s["name"] for s in P.Plan(44100.0, 96000.0, 1024, 2.0, A24).stages()]
    trim = [s["name"] for s in P.Plan.trim(44100.0, 96000.0, 1024, 2.0, A24, 1e-3).stages()]
    assert nominal == ["blockconv", "frac_whole"]
    assert trim == ["blockconv", "frac_poly"]


def test_simulate_trim_refusals():
    P = _pkg()
    tp = P.Plan.trim(44100.0, 48000.0, 1024, 2.0, A24, 2e-4)
    m = _err(lambda: tp.simulate_trim([100], [1.0 + 3e-4]))
    assert "factor outside [1 - max_trim, 1 + max_trim]" in m, m
    m = _err(lambda: tp.simulate_trim([1025], [1.0]))
    assert "block length" in m, m
    m = _err(lambda: P.Plan(44100.0, 48000.0, 1024, 2.0, A24).simulate_trim([100], [1.0]))
    assert "not a trim plan" in m, m


def test_default_flush_refused_on_a_trim_plan():
    P = _pkg()
    tp = P.Plan.trim(44100.0, 48000.0, 1024, 2.0, A24, 1e-3)
    assert P.lib().r8bgpu_plan_flush_max_out_len(tp._h) < 0
    assert "explicit" in P._err() and "targets" in P._err()
    m = _err(lambda: tp.simulate_flush([1000, 1000]))
    assert "no default flush target" in m, m
    z, n = tp.simulate_flush([1000, 1000], target=2500)  # explicit targets work
    assert n == 2500 - int(np.sum(tp.simulate([1000, 1000])))


def test_max_out_len_is_the_largest_factors():
    P = _pkg()
    for src, dst in [(44100.0, 48000.0), (48000.0, 44100.0), (44100.0, 192000.0), (96000.0, 44100.0)]:
        M = 4096
        mt = 0.01
        tp = P.Plan.trim(src, dst, M, 2.0, A24, mt)
        assert tp.max_trim == mt
        assert tp.max_out_len >= P.Plan(src, dst, M, 2.0, A24).max_out_len
        # every factor's schedule fits: the longest call after any history produces at most max_out_len
        rng = np.random.default_rng(5)
        for f in (1 - mt, 1.0, 1 + mt):
            counts = tp.simulate_trim([M] * 40 + list(rng.integers(0, M + 1, 40)), [f] * 80)
            assert counts.max() <= tp.max_out_len


# ---- constant factor: the reference at (src, fl(dst * f)) --------------------------------------------------------------

# upsampling chains 2x BlockConvolver + interpolator, whose filters depend on src and the attenuation only; the
# transition band keeps the reference's chain the same over +-1 % (no intermediate 2x step)
UP_CHAINS = [(44100.0, 48000.0, 2.0), (44100.0, 96000.0, 6.0), (22050.0, 48000.0, 6.0)]


def _factors(seed, n=20, span=0.01):
    return np.random.default_rng(seed).uniform(1.0 - span, 1.0 + span, n)


@pytest.mark.skipif(not oracle_util.have_ref(), reason="compiled reference (oracle/_ref) not built")
@pytest.mark.parametrize("atten", [A16, A24])
@pytest.mark.parametrize("src,dst,tb", UP_CHAINS)
def test_constant_factor_counts_match_the_reference(src, dst, tb, atten):
    P = _pkg()
    ref = oracle_util.RefOracle("e0")
    M = 2048
    tp = P.Plan.trim(src, dst, M, tb, atten, 0.01)
    kinds = [(s["name"], s["kernel_len"]) for s in tp.stages()]
    assert [k for k, _ in kinds] == ["blockconv", "frac_poly"]
    for i, f in enumerate(_factors(int(src + dst + atten))):
        d2 = dst * f  # fl(dst * f)
        # our planner picks the order-2 bank at fl(dst * f), on the same chain with the same filters
        op = P.Plan(src, d2, M, tb, atten)
        assert [(s["name"], s["kernel_len"]) for s in op.stages()] == kinds
        ok, _, _ = ref.whole_stepping(2.0 * src, d2)
        assert not ok
        rng = np.random.default_rng(i)
        lens = rng.integers(0, M + 1, 24)
        lens[rng.random(24) < 0.2] = 0
        want = []
        r = ref.Resampler(src, d2, M, tb, atten)
        for l in lens:
            want.append(len(r.process(np.zeros(int(l)))))
        got = tp.simulate_trim(lens, [f] * len(lens))
        assert list(got) == want, (f, list(got), want)
        assert list(got) == op.simulate(lens)


# ---- f = 1: an ordinary plan's schedule --------------------------------------------------------------------------------

@pytest.mark.parametrize("dst", [47999.0, 48001.0, 47990.0])
def test_unit_factor_counts_equal_the_ordinary_plan(dst):
    P = _pkg()
    M = 4096
    op = P.Plan(48000.0, dst, M, 2.0, A24)
    assert [s["name"] for s in op.stages()] == ["blockconv", "frac_poly"]
    tp = P.Plan.trim(48000.0, dst, M, 2.0, A24, 1e-3)
    assert [(s["name"], s["kernel_len"], s["latency"]) for s in tp.stages()] == \
        [(s["name"], s["kernel_len"], s["latency"]) for s in op.stages()]
    rng = np.random.default_rng(int(dst))
    lens = rng.integers(0, M + 1, 300)
    assert list(tp.simulate_trim(lens, np.ones(len(lens)))) == op.simulate(lens)


# ---- piecewise factors: a float64 restatement of the timing ------------------------------------------------------------

def restate(plan, src, dst, lens, factors, outputs=None):
    """The order-2 timing of a BlockConvolver (1x or 2x) + interpolator chain, call by call, in the reference's float64
    order: NextInPos = ((InCounter + InPosShift) * ssr) / dsr; a factor change re-bases (InPosShift = fpos * dsr / ssr,
    InCounter = InPosInt = 0); after a call, InCounter > 1000 re-bases with the same dsr.  Returns (counts, p, fpos)
    after each call; `outputs` (a list) receives (p, fpos) of every output."""
    st = plan.stages()
    assert [s["name"] for s in st] == ["blockconv", "frac_poly"] and st[0]["down"] == 1
    up, lat = st[0]["up"], st[0]["latency"]
    fl2 = st[1]["kernel_len"] // 2
    ssr = up * src
    ic, ipi, ips, fpos, p = 0, 0, 0.0, 0.0, 0
    dsr = dst
    n_in = 0
    counts, ps, fs = [], [], []
    for l, f in zip(lens, factors):
        d = dst * f
        if d != dsr:
            dsr = d
            ips = fpos * dsr / ssr
            ic, ipi = 0, 0
        n_in += int(l)
        n1 = max(0, up * n_in - lat)  # the BlockConvolver's output so far
        pmax = n1 - 1 - fl2
        cnt = 0
        while p <= pmax:
            if outputs is not None:
                outputs.append((p, fpos))
            cnt += 1
            ic += 1
            npos = (float(ic) + ips) * ssr / dsr
            ni = int(npos)
            p += ni - ipi
            ipi = ni
            fpos = npos - ni
        if ic > 1000:
            ic, ipi = 0, 0
            ips = fpos * dsr / ssr
        counts.append(cnt)
        ps.append(p)
        fs.append(fpos)
    return counts, ps, fs


def random_walk(rng, n, ppm=200.0, step=20.0):
    f = np.empty(n)
    x = 0.0
    for i in range(n):
        x = float(np.clip(x + rng.normal(0.0, step), -ppm, ppm))
        f[i] = 1.0 + x * 1e-6
    return f


@pytest.mark.parametrize("src,dst", [(44100.0, 48000.0), (48000.0, 44100.0), (48000.0, 47999.0), (96000.0, 44100.0)])
@pytest.mark.parametrize("seed", [1, 2])
def test_piecewise_factors_match_the_restated_timing(src, dst, seed):
    P = _pkg()
    M = 1024
    tp = P.Plan.trim(src, dst, M, 2.0, A24, 2e-4)
    rng = np.random.default_rng(seed)
    n = 120
    lens = rng.integers(0, M + 1, n)
    fs = random_walk(rng, n)
    fs[10:20] = fs[9]  # runs of equal factors: no re-base, the 1000-output re-base alone
    counts, pos, frac = tp.simulate_trim(lens, fs, timing=True)
    c2, p2, f2 = restate(tp, src, dst, lens, fs)
    assert list(counts) == c2
    assert list(pos) == p2
    assert frac.tobytes() == np.array(f2).tobytes()
    # the factors do move the timing: the same lengths at f = 1 read elsewhere
    _, _, fr1 = tp.simulate_trim(lens, np.ones(n), timing=True)
    assert fr1.tobytes() != frac.tobytes()


def test_same_factor_again_does_nothing():
    P = _pkg()
    tp = P.Plan.trim(44100.0, 48000.0, 1024, 2.0, A24, 1e-3)
    lens = [700] * 30
    f = 1.0 + 1.234e-4
    a = tp.simulate_trim(lens, [f] * 30, timing=True)
    # setting f anew before every call is the same as setting it once: no re-base
    c, p, fr = restate(tp, 44100.0, 48000.0, lens, [f] * 30)
    assert list(a[0]) == c and list(a[1]) == p and a[2].tobytes() == np.array(fr).tobytes()


def test_trim_symbols_bound():
    P = _pkg()
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "r8bgpu.h")).read()
    for name in ("r8bgpu_plan_create_trim", "r8bgpu_plan_max_trim", "r8bgpu_plan_simulate_trim", "r8bgpu_batch_set_trim",
                 "r8bgpu_batch_trim"):
        assert name in hdr and name in P._SYMBOLS
        assert getattr(P.lib(), name) is not None
