"""Trim plans for every rate pair (Plan.asrc, r8bgpu_plan_create_asrc) on the host (no GPU).

Where Plan.trim accepts a pair, Plan.asrc is the same plan.  Elsewhere -- src == dst, and the integer and power-of-two
ratios the reference plans without an interpolator -- it skips exactly the constructor's shortcuts that build none
(CDSPResampler.h:135-216, 354-363) and keeps every other decision.  These tests pin those chains and hold their timing
to the compiled reference at (src, fl(dst * f)) where the ordinary planner builds the same stages, and everywhere to a
float64 restatement of the whole chain's counts and the interpolator's read positions.
"""
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import oracle_util  # noqa: E402
from test_trim_cpu import A16, A24, random_walk  # noqa: E402


def _pkg():
    import __graft_entry__
    return __graft_entry__.load_package()


def _err(fn):
    with pytest.raises(_pkg().R8bGpuError) as ei:
        fn()
    return str(ei.value)


# ---- the forced chains -------------------------------------------------------------------------------------------------

# (src, dst, tb) -> [(stage, up, down), ...] and the interpolator's (src, dst) as the stage sees them
FORCED = {
    (48000.0, 48000.0, 2.0): ([("blockconv", 2, 1), ("frac_poly", 1, 1)], (96000.0, 48000.0)),
    (44100.0, 88200.0, 2.0): ([("blockconv", 2, 1), ("frac_poly", 1, 1)], (88200.0, 88200.0)),
    (48000.0, 96000.0, 2.0): ([("blockconv", 2, 1), ("frac_poly", 1, 1)], (96000.0, 96000.0)),
    (16000.0, 48000.0, 2.0): ([("blockconv", 2, 1), ("frac_poly", 1, 1)], (32000.0, 48000.0)),
    (44100.0, 176400.0, 2.0): ([("blockconv", 2, 1), ("frac_poly", 1, 1)], (88200.0, 176400.0)),
    (44100.0, 352800.0, 2.0): ([("blockconv", 2, 1), ("frac_poly", 1, 1), ("blockconv", 2, 1), ("hbup", 1, 1)],
                               (352800.0, 352800.0)),
    (48000.0, 32000.0, 2.0): ([("blockconv", 2, 1), ("frac_poly", 1, 1)], (96000.0, 32000.0)),
    (32000.0, 48000.0, 2.0): ([("blockconv", 2, 1), ("frac_poly", 1, 1)], (64000.0, 48000.0)),
    (48000.0, 36000.0, 2.0): ([("blockconv", 2, 1), ("frac_poly", 1, 1)], (96000.0, 36000.0)),
    (96000.0, 48000.0, 2.0): ([("blockconv", 1, 1), ("frac_poly", 1, 1)], (96000.0, 48000.0)),
    (48000.0, 16000.0, 2.0): ([("blockconv", 1, 1), ("frac_poly", 1, 1)], (48000.0, 16000.0)),
    (192000.0, 48000.0, 2.0): ([("hbdown", 1, 1), ("blockconv", 1, 1), ("frac_poly", 1, 1)], (192000.0, 96000.0)),
}
PAIRS = sorted({(s, d) for s, d, _ in FORCED})
# At TB 40 the intermediate 2x steps start further up: 44100 -> 352800 interpolates 88200 -> 352800 directly (c = 1, and
# 88200 -> 352800 steps in whole numbers, so the whole-stepping preference gives c = 0); every other chain is the TB 2 one.
for _s, _d in PAIRS:
    FORCED[(_s, _d, 40.0)] = FORCED[(_s, _d, 2.0)]
FORCED[(44100.0, 352800.0, 40.0)] = ([("blockconv", 2, 1), ("frac_poly", 1, 1)], (88200.0, 352800.0))

# the BlockConvolvers' normalised cut-off (describe(), 4 digits) and the interpolator's third-band flag, at any TB
NORM_FREQ = {(48000.0, 32000.0): [0.3333], (48000.0, 36000.0): [0.375], (48000.0, 16000.0): [0.3333]}
THIRD = {(48000.0, 16000.0)}


def describe_rates(plan):
    """(normalised cut-offs of the BlockConvolvers, (src, dst, third) of the interpolator) from plan.describe()."""
    d = plan.describe()
    nf = [float(v) for v in re.findall(r"nfreq=([0-9.]+)", d)]
    m = re.search(r"FracInterp: src=([0-9.]+) dst=([0-9.]+) .* third=(\d)", d)
    return nf, (float(m.group(1)), float(m.group(2)), int(m.group(3)))


@pytest.mark.parametrize("atten", [A16, A24])
@pytest.mark.parametrize("tb", [2.0, 40.0])
@pytest.mark.parametrize("src,dst", PAIRS)
def test_forced_chain_is_pinned(src, dst, tb, atten):
    P = _pkg()
    with pytest.raises(P.R8bGpuError):  # the pairs Plan.trim refuses
        P.Plan.trim(src, dst, 1024, tb, atten, 1e-3)
    ap = P.Plan.asrc(src, dst, 1024, tb, atten, 1e-3)
    want, (fs, fd) = FORCED[(src, dst, tb)]
    assert [(s["name"], s["up"], s["down"]) for s in ap.stages()] == want
    nf, frac = describe_rates(ap)
    assert frac == (fs, fd, int((src, dst) in THIRD))
    assert nf[0] == NORM_FREQ.get((src, dst), [0.5])[0]
    if len(nf) > 1:  # the 2x BlockConvolver behind the interpolator
        assert nf[1] == 0.5
    assert ap.max_trim == 1e-3 and not ap.passthrough


# ---- where Plan.trim accepts the pair: the same plan -------------------------------------------------------------------

RATES = [8000.0, 11025.0, 16000.0, 22050.0, 32000.0, 44100.0, 48000.0, 88200.0, 96000.0, 176400.0, 192000.0, 384000.0]


def seeded_pairs(rng, n):
    """Rate pairs within 40x, a quarter of them moved off the standard rates (odd ratios)."""
    out = []
    while len(out) < n:
        a, b = rng.choice(RATES, 2, replace=False)
        if rng.random() < 0.25:
            b = float(b) + float(rng.integers(1, 50))
        if a / b > 40 or b / a > 40:
            continue
        out.append((float(a), float(b)))
    return out


def plan_bytes(plan):
    return ([(s["name"], s["up"], s["down"], s["kernel_len"], s["latency"], s["max_out_len"]) for s in plan.stages()],
            [plan.stage_data(i).tobytes() for i in range(len(plan.stages()))], plan.state_fingerprint, plan.max_out_len)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_same_plan_where_trim_accepts(seed):
    P = _pkg()
    rng = np.random.default_rng(seed)
    same = 0
    for src, dst in seeded_pairs(rng, 24):
        tb = float(rng.choice([2.0, 3.0, 8.0, 40.0]))
        atten = float(rng.choice([A16, A24, 206.91]))
        M = int(rng.choice([512, 2048, 4096]))
        mt = float(rng.choice([1e-4, 2e-4, 0.01]))
        ap = P.Plan.asrc(src, dst, M, tb, atten, mt)
        try:
            tp = P.Plan.trim(src, dst, M, tb, atten, mt)
        except P.R8bGpuError:
            assert "frac_poly" in [s["name"] for s in ap.stages()]
            continue
        same += 1
        assert plan_bytes(ap) == plan_bytes(tp)
        lens = rng.integers(0, M + 1, 60)
        fs = random_walk(rng, 60, ppm=mt * 1e6, step=mt * 1e5)
        a, t = ap.simulate_trim(lens, fs, timing=True), tp.simulate_trim(lens, fs, timing=True)
        for u, v in zip(a, t):
            assert u.tobytes() == v.tobytes()
    assert same >= 12


# ---- the timing of the forced chains -----------------------------------------------------------------------------------

def emitted(s, n):
    """A stage's closed-form output count after n inputs (r8b_plan.h)."""
    if s["name"] == "blockconv":
        a = s["up"] * n - s["latency"]
        return 0 if a <= 0 else -(-a // s["down"])
    if s["name"] == "hbup":
        return 2 * max(0, n - s["kernel_len"])
    if s["name"] == "hbdown":
        return max(0, n // 2 - (s["kernel_len"] - 1))
    raise AssertionError(s["name"])


def restate_chain(plan, dst, lens, factors, outputs=None, frac_counts=None):
    """The order-2 timing of any chain with one interpolator, call by call, in the reference's float64 order (as
    test_trim_cpu.restate), with the stages before and after it counted by their closed forms.  The interpolator runs at
    ssr = its own src rate and dsr = fl(dst * f) * (its dst rate / dst).  Returns (counts, p, fpos) after each call;
    `outputs` (a list) receives (p, fpos) of every interpolator output, `frac_counts` (a list) the interpolator's
    output count of every call."""
    st = plan.stages()
    k = next(i for i, s in enumerate(st) if s["name"] == "frac_poly")
    _, (ssr, sdst, _) = describe_rates(plan)
    fl2 = st[k]["kernel_len"] // 2
    ic, ipi, ips, fpos, p = 0, 0, 0.0, 0.0, 0
    dsr = sdst
    n_in, n_frac = 0, 0
    counts, ps, fs = [], [], []
    for l, f in zip(lens, factors):
        d = (dst * f) * (sdst / dst)
        if d != dsr:
            dsr = d
            ips = fpos * dsr / ssr
            ic, ipi = 0, 0
        n_in += int(l)
        n = n_in
        for s in st[:k]:
            n = emitted(s, n)
        pmax = n - 1 - fl2
        while p <= pmax:
            if outputs is not None:
                outputs.append((p, fpos))
            n_frac += 1
            ic += 1
            npos = (float(ic) + ips) * ssr / dsr
            ni = int(npos)
            p += ni - ipi
            ipi = ni
            fpos = npos - ni
        if ic > 1000:
            ic, ipi = 0, 0
            ips = fpos * dsr / ssr
        if frac_counts is not None:
            frac_counts.append(n_frac - sum(frac_counts))
        n = n_frac
        for s in st[k + 1:]:
            n = emitted(s, n)
        counts.append(n - sum(counts))
        ps.append(p)
        fs.append(fpos)
    return counts, ps, fs


FACTORS = [1.0 - 1.7e-4, 1.0 - 3e-6, 1.0, 1.0 + 4e-7, 1.0 + 2e-4]


@pytest.mark.parametrize("tb", [2.0, 40.0])
@pytest.mark.parametrize("src,dst", PAIRS)
def test_forced_chain_timing_matches_the_restatement(src, dst, tb):
    P = _pkg()
    M = 2048
    ap = P.Plan.asrc(src, dst, M, tb, A24, 2e-4)
    rng = np.random.default_rng(int(src + dst + tb))
    n = 150
    lens = rng.integers(0, M + 1, n)
    lens[rng.random(n) < 0.1] = 0
    for fs in [np.full(n, f) for f in FACTORS] + [random_walk(rng, n)]:
        counts, pos, frac = ap.simulate_trim(lens, fs, timing=True)
        c2, p2, f2 = restate_chain(ap, dst, lens, fs)
        assert list(counts) == c2
        assert list(pos) == p2
        assert frac.tobytes() == np.array(f2).tobytes()
        assert sum(c2) > 0


def test_unit_factor_ratio_one_reads_every_sample_at_fraction_zero():
    """44100 -> 88200 interpolates 88200 -> 88200: at f = 1 every output reads one whole input sample further on."""
    P = _pkg()
    ap = P.Plan.asrc(44100.0, 88200.0, 1024, 2.0, A24, 1e-3)
    outs = []
    restate_chain(ap, 88200.0, [1024] * 20, np.ones(20), outs)
    assert len(outs) > 10000
    assert [p for p, _ in outs] == list(range(len(outs))) and all(f == 0.0 for _, f in outs)


def same_stage_data(a, b):
    sa, sb = a.stages(), b.stages()
    return [s["name"] for s in sa] == [s["name"] for s in sb] and \
        all(a.stage_data(i).tobytes() == b.stage_data(i).tobytes() for i in range(len(sa)))


@pytest.mark.skipif(not oracle_util.have_ref(), reason="compiled reference (oracle/_ref) not built")
@pytest.mark.parametrize("atten", [A16, A24])
@pytest.mark.parametrize("tb", [2.0, 40.0])
@pytest.mark.parametrize("src,dst", PAIRS)
def test_constant_factor_counts_match_the_reference(src, dst, tb, atten):
    """Wherever the ordinary planner at (src, fl(dst * f)) builds the same stages with the same data, a constant factor
    f gives the reference's own counts at that rate, call by call."""
    P = _pkg()
    ref = oracle_util.RefOracle("e0")
    M = 2048
    ap = P.Plan.asrc(src, dst, M, tb, atten, 2e-4)
    checked = 0
    for i, f in enumerate([1.0 - 2e-4, 1.0 - 1e-5, 1.0 + 1e-5, 1.0 + 2e-4]):
        d2 = dst * f
        op = P.Plan(src, d2, M, tb, atten)
        if not same_stage_data(ap, op):
            continue
        checked += 1
        rng = np.random.default_rng(i)
        lens = rng.integers(0, M + 1, 30)
        lens[rng.random(30) < 0.2] = 0
        r = ref.Resampler(src, d2, M, tb, atten)
        want = [len(r.process(np.zeros(int(l)))) for l in lens]
        assert list(ap.simulate_trim(lens, [f] * len(lens))) == want, f
        assert op.simulate(lens) == want
    assert checked == SAME_DATA_SIDES.get((src, dst, tb), 0)


# How many of the four factors above give the ordinary planner the forced chain's stages and data.  Upsampling chains
# 2x BlockConvolver + interpolator whose ordinary neighbours keep that chain match on both sides (their filters depend on
# src and the attenuation only); 48000 -> 48000 matches above 1 only (below, the BlockConvolver's cut-off follows dst).
# 16000 -> 48000 and 44100 -> 176400 at TB 2 owe their chain to the whole-stepping preference, which no neighbour has.
SAME_DATA_SIDES = {(48000.0, 48000.0, 2.0): 2, (48000.0, 48000.0, 40.0): 2}
for _s, _d in [(44100.0, 88200.0), (48000.0, 96000.0), (32000.0, 48000.0)]:
    SAME_DATA_SIDES[(_s, _d, 2.0)] = SAME_DATA_SIDES[(_s, _d, 40.0)] = 4
SAME_DATA_SIDES[(16000.0, 48000.0, 40.0)] = SAME_DATA_SIDES[(44100.0, 176400.0, 40.0)] = 4


# ---- plan properties ---------------------------------------------------------------------------------------------------

def test_same_rate_plan_is_not_a_passthrough_plan():
    P = _pkg()
    ap = P.Plan.asrc(48000.0, 48000.0, 1024, 2.0, A24, 1e-3)
    pp = P.Plan(48000.0, 48000.0, 1024, 2.0, A24)
    assert pp.passthrough and not ap.passthrough
    assert P.lib().r8bgpu_plan_is_passthrough(ap._h) == 0
    assert len(ap.stages()) == 2 and len(pp.stages()) == 0
    assert ap.state_fingerprint != pp.state_fingerprint
    assert ap.max_out_len == int(np.ceil(ap.stages()[0]["max_out_len"] * (48000.0 * (1.0 + 1e-3)) / 96000.0)) + 1


def test_default_flush_refused():
    P = _pkg()
    ap = P.Plan.asrc(48000.0, 48000.0, 1024, 2.0, A24, 1e-3)
    assert P.lib().r8bgpu_plan_flush_max_out_len(ap._h) < 0
    assert "explicit" in P._err()
    m = _err(lambda: ap.simulate_flush([1000, 1000]))
    assert "no default flush target" in m, m
    z, n = ap.simulate_flush([1000, 1000], target=2500)
    assert n == 2500 - int(np.sum(ap.simulate([1000, 1000])))


@pytest.mark.parametrize("mt", [0.0, -1e-4, 0.0100001, float("nan")])
def test_max_trim_out_of_range(mt):
    m = _err(lambda: _pkg().Plan.asrc(48000.0, 48000.0, 1024, 2.0, A24, mt))
    assert m.startswith("plan_create_asrc: ") and "max_trim must lie in (0, 0.01]" in m, m


@pytest.mark.parametrize("src,dst", [(float("nan"), 48000.0), (48000.0, float("nan")), (0.0, 48000.0), (48000.0, -1.0)])
def test_bad_rates_refused(src, dst):
    m = _err(lambda: _pkg().Plan.asrc(src, dst, 1024, 2.0, A24, 1e-3))
    assert "invalid sample rates or MaxInLen" in m, m


def test_trim_keeps_refusing_these_pairs():
    P = _pkg()
    assert "passthrough" in _err(lambda: P.Plan.trim(48000.0, 48000.0, 1024, 2.0, A24, 1e-3))
    assert "no fractional interpolator" in _err(lambda: P.Plan.trim(44100.0, 88200.0, 1024, 2.0, A24, 1e-3))


def test_asrc_symbol_bound():
    P = _pkg()
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "r8bgpu.h")).read()
    assert "r8bgpu_plan_create_asrc" in hdr and "r8bgpu_plan_create_asrc" in P._SYMBOLS
    assert P.lib().r8bgpu_plan_create_asrc is not None
