"""Long streams on the host scheduler (no GPU): plan buffer lengths at the R8BGPU_MAX_LEN boundary, and per-call counts
of streams that run past 2^32 input samples.

Every stage is a pure function of absolutely indexed streams, so a live stream's sample indices only grow: an always-on
48 kHz stream passes 2^32 after about a day, a DSD64 input after 25 minutes.  These tests hold the planner and the
scheduler to Python big-integer restatements of the reference's formulas there:
  - the getMaxOutLen() chain (CDSPResampler.h:677-700 and each stage's getMaxOutLen) is exact, the largest MaxInLen whose
    chain stays within R8BGPU_MAX_LEN is accepted and the next one is refused, with a message naming the stage;
  - per-call counts equal the closed-form emitted counts (r8b_plan.h, DESIGN.md section 1) call by call, past 2^32;
  - the order-2 interpolator's counts equal a float64 restatement of its timing, past 2^32.
"""
import math
import time
from fractions import Fraction

import pytest

import test_trim_cpu

LIMIT = 2 ** 31 - 2 ** 16  # R8BGPU_MAX_LEN (include/r8bgpu.h)
A24 = 180.15


def test_limit_is_the_headers():
    import os
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "r8bgpu.h")).read()
    assert "#define R8BGPU_MAX_LEN %d" % LIMIT in hdr


# ---- the buffer-length chain, restated -----------------------------------------------------------------------------------

def _ratio(st):
    """Exact output/input rate ratio of a stage other than an order-2 interpolator."""
    k = st["name"]
    if k == "blockconv":
        return Fraction(st["up"], st["down"])
    if k == "frac_whole":
        return Fraction(st["out_step"], st["in_step"])
    return Fraction(2) if k == "hbup" else Fraction(1, 2)


def _chain_ratios(stages, src, dst):
    """Per stage the exact ratio; an order-2 interpolator's is what the rest of the chain leaves of dst / src."""
    others = Fraction(1)
    for st in stages:
        if st["name"] != "frac_poly":
            others *= _ratio(st)
    return [_ratio(st) if st["name"] != "frac_poly" else Fraction(dst) / Fraction(src) / others for st in stages]


def _ceil(q):
    return -((-q.numerator) // q.denominator)


def max_out_chain(stages, ratios, m, trim=None):
    """getMaxOutLen of every stage for MaxInLen m: BlockConv ceil(m U / D), interpolators ceil(m dst / src) + 1, HBUp 2 m,
    HBDown (m + 1) / 2.  trim = (stage, dsr, ssr): that interpolator's bound at the largest factor, in the planner's
    float64 (the factor is a double by definition)."""
    out = []
    for i, (st, r) in enumerate(zip(stages, ratios)):
        k = st["name"]
        if trim is not None and i == trim[0]:
            m = math.ceil(float(m) * trim[1] / trim[2]) + 1
        elif k == "blockconv":
            m = _ceil(m * r)
        elif k in ("frac_whole", "frac_poly"):
            m = _ceil(m * r) + 1
        elif k == "hbup":
            m = 2 * m
        else:
            m = (m + 1) // 2
        out.append(m)
    return out


def largest_max_in(chain):
    """The largest MaxInLen <= LIMIT whose chain stays within LIMIT (the chain never decreases with MaxInLen)."""
    lo, hi = 1, LIMIT
    assert max(chain(1)) <= LIMIT
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if max(chain(mid)) <= LIMIT:
            lo = mid
        else:
            hi = mid - 1
    return lo


def _plan(pkg, spec, m):
    kind = spec[0]
    if kind == "rate":
        _, src, dst, ext = spec
        return pkg.Plan(src, dst, m, 2.0, A24, extfft=ext)
    if kind == "trim":
        _, src, dst, mt = spec
        return pkg.Plan.trim(src, dst, m, 2.0, A24, mt)
    _, sk, params = spec
    return pkg.Plan.single_stage(sk, params, m)


BOUNDARY = [
    ("rate", 44100.0, 2822400.0, 1),
    ("rate", 8000.0, 48000.0, 0),
    ("rate", 44100.0, 96000.0, 0),
    ("rate", 48000.0, 47999.0, 0),
    ("rate", 2822400.0, 44100.0, 0),
    ("trim", 44100.0, 48000.0, 0.01),
    ("stage", 3, [A24, 0, 0]),                           # HBUp
    ("stage", 0, [1.0 / 3.0, 2.0, A24, 3.0, 3, 1]),     # BlockConv 3/1
]


def _boundary_ids(s):
    return "%s-%s" % (s[0], "-".join(str(v) for v in (s[1:3] if s[0] != "stage" else (s[1], s[2][-2:]))))


def _chain_of(pkg, spec):
    """(stages, chain function) of spec, restated from a small plan's stage descriptions."""
    p = _plan(pkg, spec, 4096)
    stages = p.stages()
    if spec[0] == "stage":
        ratios = [Fraction(2) if stages[0]["name"] == "hbup" else Fraction(spec[2][4], spec[2][5])]
        return stages, lambda m: max_out_chain(stages, ratios, m)
    src, dst = spec[1], spec[2]
    ratios = _chain_ratios(stages, src, dst)
    trim = None
    if spec[0] == "trim":
        i = [s["name"] for s in stages].index("frac_poly")
        # this chain's interpolator runs from 2 src to dst itself (Plan::trim_dsr's power-of-two factor is 1)
        assert [s["name"] for s in stages] == ["blockconv", "frac_poly"] and stages[0]["up"] == 2
        trim = (i, dst * (1.0 + spec[3]), 2.0 * src)
    return stages, lambda m: max_out_chain(stages, ratios, m, trim)


@pytest.mark.parametrize("spec", BOUNDARY, ids=_boundary_ids)
def test_max_in_len_boundary(pkg, spec):
    stages, chain = _chain_of(pkg, spec)
    # the restatement holds at ordinary lengths too
    for m in (1, 4096, 100000):
        assert [s["max_out_len"] for s in _plan(pkg, spec, m).stages()] == chain(m)
    m = largest_max_in(chain)
    p = _plan(pkg, spec, m)
    want = chain(m)
    assert [s["max_out_len"] for s in p.stages()] == want
    assert p.max_out_len == want[-1] <= LIMIT
    with pytest.raises(pkg.R8bGpuError) as ei:
        _plan(pkg, spec, m + 1)
    msg = str(ei.value)
    assert "R8BGPU_MAX_LEN = %d" % LIMIT in msg, msg
    if m < LIMIT:
        # the refused stage is named with the length it would need
        bad = chain(m + 1)
        i = next(i for i, v in enumerate(bad) if v > LIMIT)
        assert "stage %d " % i in msg and "max_out_len %d," % bad[i] in msg, msg
    else:
        assert "MaxInLen %d" % (m + 1) in msg, msg


# The wrapped values the int chain produced (the reference computes it in int too) are refused now.
@pytest.mark.parametrize("src,dst,m,ext", [(44100.0, 2822400.0, 2 ** 25, 1), (44100.0, 2822400.0, 2 ** 26, 1),
                                           (44100.0, 96000.0, 10 ** 9, 0), (8000.0, 48000.0, 4 * 10 ** 8, 0)])
def test_overflowing_chains_are_refused(pkg, src, dst, m, ext):
    with pytest.raises(pkg.R8bGpuError, match="above R8BGPU_MAX_LEN"):
        pkg.Plan(src, dst, m, 2.0, A24, extfft=ext)


def test_overflowing_max_in_len_is_refused(pkg):
    with pytest.raises(pkg.R8bGpuError, match="MaxInLen 2147483647 is above R8BGPU_MAX_LEN"):
        pkg.Plan(96000.0, 44100.0, 2 ** 31 - 1, 2.0, A24)
    with pytest.raises(pkg.R8bGpuError, match="MaxInLen 2147483647 is above R8BGPU_MAX_LEN"):
        pkg.Plan.single_stage(4, [A24, 0, 0], 2 ** 31 - 1)


# ---- closed-form counts ----------------------------------------------------------------------------------------------------

def emitted(st, n):
    """Samples stage st has emitted after n inputs (r8b_plan.cpp blockconv_emitted .. hbdown_emitted, DESIGN.md section 1)."""
    k = st["name"]
    if k == "blockconv":
        avail = st["up"] * n - st["latency"]
        return 0 if avail <= 0 else -((-avail) // st["down"])
    if k == "frac_whole":
        pmax = n - 1 - st["kernel_len"] // 2
        if pmax < 0:
            return 0
        a, b = st["in_step"], st["out_step"]
        return (pmax * b + b - 1) // a + 1
    if k == "hbup":
        c = n - st["kernel_len"]
        return 2 * c if c > 0 else 0
    assert k == "hbdown"
    c = n // 2 - (st["kernel_len"] - 1)
    return c if c > 0 else 0


def chain_total(stages, n):
    for st in stages:
        n = emitted(st, n)
    return n


INTEGER_BOUNDARY = [s for s in BOUNDARY if s[0] != "trim" and s[1:3] != (48000.0, 47999.0)]


@pytest.mark.parametrize("spec", INTEGER_BOUNDARY, ids=_boundary_ids)
def test_counts_at_the_boundary(pkg, spec):
    stages, chain = _chain_of(pkg, spec)
    m = largest_max_in(chain)
    p = _plan(pkg, spec, m)
    counts = p.simulate([m] * 3)
    assert min(counts) >= 0 and max(counts) <= p.max_out_len
    assert [sum(counts[:k + 1]) for k in range(3)] == [chain_total(stages, (k + 1) * m) for k in range(3)]


# ---- past 2^32: integer chains call by call ----------------------------------------------------------------------------

L20 = 2 ** 20
N_CALLS = 4099  # 2^32 + 3 * 2^20 input samples
# The scheduler's cost per call is a few closed forms (and one binary search for an order-2 interpolator): 4099 calls take
# 2-5 ms on a desktop CPU core.  The bound leaves 10x room for slow or loaded machines; a loop over the samples (minutes),
# or a per-call cost ten times today's, exceeds it.
SIM_BOUND_S = 0.05


def _timed_simulate(p, lens):
    """(counts, the best of three wall times of Plan.simulate(lens))."""
    best = float("inf")
    for _ in range(3):
        t = time.perf_counter()
        counts = p.simulate(lens)
        best = min(best, time.perf_counter() - t)
    return counts, best

WHOLE_CHAINS = [(44100.0, 96000.0, 0), (48000.0, 44100.0, 0), (96000.0, 44100.0, 0), (192000.0, 44100.0, 0),
                (2822400.0, 44100.0, 0), (44100.0, 2822400.0, 1), (48000.0, 16000.0, 0)]


@pytest.mark.parametrize("src,dst,ext", WHOLE_CHAINS)
def test_integer_chain_counts_past_2_32(pkg, src, dst, ext):
    p = pkg.Plan(src, dst, L20, 2.0, A24, extfft=ext)
    stages = p.stages()
    assert "frac_poly" not in [s["name"] for s in stages]
    counts, dt = _timed_simulate(p, [L20] * N_CALLS)
    assert dt < SIM_BOUND_S, dt
    totals = [chain_total(stages, k * L20) for k in range(N_CALLS + 1)]
    want = [totals[k + 1] - totals[k] for k in range(N_CALLS)]
    assert counts == want
    assert sum(counts) == totals[-1]
    assert totals[-1] > 2 ** 31 * min(1.0, dst / src)  # the outputs run past 2^31 too


# ---- past 2^32: the order-2 interpolator ---------------------------------------------------------------------------------

def restate_calls(plan, src, dst, lens, factors):
    """test_trim_cpu.restate with one binary search per call instead of a loop over the outputs: the read position of the
    k-th output after the call starts, p + int(((InCounter + k) + InPosShift) * ssr / dsr) - InPosInt, never decreases in
    k, so the call's count is one past the largest k with position <= n1 - 1 - fl2.  Returns (counts, p, fpos) after each
    call."""
    st = plan.stages()
    assert [s["name"] for s in st] == ["blockconv", "frac_poly"] and st[0]["down"] == 1
    up, lat = st[0]["up"], st[0]["latency"]
    fl2 = st[1]["kernel_len"] // 2
    ssr = up * src
    ic, ipi, ips, fpos, p = 0, 0, 0.0, 0.0, 0
    dsr = dst
    n_in = 0
    counts, ps, fs = [], [], []

    def at(k):
        npos = (float(ic + k) + ips) * ssr / dsr
        ni = int(npos)
        return p + (ni - ipi), ni, npos - ni

    for l, f in zip(lens, factors):
        d = dst * f
        if d != dsr:
            dsr = d
            ips = fpos * dsr / ssr
            ic, ipi = 0, 0
        n_in += int(l)
        pmax = max(0, up * n_in - lat) - 1 - fl2
        cnt = 0
        if p <= pmax:
            lo, hi = 0, int((pmax - p + 2) * dsr / ssr) + 4
            while at(hi)[0] <= pmax:
                hi *= 2
            while hi - lo > 1:
                mid = (lo + hi) // 2
                if at(mid)[0] <= pmax:
                    lo = mid
                else:
                    hi = mid
            cnt = lo + 1
            p, ipi, fpos = at(cnt)
            ic += cnt
        if ic > 1000:
            ic, ipi = 0, 0
            ips = fpos * dsr / ssr
        counts.append(cnt)
        ps.append(p)
        fs.append(fpos)
    return counts, ps, fs


def test_binary_search_restatement_equals_the_per_output_one(pkg):
    tp = pkg.Plan.trim(44100.0, 48000.0, 4096, 2.0, A24, 0.01)
    import numpy as np
    rng = np.random.default_rng(3)
    lens = rng.integers(0, 4097, 200)
    fs = test_trim_cpu.random_walk(rng, 200)
    assert restate_calls(tp, 44100.0, 48000.0, lens, fs) == test_trim_cpu.restate(tp, 44100.0, 48000.0, lens, fs)


def test_order2_counts_past_2_32(pkg):
    p = pkg.Plan(48000.0, 47999.0, L20, 2.0, A24)
    lens = [L20] * N_CALLS
    counts, dt = _timed_simulate(p, lens)
    assert dt < SIM_BOUND_S, dt
    c2, _, _ = restate_calls(p, 48000.0, 47999.0, lens, [1.0] * N_CALLS)
    assert counts == c2
    assert sum(counts) > 2 ** 32 - 2 ** 20


def test_trim_counts_and_timing_past_2_32(pkg):
    import numpy as np
    tp = pkg.Plan.trim(44100.0, 48000.0, L20, 2.0, A24, 0.01)
    rng = np.random.default_rng(7)
    lens = np.full(N_CALLS, L20, np.int32)
    short = rng.random(N_CALLS) < 0.05
    lens[short] = rng.integers(0, L20, int(short.sum()))
    fs = test_trim_cpu.random_walk(rng, N_CALLS)  # a new factor (a re-base) nearly every call
    counts, pos, frac = tp.simulate_trim(lens, fs, timing=True)
    c2, p2, f2 = restate_calls(tp, 44100.0, 48000.0, lens, fs)
    assert list(counts) == c2
    assert list(pos) == p2
    assert frac.tobytes() == np.array(f2).tobytes()
    assert int(lens.astype(np.int64).sum()) > 2 ** 32 - 2 ** 29 and pos[-1] > 2 ** 32
