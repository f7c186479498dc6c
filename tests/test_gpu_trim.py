"""GPU: per-channel rate trim (trim plans, Batch.set_trim) -- drift-compensating resampling on the order-2 interpolator.

Yardsticks:
  - a constant factor f from clear is the reference at (src, fl(dst * f)), channel by channel (counts equal, max|d| <=
    32 eps and rms <= 4 eps of the signal); each channel has its own factor, so every call is ragged;
  - factors of exactly 1 are an ordinary batch, bit for bit;
  - factors that change every call match an oracle built from the reference's own BlockConvolver stage and bank,
    followed by a long-double restatement of convolve2 (CDSPFracInterpolator.h:1069-1179) at the restated timing;
  - an ordinary part of a mixed batch is unaffected by a trim part next to it, bit for bit."""
import numpy as np
import pytest

import oracle_util as ou
from test_trim_cpu import A16, A24, UP_CHAINS, random_walk, restate

pytestmark = pytest.mark.gpu


def parity(y, yr):
    assert len(y) == len(yr)
    if len(yr) == 0:
        return
    mx, rms = ou.parity_metrics(y, yr)
    assert mx <= 32 * ou.EPS and rms <= 4 * ou.EPS, (mx / ou.EPS, rms / ou.EPS)


def blocks(rng, n_calls, n_ch, M):
    lens = rng.integers(0, M + 1, size=(n_calls, n_ch))
    lens[rng.random((n_calls, n_ch)) < 0.1] = 0
    return lens


# ---- 1. constant factor per channel against the reference at (src, fl(dst * f)) ---------------------------------------

# 8000 -> 176400 at TransBand 40: 2x BlockConvolver, interpolator, 2x BlockConvolver (transition band capped at 45 for
# every factor in +-1 %), half-band upsampler
HB_CHAIN = (8000.0, 176400.0, 40.0)


@pytest.mark.parametrize("src,dst,tb,atten", [c + (A24,) for c in UP_CHAINS] + [UP_CHAINS[0] + (A16,), HB_CHAIN + (A24,)])
def test_constant_factors_match_the_reference(pkg, ref, src, dst, tb, atten):
    M, n_ch, n_calls = 4096, 6, 12
    tp = pkg.Plan.trim(src, dst, M, tb, atten, 0.01)
    names = [s["name"] for s in tp.stages()]
    if (src, dst) == HB_CHAIN[:2]:
        assert names == ["blockconv", "frac_poly", "blockconv", "hbup"]
    rng = np.random.default_rng(int(src + dst))
    fs = rng.uniform(0.99, 1.01, n_ch)  # (at f = 1 exactly these pairs step whole rows: the reference's bank differs)
    for f in fs:  # the ordinary planner at fl(dst * f) builds the same chain
        assert [s["name"] for s in pkg.Plan(src, dst * f, M, tb, atten).stages()] == names
    b = pkg.Batch(tp, n_ch, 0)
    b.set_trim(np.arange(n_ch), fs)
    assert np.array_equal(b.trim(), fs)
    refs = [ref.Resampler(src, dst * f, M, tb, atten) for f in fs]
    x = ou.white_noise(n_ch, M * n_calls, seed=3)
    pos = np.zeros(n_ch, dtype=np.int64)
    got = [[] for _ in range(n_ch)]
    want = [[] for _ in range(n_ch)]
    for lens in blocks(rng, n_calls, n_ch, M):
        xs = [x[c, pos[c]:pos[c] + lens[c]] for c in range(n_ch)]
        ys = b.process_ragged(xs)
        for c in range(n_ch):
            got[c].append(ys[c])
            want[c].append(refs[c].process(xs[c]))
            assert len(ys[c]) == len(want[c][-1])
        pos += lens
    for c in range(n_ch):
        parity(np.concatenate(got[c]), np.concatenate(want[c]))


def test_power_of_two_ratio_has_no_interpolator(pkg):
    with pytest.raises(pkg.R8bGpuError, match="no fractional interpolator"):
        pkg.Plan.trim(44100.0, 352800.0, 1024, 2.0, A24, 1e-3)


# ---- 2. factors of 1: an ordinary batch, bit for bit -------------------------------------------------------------------

@pytest.mark.parametrize("dst", [47999.0, 48001.0, 47990.0])
def test_unit_factors_are_an_ordinary_batch(pkg, dst):
    M, n_ch = 4096, 5
    op = pkg.Plan(48000.0, dst, M, 2.0, A24)
    tp = pkg.Plan.trim(48000.0, dst, M, 2.0, A24, 1e-3)
    bo, bt = pkg.Batch(op, n_ch, 0), pkg.Batch(tp, n_ch, 0)
    bt.set_trim(np.arange(n_ch), np.ones(n_ch))  # the same factor again: nothing happens
    assert bt.channel_groups == 1
    x = ou.white_noise(n_ch, 40 * M, seed=7)
    rng = np.random.default_rng(11)
    off = 0
    for l in rng.integers(0, M + 1, 6):  # lock-step calls (the fused order-2 path)
        yo, yt = bo.process_host(x[:, off:off + l]), bt.process_host(x[:, off:off + l])
        assert yo.tobytes() == yt.tobytes()
        off += l
    pos = np.full(n_ch, off)
    for lens in blocks(rng, 8, n_ch, M):  # ragged calls
        xs = [x[c, pos[c]:pos[c] + lens[c]] for c in range(n_ch)]
        for a, t in zip(bo.process_ragged(xs), bt.process_ragged(xs)):
            assert a.tobytes() == t.tobytes()
        pos += lens


# ---- 3. factors that change every call: the stage-built oracle ---------------------------------------------------------

def oracle_outputs(ref, plan, src, dst, tb, atten, x_all, lens, factors):
    """Reference BlockConvolver stage over the whole input, then convolve2 in long double at the restated timing."""
    st = plan.stages()
    up = st[0]["up"]
    nf = 0.5 if dst > src else (0.5 * dst / src if up == 2 else dst / src)
    bc = ref.stage_blockconv(nf, tb, atten, 2.0 if up == 2 else 1.0, up, 1)
    z = np.concatenate([bc.process(x_all[i:i + 4096]) for i in range(0, len(x_all), 4096)])
    flen = st[1]["kernel_len"]
    bank = ref.fracbank(-1, 3, 8, atten)
    tab = bank["table"].astype(np.longdouble)
    assert tab.shape[1] == flen
    outs = []
    counts, _, _ = restate(plan, src, dst, lens, factors, outs)
    P = np.array([p for p, _ in outs], dtype=np.int64)
    F = np.array([f for _, f in outs], dtype=np.float64)
    xf = F * bank["fracs"]
    fti = xf.astype(np.int64)
    xr = (xf - fti).astype(np.longdouble)
    fll = flen // 2 - 1
    zp = np.concatenate([np.zeros(flen), z, np.zeros(flen)]).astype(np.longdouble)
    y = np.empty(len(P), dtype=np.longdouble)
    for a in range(0, len(P), 8192):
        s = slice(a, a + 8192)
        rows = tab[fti[s]]
        coef = rows[..., 0] + rows[..., 1] * xr[s, None] + rows[..., 2] * (xr[s, None] * xr[s, None])
        idx = (P[s, None] - fll + np.arange(flen)[None, :]) + flen
        y[s] = np.sum(coef * zp[idx], axis=1)
    return counts, y.astype(np.float64)


@pytest.mark.parametrize("src,dst", [(44100.0, 48000.0), (48000.0, 44100.0), (96000.0, 44100.0)])
def test_piecewise_factors_match_the_stage_oracle(pkg, ref, src, dst):
    M, n_ch, n_calls, tb = 2048, 4, 60, 2.0
    tp = pkg.Plan.trim(src, dst, M, tb, A24, 2e-4)
    rng = np.random.default_rng(int(dst))
    lens = blocks(rng, n_calls, n_ch, M)
    fs = np.stack([random_walk(rng, n_calls) for _ in range(n_ch)], axis=1)
    x = ou.white_noise(n_ch, int(lens.sum(axis=0).max()) + 1, seed=9)
    b = pkg.Batch(tp, n_ch, 0)
    pos = np.zeros(n_ch, dtype=np.int64)
    got = [[] for _ in range(n_ch)]
    for i in range(n_calls):
        b.set_trim(np.arange(n_ch), fs[i])
        xs = [x[c, pos[c]:pos[c] + lens[i, c]] for c in range(n_ch)]
        for c, y in enumerate(b.process_ragged(xs)):
            got[c].append(y)
        pos += lens[i]
    for c in range(n_ch):
        counts, y = oracle_outputs(ref, tp, src, dst, tb, A24, x[c, :pos[c]], lens[:, c], fs[:, c])
        assert [len(g) for g in got[c]] == counts
        parity(np.concatenate(got[c]), y)


# ---- 4. channels regroup once their factors and calls agree ------------------------------------------------------------

def test_channels_regroup(pkg):
    M, n_ch = 2048, 8
    tp = pkg.Plan.trim(44100.0, 48000.0, M, 2.0, A24, 1e-3)
    b = pkg.Batch(tp, n_ch, 0)
    x = ou.white_noise(n_ch, 4 * M, seed=1)
    b.set_trim(np.arange(n_ch), 1.0 + 1e-5 * np.arange(n_ch))
    assert b.channel_groups == n_ch
    b.process_ragged(list(x[:, :M]))  # equal lengths, different factors: every channel its own group
    assert b.channel_groups == n_ch
    b.set_trim(np.arange(n_ch), np.full(n_ch, 1.0 + 3e-4))
    assert b.channel_groups == n_ch  # one factor again, but histories differ
    b.clear()
    assert b.channel_groups == 1 and np.all(b.trim() == 1.0 + 3e-4)  # factors survive clear()
    y1 = b.process_host(x[:, :M])  # one factor, one state: lock-step again
    b.clear_channels([3])
    assert b.channel_groups == 2
    b.set_trim([3], [1.0 + 3e-4])  # no change: no re-base
    assert b.channel_groups == 2
    with pytest.raises(pkg.R8bGpuError, match="named twice"):
        b.set_trim([1, 1], [1.0, 1.0])
    with pytest.raises(pkg.R8bGpuError, match="outside"):
        b.set_trim([0, 1], [1.0, 1.002])
    assert np.all(b.trim() == 1.0 + 3e-4)  # the refused calls changed nothing
    ob = pkg.Batch(pkg.Plan(44100.0, 48000.0, M, 2.0, A24), 2, 0)
    with pytest.raises(pkg.R8bGpuError, match="not a trim plan"):
        ob.set_trim([0], [1.0])
    assert y1.shape[0] == n_ch


# ---- 5. mixed batch: a trim part next to an ordinary part --------------------------------------------------------------

def test_mixed_trim_part_leaves_the_ordinary_part_alone(pkg):
    M = 4096
    po = np.array([0, 1, 0, 1, 1, 0], dtype=np.int32)
    ordinary = pkg.Plan(48000.0, 44100.0, M, 2.0, A24)
    trim = pkg.Plan.trim(44100.0, 48000.0, M, 2.0, A24, 2e-4)
    mb = pkg.Batch.mixed([ordinary, trim], po, 0)
    alone = pkg.Batch.mixed([ordinary], np.zeros(3, np.int32), 0)
    tw = pkg.Batch(trim, 3, 0)
    with pytest.raises(pkg.R8bGpuError, match="not a trim plan"):
        mb.set_trim([0], [1.0])
    rng = np.random.default_rng(2)
    x = ou.white_noise(6, 30 * M, seed=4)
    pos = np.zeros(6, dtype=np.int64)
    oc, tc = np.nonzero(po == 0)[0], np.nonzero(po == 1)[0]
    for i in range(10):
        f = 1.0 + rng.uniform(-2e-4, 2e-4, 3)
        mb.set_trim(tc, f)
        tw.set_trim(np.arange(3), f)
        lens = blocks(rng, 1, 6, M)[0]
        xs = [x[c, pos[c]:pos[c] + lens[c]] for c in range(6)]
        ys = mb.process_ragged(xs)
        ya = alone.process_ragged([xs[c] for c in oc])
        yt = tw.process_ragged([xs[c] for c in tc])
        for k, c in enumerate(oc):
            assert ys[c].tobytes() == ya[k].tobytes()
        for k, c in enumerate(tc):
            assert ys[c].tobytes() == yt[k].tobytes()
        pos += lens
    got = mb.trim()
    assert np.all(got[oc] == 1.0) and np.array_equal(got[tc], f)


# ---- 6. typed ragged buffers and an explicit-target flush on a drifting batch ------------------------------------------

def test_typed_buffers_and_flush_while_drifting(pkg):
    M, n_ch = 2048, 4
    tp = pkg.Plan.trim(44100.0, 48000.0, M, 2.0, A24, 2e-4)
    a, b = pkg.Batch(tp, n_ch, 0), pkg.Batch(tp, n_ch, 0)  # a: typed int16 buffers, b: fp64 twin
    rng = np.random.default_rng(8)
    xi = (rng.uniform(-1, 1, (n_ch, M)) * 32000).astype(np.int16)
    for i in range(12):
        f = random_walk(rng, n_ch)
        a.set_trim(np.arange(n_ch), f)
        b.set_trim(np.arange(n_ch), f)
        lens = blocks(rng, 1, n_ch, M)[0]
        ya, ca = a.process_ragged_fmt(xi, lens, out_dtype=np.float64)
        yb = b.process_ragged([xi[c, :lens[c]].astype(np.float64) for c in range(n_ch)])
        for c in range(n_ch):
            assert ya[c, :ca[c]].tobytes() == yb[c].tobytes()
    with pytest.raises(pkg.R8bGpuError, match="explicit"):
        a.flush([0, 1])
    _, n_out = a.channel_totals()
    tg = n_out[[0, 2]] + np.array([5000, 7])
    ya, ca = a.flush([0, 2], targets=tg)
    yb, cb = b.flush([0, 2], targets=tg)
    assert list(ca) == list(cb) and ca[0] == 5000 and ca[2] == 7 and ca[1] == 0
    assert ya.tobytes() == yb.tobytes()
    assert np.all(a.trim() == b.trim())  # factors survive the flush's clear
