"""GPU: the half-band cascades over the plans of CASCADES and every tap vector of the walk (tests/test_hb_geometry_cpu.py)
-- against the reference, with the kernel and tile plan pinned to the report, and bit for bit against one kernel per
stage.

k_hbup and k_hbdown sum each output in the cascade's order (DESIGN K3/K4), and the fused last-two pass equals two plain
stages bit for bit (tests/cpp/hbfuse_check.cpp).  So the cascade, any tile width, the unfused last stage and the
scalar stores must all give the bytes of R8BGPU_NO_HB_CASCADE, and DSD bytes those of the fp64 batch fed the same
+-scale values.  A halo one sample short corrupts only tile edges of some tap vectors: every vector is run.

The reference's 1-tap half-band upsampler (49 dB, steepness family 3 and up) reads one ring slot it never wrote for
the odd output at its stream start: CDSPHBUpsampler::clear() leaves ReadPos at BufLen when the stage consumes its
latency, and the "beyond bounds" copy mirrors only flo = 2T - 1 = 1 sample, so rp[1] of the first output pair is
Buf[BufLen + 1] instead of the second input sample.  This engine computes the defined stream there.  The reference
comparisons skip the final outputs that sample reaches (ref_skip); the bit-for-bit tests still hold them to one kernel per stage."""

import numpy as np
import pytest

import oracle_util as ou
from test_hb_geometry_cpu import CASCADES, SHAPES, chain_rates, make_plan, max_in, runs, walk

pytestmark = pytest.mark.gpu

N_CH = 3
DSD_LSB = 16


def expected_kernels(plan, rs):
    """Batch.stage_kernels() a lock-step batch of the plan shows for its half-band stages, from the reports."""
    out = {}
    for i, info in rs:
        c = info["n_stages"]
        name = plan.stages()[i]["name"]
        out[i] = ("k_%s_cascade" % name if c >= 2 else "k_%s" % name, c)
        for k in range(1, c):
            out[i + k] = ("(fused)", 0)
    return out


def expected_variant(info, dsd=False):
    taps = "/".join(map(str, info["ntaps"]))
    if info["kind"] == "up-cascade":
        return "k_hbup_cascade stages=%d taps=%s last2=%d w=%d" % (info["n_stages"], taps, info["fuse_last2"], info["w"])
    return "k_hbdown_cascade%s stages=%d taps=%s w=%d" % ("<DSD>" if dsd else "", info["n_stages"], taps, info["w"])


def check_kernels(b, plan, rs, dsd=False):
    ks = b.stage_kernels()
    for i, k in expected_kernels(plan, rs).items():
        assert ks[i] == k, (i, ks, k)
    for i, info in rs:
        if info["n_stages"] >= 2:
            assert b.last_variant(i) == expected_variant(info, dsd), (b.last_variant(i), info)
    return ks


# ---- call lengths: the cascade's first output e0 at each residue ------------------------------------------------------

def cascade_e(plan, info, lens):
    """Output index e of the cascade's last stage after each prefix of lens, from the emitted-count rules of the plan's
    stages: hbdown n -> max(0, n / 2 - T + 1), hbup n -> max(0, 2 (n - T)), BlockConvolver n -> max(0, up n - latency);
    behind the interpolator the cascade is the chain's end and e counts the outputs."""
    st = plan.stages()
    first, c = info["first"], info["n_stages"]
    if st[first - 1]["name"] == "blockconv" and first == 1:
        bc = st[0]
        e0 = [max(0, bc["up"] * int(n) - bc["latency"]) for n in np.cumsum([0] + list(lens))]
    elif first == 0:
        e0 = [int(n) for n in np.cumsum([0] + list(lens))]
    else:
        assert first + c == len(st)
        return [int(t) for t in np.cumsum([0] + plan.simulate(lens))]
    out = []
    for e in e0:
        for s in st[first:first + c]:
            e = max(0, e // 2 - (s["kernel_len"] - 1)) if s["name"] == "hbdown" else max(0, 2 * (e - s["kernel_len"]))
        out.append(e)
    return out


def residues(plan, info, lens):
    """Which of: e0 = 0 mod 2^c, e0 != 0 mod 2^c, e0 != 0 mod 8, fewer than 8 outputs -- the calls that run the cascade
    reach."""
    c = info["n_stages"]
    e = cascade_e(plan, info, lens)
    hit = set()
    for j in range(len(lens)):
        if e[j + 1] <= e[j]:
            continue
        hit.add("0 mod 2^c" if e[j] % (1 << c) == 0 else "!0 mod 2^c")
        if e[j] % 8:
            hit.add("!0 mod 8")
        if e[j + 1] - e[j] < 8:
            hit.add("under 8")
    return hit


def reachable(plan, info):
    """An up cascade's output is e = 2^c e_in - K, K = sum_k 2^(c-k) T_k, once it runs: e0 mod 2^c is 0 (the first call)
    or -K, and e_in behind a 2x BlockConvolver (2 n - latency) keeps the latency's parity.  A down cascade's calls can
    start anywhere and be as short as one output."""
    c = info["n_stages"]
    if info["kind"] == "down-cascade":
        return {"0 mod 2^c", "!0 mod 2^c", "!0 mod 8", "under 8"}
    st = plan.stages()
    k = sum(t << (c - j) for j, t in enumerate(info["ntaps"]))
    xs = range(8)
    if info["first"] == 1 and st[0]["up"] == 2:
        xs = [x for x in xs if x % 2 == st[0]["latency"] % 2]
    out = {"0 mod 2^c"}
    for x in xs:
        r = (x << c) - k
        if r % (1 << c):
            out.add("!0 mod 2^c")
        if r % 8:
            out.add("!0 mod 8")
    return out


def call_lens(plan, info):
    """Full, empty, 1-sample, short and max - 1 blocks, extended until the cascade's calls start at every residue class
    they can reach."""
    m = plan.max_in_len
    lens = [m, 0, 1, 7, m, 333, m - 1, m]
    want = reachable(plan, info)
    step = 1 << info["n_stages"] if info["kind"] == "down-cascade" else 1
    for _ in range(12):
        missing = want - residues(plan, info, lens)
        if not missing:
            break
        for l in range(1, 64 * step):
            trial = lens + [l, m] if "under 8" not in missing else lens + [m, l]
            if missing & residues(plan, info, trial):
                lens = trial
                break
    assert want <= residues(plan, info, lens), (residues(plan, info, lens), want)
    return lens


def ref_skip(plan):
    """Final outputs at the stream start that depend on the reference's unwritten ring slot of a 1-tap upsampler: its
    output 1, widened by 2x per later stage and rounded up to whole items of 8."""
    st = [s for s in plan.stages() if s["name"] == "hbup"]
    one = [k for k, s in enumerate(st) if s["kernel_len"] == 1]
    return 8 << (len(st) - 1 - one[0]) if one else 0


def cascade_of(plan):
    rs = runs(plan)[0]
    return rs, next((info for _, info in rs if info["n_stages"] >= 2), rs[0][1])


# ---- against the reference ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(CASCADES))
def test_reference_parity_and_tile_plan(pkg, ref, name):
    src, dst, m, at = CASCADES[name]
    plan = make_plan(pkg, name)
    rs, info = cascade_of(plan)
    lens = call_lens(plan, info) if info["n_stages"] >= 2 else [m, 0, 1, 7, m, 333, m - 1, m]
    b = pkg.Batch(plan, N_CH, 0)
    refs = [ref.Resampler(src, dst, m, 2.0, at) for _ in range(N_CH)]
    rng = np.random.default_rng(31)
    got, exp = [[] for _ in range(N_CH)], [[] for _ in range(N_CH)]
    for call, l in enumerate(lens):
        x = rng.uniform(-1.0, 1.0, size=(N_CH, l))
        y = b.process_host(x)
        for c in range(N_CH):
            r = refs[c].process(x[c])
            assert len(r) == y.shape[1], (call, l, len(r), y.shape[1])
            got[c].append(y[c])
            exp[c].append(r)
    check_kernels(b, plan, rs)
    k = ref_skip(plan)
    assert sum(len(g) for g in got[0]) > k
    for c in range(N_CH):
        mx, rms = ou.parity_metrics(np.concatenate(got[c])[k:], np.concatenate(exp[c])[k:])
        assert mx <= 32 * ou.EPS and rms <= 4 * ou.EPS, (c, mx / ou.EPS, rms / ou.EPS)


@pytest.mark.parametrize("name", list(CASCADES))
def test_ragged_after_lockstep(pkg, ref, name):
    """Lock-step calls, then ragged calls of other lengths per channel: the rings the cascade kept in shared memory are
    refilled from the source; each channel equals its own reference object."""
    src, dst, m, at = CASCADES[name]
    plan = make_plan(pkg, name)
    b = pkg.Batch(plan, N_CH, 0)
    refs = [ref.Resampler(src, dst, m, 2.0, at) for _ in range(N_CH)]
    rng = np.random.default_rng(47)
    got, exp = [[] for _ in range(N_CH)], [[] for _ in range(N_CH)]
    for l in (m, 333, m):
        x = rng.uniform(-1.0, 1.0, size=(N_CH, l))
        y = b.process_host(x)
        for c in range(N_CH):
            got[c].append(y[c])
            exp[c].append(refs[c].process(x[c]))
    for ls in ((m, 17, 0), (1, m, m // 2 + 3), (m - 1, 7, m), (m, m, 1)):
        xs = [rng.uniform(-1.0, 1.0, size=l) for l in ls]
        ys = b.process_ragged(xs)
        for c in range(N_CH):
            r = refs[c].process(xs[c])
            assert len(r) == len(ys[c]), (ls, c, len(r), len(ys[c]))
            got[c].append(ys[c])
            exp[c].append(r)
    k = ref_skip(plan)
    for c in range(N_CH):
        a, e = np.concatenate(got[c])[k:], np.concatenate(exp[c])[k:]
        assert len(a) > 0
        mx, rms = ou.parity_metrics(a, e)
        assert mx <= 32 * ou.EPS and rms <= 4 * ou.EPS, (c, mx / ou.EPS, rms / ou.EPS)


# ---- bit for bit over every walked tap vector ---------------------------------------------------------------------------

def _run(pkg, plan, xs, monkeypatch, env=None, odd_stride=False, dsd_bits=None, scale=0.5):
    """A fresh lock-step batch under env fed xs; returns (outputs per call, stage_kernels()).  odd_stride: device buffers
    whose rows are an odd number of doubles apart.  dsd_bits: feed these bits as DSD bytes (xs is then their values)."""
    import torch
    with monkeypatch.context() as mp:
        for k, v in (env or {}).items():
            mp.setenv(k, v)
        b = pkg.Batch(plan, N_CH, 0)
        rs = runs(plan)[0]
        ys = []
        cap = max(plan.max_out_len, 1)
        for j, x in enumerate(xs):
            if dsd_bits is not None:
                byt = np.packbits(dsd_bits[j].astype(np.uint8), axis=-1, bitorder="little")
                ys.append(b.process_host_fmt(byt, fmt=DSD_LSB, in_scale=scale))
            elif odd_stride and x.shape[1]:
                out = torch.zeros((N_CH, cap | 1), dtype=torch.float64, device="cuda")
                ys.append(b.process(torch.from_numpy(x).cuda(), out=out).cpu().numpy())
            else:
                ys.append(b.process_host(x))
        ks = check_kernels(b, plan, rs, dsd=dsd_bits is not None) if env is None else b.stage_kernels()
        return ys, ks


def _same(got, want, what):
    for call, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape, (what, call, g.shape, w.shape)
        if g.tobytes() != w.tobytes():
            c, j = [int(v[0]) for v in np.nonzero(g.view(np.int64) != w.view(np.int64))]
            pytest.fail("%s, call %d: channel %d first differs at output %d: %r vs %r" % (what, call, c, j, g[c, j], w[c, j]))


def _outside(ks, plan):
    return [k for i, k in enumerate(ks) if plan.stages()[i]["name"] not in ("hbup", "hbdown")]


@pytest.mark.parametrize("direction,third,c", SHAPES, ids=["%s-%s-%d" % (d, "third" if t else "plain", c) for d, t, c in SHAPES])
def test_bit_exact_against_one_kernel_per_stage(pkg, direction, third, c, monkeypatch):
    src, dst = chain_rates(direction, third, c)
    m = max_in(direction, c)
    vectors = walk(pkg, src, dst, m)
    rng = np.random.default_rng(7 * c + third)
    lens = [m, 8, 0, 16, m - 8, 336, m]            # multiples of 8: the same calls as DSD bytes
    checked = {"no-cascade": 0, "no-last2": 0, "budget": 0, "odd-stride": 0, "dsd": 0}
    for taps, (a, plan) in vectors.items():
        rs = runs(plan)[0]
        bits = [rng.integers(0, 2, size=(N_CH, l)) for l in lens]
        xs = [np.where(bt != 0, 0.5, -0.5) for bt in bits]
        want, ks = _run(pkg, plan, xs, monkeypatch)
        casc = [info for _, info in rs if info["n_stages"] >= 2]
        variants = [("no-cascade", {"R8BGPU_NO_HB_CASCADE": "1"})]
        if any(info["fuse_last2"] for info in casc):
            variants.append(("no-last2", {"R8BGPU_HB_NO_LAST2": "1"}))
        key = "R8BGPU_HB_SMEM_DOUBLES" if direction == "up" else "R8BGPU_HBD_SMEM_DOUBLES"
        for budget in ("3500", "3200", "12800", "25000"):     # the first that moves w and nothing else
            with monkeypatch.context() as mp:
                mp.setenv(key, budget)
                other = [info for _, info in runs(plan)[0] if info["n_stages"] >= 2]
            if ([i["n_stages"] for i in other] == [i["n_stages"] for i in casc] and
                    [i["w"] for i in other] != [i["w"] for i in casc]):
                variants.append(("budget", {key: budget}))
                break
        for what, env in variants:
            got, gks = _run(pkg, plan, xs, monkeypatch, env)
            assert _outside(gks, plan) == _outside(ks, plan), (what, gks, ks)
            if what == "no-cascade":
                assert all(k[1] == 1 for i, k in enumerate(gks) if plan.stages()[i]["name"] in ("hbup", "hbdown")), gks
            else:
                assert gks == ks, (what, gks, ks)
            _same(got, want, "%s %s" % (taps, what))
            checked[what] += 1
        if direction == "up" and not casc[0]["writes_ring"]:
            got, _ = _run(pkg, plan, xs, monkeypatch, odd_stride=True)
            _same(got, want, "%s odd stride" % (taps,))
            checked["odd-stride"] += 1
        if direction == "down":
            got, _ = _run(pkg, plan, xs, monkeypatch, dsd_bits=bits)
            _same(got, want, "%s DSD" % (taps,))
            checked["dsd"] += 1
    print("\n%s %s %d: %d tap vectors, %s" % (direction, "third" if third else "plain", c, len(vectors), checked))
    assert checked["no-cascade"] == len(vectors) and checked["budget"] > 0
    assert checked["dsd" if direction == "down" else "odd-stride"] > 0 or c == 7

