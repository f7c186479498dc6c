"""GPU: the unfused BlockConvolvers (k_blockconv, the large-tile trio) and the stand-alone interpolators (k_frac) over the
plans of BLOCKCONVS (tests/test_blockconv_geometry_cpu.py) -- against the reference with the kernel and its call
fields pinned to the report, and bit for bit across the variants that must not change a result.

Each k_frac output depends only on its global output index (frac_position), so every admissible R8BGPU_FRAC_TILE gives
the bytes of the default tile.  A k_blockconv tile pair and a k_bcl unit read only their own channel's records, so ragged
calls of equal lengths, one channel per large-tile group, and a batch wider than one wave give the bytes of the
lock-step call, one group and a 5-channel twin."""

import zlib

import numpy as np
import pytest

import oracle_util as ou
from test_blockconv_geometry_cpu import BLOCKCONVS, FRAC_CAP, make_plan, settings_of

pytestmark = pytest.mark.gpu

N_CH = 3


def _env(mp, name, extra=None):
    for k, v in dict(settings_of(name), **(extra or {})).items():
        mp.setenv(k, v)


def unfused(plan, n_ch=N_CH):
    """{stage: report} of the stages a lock-step call runs on k_blockconv, k_bcl or k_frac."""
    out = {}
    for i, s in enumerate(plan.stages()):
        if s["name"] == "blockconv":
            info = plan.blockconv_info(i, n_ch)
            if info["kernel"] in ("k_blockconv", "k_bcl"):
                out[i] = info
        elif s["name"].startswith("frac"):
            info = plan.frac_info(i)
            if info["kernel"] != "fused":
                out[i] = info
    return out


def expected_kernel(info):
    return {"k_blockconv": "k_blockconv", "k_bcl": "k_bcl_gather+k_bcl_conv+k_bcl_scatter",
            "k_frac<false>": "k_frac<false>", "k_frac<true>": "k_frac<true>"}[info["kernel"]]


def variant_prefix(info, n_ch=N_CH):
    if info["kernel"] == "k_blockconv":
        return "k_blockconv M=%d up=%d src_up=%d down=%d trunc=%d tiles=" % (
            1 << info["fft_log2"], info["up"], info["src_up"], info["down"], info["trunc"])
    if info["kernel"] == "k_bcl":
        return "k_bcl M=%d R0=%d src_up=%d down=%d trunc=%d tiles=" % (
            1 << info["fft_log2"], info["r0"], info["src_up"], info["down"], info["trunc"])
    return "k_frac poly=%d tile=%d flen=%d" % (int(info["kernel"] == "k_frac<true>"), info["tile"], info["flen"])


def pin(b, rep, tiles, n_ch=N_CH):
    """stage_kernels() and last_variant() of every unfused stage against its report; collects k_blockconv's tile counts."""
    ks = b.stage_kernels()
    for i, info in rep.items():
        assert ks[i] == (expected_kernel(info), 1), (i, ks[i], info)
        v = b.last_variant(i)
        if v == "":
            continue            # no call has launched it yet (no outputs)
        p = variant_prefix(info, n_ch)
        assert v.startswith(p), (i, v, p)
        if info["kernel"] == "k_bcl":
            nt = int(v[len(p):].split()[0])
            groups = int(v.split("groups=")[1])
            # the report's group_ch fits the largest call; a shorter call may put more channels in a group
            assert 1 <= groups <= -(-n_ch // info["group_ch"]), (v, info)
            tiles.setdefault(i, set()).add(nt)
        elif info["kernel"] == "k_blockconv":
            tiles.setdefault(i, set()).add(int(v[len(p):]))
        else:
            assert v == p, (v, p)


def reference(ref, ref_e1, name, plan):
    """One reference object per channel: the whole resampler for chains, the stage for single stages."""
    e = BLOCKCONVS[name]
    if name.startswith("single:"):
        kind, params = e[0], e[1]
        if kind == 0:
            return [ref.stage_blockconv(*params) for _ in range(N_CH)]
        return [ref.stage_frac(params[0], params[1], params[2], bool(params[3])) for _ in range(N_CH)]
    src, dst, m, tb, at, ext, _ = e
    r = ref_e1 if ext else ref
    return [r.Resampler(src, dst, m, tb, at) for _ in range(N_CH)]


def call_lens(plan):
    """Full, empty, one-sample, short and MaxInLen - 1 blocks (the first call's first tile window starts before sample 0,
    and most calls end on a tile of fewer positions than its advance)."""
    m = plan.max_in_len
    return [m, 0, 1, 7, m, 333, m - 1, m // 2 + 5, 64, 3 * m // 4, 2, m]


def wanted_tiles(plan, i, info):
    """Tile counts a call can give: 1; an even count where the largest call spans more than one tile advance; an odd count
    above 1 (block-exact tiles are not paired up) where it spans more than two."""
    st = plan.stages()
    span = (plan.max_in_len if i == 0 else st[i - 1]["max_out_len"]) * info["src_up"]
    want = {"1"}
    if span > info["adv"] + 2:
        want.add("even")
    if info["block_exact"] and span > 2 * info["adv"] + 2:
        want.add("odd")
    return want


def tile_kinds(ts):
    return {"1" if t == 1 else "even" if t % 2 == 0 else "odd" for t in ts}


def _run_ref_calls(b, refs, lens, rng, got, exp, rep, tiles):
    for call, l in enumerate(lens):
        x = rng.uniform(-1.0, 1.0, size=(N_CH, l))
        y = b.process_host(x)
        for c in range(N_CH):
            r = refs[c].process(x[c])
            assert len(r) == y.shape[1], (call, l, len(r), y.shape[1])
            got[c].append(y[c])
            exp[c].append(r)
        pin(b, rep, tiles)


def _parity(got, exp, what=""):
    for c in range(N_CH):
        a, e = np.concatenate(got[c]), np.concatenate(exp[c])
        assert len(a) > 0
        mx, rms = ou.parity_metrics(a, e)
        assert mx <= 32 * ou.EPS and rms <= 4 * ou.EPS, (what, c, mx / ou.EPS, rms / ou.EPS)


@pytest.mark.parametrize("name", list(BLOCKCONVS))
def test_reference_parity_and_tiles(pkg, ref, ref_e1, name, monkeypatch):
    """Lock-step calls against the reference, each call's instantiation pinned; then ragged calls of other lengths per
    channel, each channel against its own reference object."""
    _env(monkeypatch, name)
    plan = make_plan(pkg, name)
    rep = unfused(plan)          # may be empty: the ragged calls still run every stage on its own kernel
    refs = reference(ref, ref_e1, name, plan)
    b = pkg.Batch(plan, N_CH, 0)
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    got, exp, tiles = [[] for _ in range(N_CH)], [[] for _ in range(N_CH)], {}
    lens = call_lens(plan)
    _run_ref_calls(b, refs, lens, rng, got, exp, rep, tiles)
    m = plan.max_in_len
    for i, info in rep.items():
        if info["kernel"] not in ("k_blockconv", "k_bcl"):
            continue
        want = wanted_tiles(plan, i, info)
        missing = want - tile_kinds(tiles.get(i, ()))
        for l in list(range(m, 0, -max(1, m // 61))):
            if not missing:
                break
            _run_ref_calls(b, refs, [l], rng, got, exp, rep, tiles)
            missing -= tile_kinds(tiles.get(i, ()))
        assert not missing, (name, i, want, tiles.get(i), info)
    _parity(got, exp, name)
    for ls in ((m, 17, 0), (1, m, m // 2 + 3), (m - 1, 7, m), (m, m, 1)):
        xs = [rng.uniform(-1.0, 1.0, size=l) for l in ls]
        ys = b.process_ragged(xs)
        for c in range(N_CH):
            r = refs[c].process(xs[c])
            assert len(r) == len(ys[c]), (ls, c, len(r), len(ys[c]))
            got[c].append(ys[c])
            exp[c].append(r)
    _parity(got, exp, name + " ragged")


def _plain_bcs(pkg, name):
    plan = make_plan(pkg, name)
    return plan, [i for i, info in unfused(plan).items() if info["kernel"] in ("k_blockconv", "k_bcl") and not info["block_exact"]]


@pytest.mark.parametrize("name", [n for n in BLOCKCONVS if not n.startswith("trim:")])
def test_every_fft_length(pkg, ref, ref_e1, name, monkeypatch):
    """Each admissible R8BGPU_FFT_LOG2 of every plain (not block-exact) stage against the reference at the same bar."""
    with monkeypatch.context() as mp:
        _env(mp, name)
        plan, idx = _plain_bcs(pkg, name)
    if not idx:
        pytest.skip("no plain k_blockconv / k_bcl stage: block-exact tiles are the reference's blocks")
    runs = 0
    for b2 in range(10, 17):
        with monkeypatch.context() as mp:
            _env(mp, name, {"R8BGPU_FFT_LOG2": str(b2)})
            plan = make_plan(pkg, name)
            rep = unfused(plan)
            if not all(rep.get(i, {}).get("fft_log2") == b2 for i in idx):
                continue
            refs = reference(ref, ref_e1, name, plan)
            b = pkg.Batch(plan, N_CH, 0)
            rng = np.random.default_rng(b2)
            got, exp, tiles = [[] for _ in range(N_CH)], [[] for _ in range(N_CH)], {}
            m = plan.max_in_len
            _run_ref_calls(b, refs, [m, 1, m - 1, 333, m], rng, got, exp, rep, tiles)
            for _ in range(16):     # long filters: feed until the chain's latency has passed
                if sum(len(g) for g in got[0]) >= m:
                    break
                _run_ref_calls(b, refs, [m], rng, got, exp, rep, tiles)
            _parity(got, exp, "%s FFT_LOG2=%d" % (name, b2))
            runs += 1
    assert runs >= 1


# ---- bit for bit ---------------------------------------------------------------------------------------------------------

def _same(got, want, what):
    for call, (g, w) in enumerate(zip(got, want)):
        g, w = np.asarray(g), np.asarray(w)
        assert g.shape == w.shape, (what, call, g.shape, w.shape)
        if g.tobytes() != w.tobytes():
            c, j = [int(v[0]) for v in np.nonzero(g.view(np.int64) != w.view(np.int64))]
            pytest.fail("%s, call %d: channel %d first differs at output %d: %r vs %r" % (what, call, c, j, g[c, j], w[c, j]))


def _lockstep(pkg, name, xs, mp, env=None, n_ch=N_CH, odd_stride=False):
    import torch
    _env(mp, name, env)
    plan = make_plan(pkg, name)
    b = pkg.Batch(plan, n_ch, 0)
    ys = []
    cap = max(plan.max_out_len, 1)
    for x in xs:
        if odd_stride and x.shape[1]:
            out = torch.zeros((n_ch, cap | 1), dtype=torch.float64, device="cuda")
            ys.append(b.process(torch.from_numpy(x).cuda(), out=out).cpu().numpy())
        else:
            ys.append(b.process_host(x))
    return ys, b


def _inputs(plan, n_ch, seed):
    """Full, one-sample, empty, short and MaxInLen - 1 blocks, then full blocks until the chain's latency has passed and
    the calls have given at least MaxInLen / 4 outputs."""
    rng = np.random.default_rng(seed)
    m = plan.max_in_len
    lens = [m, 1, 0, 333, m - 1, m]
    while sum(plan.simulate(lens)) < m // 4 and len(lens) < 40:
        lens.append(m)
    assert sum(plan.simulate(lens)) > 0
    return [rng.uniform(-1.0, 1.0, size=(n_ch, l)) for l in lens]


@pytest.mark.parametrize("name", list(BLOCKCONVS))
def test_bit_exact_variants(pkg, name, monkeypatch):
    """Equal-length ragged calls (RAG instantiations), every admissible R8BGPU_FRAC_TILE, one channel per large-tile
    group, and odd-stride output rows: the bytes of the default lock-step call."""
    with monkeypatch.context() as mp:
        _env(mp, name)
        plan = make_plan(pkg, name)
        rep = unfused(plan)
    xs = _inputs(plan, N_CH, 5)
    with monkeypatch.context() as mp:
        want, _ = _lockstep(pkg, name, xs, mp)
    checked = []
    # a fused kernel sums in another order than k_blockconv + k_frac: ragged calls equal lock-step ones where those run
    # the same kernels (the reference test holds the others to the reference)
    n_bc = sum(s["name"] == "blockconv" for s in plan.stages())
    if sum(info["kernel"] in ("k_blockconv", "k_bcl") for info in rep.values()) == n_bc and all(
            plan.frac_info(i)["kernel"] != "fused" for i, s in enumerate(plan.stages()) if s["name"].startswith("frac")):
        with monkeypatch.context() as mp:
            _env(mp, name)
            b = pkg.Batch(make_plan(pkg, name), N_CH, 0)
            got = []
            for x in xs:
                ys = b.process_ragged([x[c] for c in range(N_CH)])
                got.append(np.array(ys).reshape(N_CH, -1))
            _same(got, want, name + " ragged")
            checked.append("ragged")
    fracs = [(i, info) for i, info in rep.items() if info["kernel"].startswith("k_frac")]
    for t in [1 << k for k in range(11)] if fracs else []:
        with monkeypatch.context() as mp:
            _env(mp, name, {"R8BGPU_FRAC_TILE": str(t)})
            plan_t = make_plan(pkg, name)
            try:
                infos = [plan_t.frac_info(i) for i, _ in fracs]
            except pkg.R8bGpuError as e:
                assert "R8BGPU_FRAC_TILE=%d" % t in str(e)
                continue
            assert all(f["tile"] == t and f["window"] <= FRAC_CAP for f in infos)
            got, b = _lockstep(pkg, name, xs, mp, {"R8BGPU_FRAC_TILE": str(t)})
            for i, _ in fracs:
                assert b.last_variant(i).startswith("k_frac poly=") and " tile=%d " % t in b.last_variant(i)
        _same(got, want, "%s FRAC_TILE=%d" % (name, t))
        checked.append("frac tile %d" % t)
    if any(info["kernel"] == "k_bcl" for info in rep.values()):
        with monkeypatch.context() as mp:
            got, b = _lockstep(pkg, name, xs, mp, {"R8BGPU_BCL_SCRATCH_MB": "1"})
            for i, info in rep.items():
                if info["kernel"] == "k_bcl":
                    g = make_plan(pkg, name).blockconv_info(i, N_CH)["group_ch"]
                    assert g < info["group_ch"] or info["group_ch"] == 1, (g, info)
                    groups = int(b.last_variant(i).split("groups=")[1])
                    assert 1 <= groups <= -(-N_CH // g), (b.last_variant(i), g)
        _same(got, want, name + " 1 MB of scratch")
        checked.append("bcl groups")
    if not plan.stages()[-1]["name"] == "hbup":
        with monkeypatch.context() as mp:
            got, _ = _lockstep(pkg, name, xs, mp, odd_stride=True)
        _same(got, want, name + " odd stride")
        checked.append("odd stride")
    print("\n%s: %s" % (name, checked))
    assert checked, name


WIDE = ["44100-7999"]   # k_blockconv<8192, 1> (1x), then k_frac<true>


@pytest.mark.parametrize("name", WIDE)
def test_wide_batch_is_the_narrow_batch(pkg, name, monkeypatch):
    """6 n_sm + 5 channels, more CTAs than one wave: the first 5 channels equal a 5-channel twin bit for bit."""
    import torch
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    n_wide = 6 * n_sm + 5
    with monkeypatch.context() as mp:
        _env(mp, name)
        plan = make_plan(pkg, name)
    xs = _inputs(plan, n_wide, 9)
    with monkeypatch.context() as mp:
        wide, _ = _lockstep(pkg, name, xs, mp, n_ch=n_wide)
    with monkeypatch.context() as mp:
        narrow, _ = _lockstep(pkg, name, [x[:5] for x in xs], mp, n_ch=5)
    _same([w[:5] for w in wide], narrow, name + " wide")


# ---- high ratios ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("src,whole", [(3072000.0, True), (3072007.0, False), (4800000.0, True), (4800011.0, False)],
                         ids=["64-whole", "64-order2", "100-whole", "100-order2"])
def test_high_ratio_single_stage(pkg, ref, src, whole):
    """Single-stage interpolators at 64:1 and 100:1 (tiles 16 and 8), against the reference's stage."""
    dst = 48000.0
    plan = pkg.Plan.single_stage(1, [src, dst, 180.15, 0], 16384)
    s = plan.stages()[0]
    assert s["name"] == ("frac_whole" if whole else "frac_poly"), s
    info = plan.frac_info(0)
    assert info["window"] <= FRAC_CAP and info["tile"] < 32, info
    refs = [ref.stage_frac(src, dst, 180.15) for _ in range(N_CH)]
    b = pkg.Batch(plan, N_CH, 0)
    rng = np.random.default_rng(3)
    got, exp, tiles = [[] for _ in range(N_CH)], [[] for _ in range(N_CH)], {}
    _run_ref_calls(b, refs, [16384, 0, 1, 99, 100, 16383, 5000, 16384], rng, got, exp, {0: info}, tiles)
    _parity(got, exp, "%g:1" % (src / dst))
