"""GPU: every plan of GEOMETRIES (tests/test_fused_geometry_cpu.py) on the fused kernels -- against the reference, with the
instantiation it reaches pinned, and bit for bit across the kernel's exact variants and store paths.

The tensor-path interpolation changes no bit relative to the sequential FMA loops (DESIGN.md section 3), the work-unit
size, phase-group shape and bulk copy change no arithmetic, and a typed store narrows the very fp64 value the linear
store writes.  So each variant is held to the default path's bytes, which the first test holds to the reference."""
import re

import numpy as np
import pytest

import oracle_util as ou
from test_fused_geometry_cpu import GEOMETRIES, make_plan, pair_stage, report

pytestmark = pytest.mark.gpu

N_CH = 3
F32, S16 = 1, 2


def tf(v):
    return "true" if v else "false"


def expected_variant(plan, i, info, typed=False):
    """Pattern of Batch.last_variant() for the pair at stage i: the template arguments the report implies (the FMA
    path's phase-group shape and the work-unit size are chosen per call)."""
    k, pad, cs = info["kernel"], tf(info["pad"]), tf(info["cs"])
    lin = tf(i + 2 == len(plan.stages()) and not typed)    # linear fp64 destination: the pair writes the call's output
    if k == "f2-tc":
        return r"k_up2_frac2<8,%s,0,true,%d,false,false,%s,%s> mbu=[246]" % (pad, info["up"], cs, lin)
    if k == "f2-fma":
        return r"k_up2_frac2<%d,%s,[012],false,2,false,false,%s,false> mbu=[246]" % (info["ir"], pad, cs)
    if k in ("v1-smem", "v1-global"):
        return r"k_up2_frac<0,%d,%s,%s>" % (info["ir"], pad, tf(k == "v1-smem"))
    assert k == "f2-copy", info
    return r"k_up2_frac2<8,false,0,true,2,true,false,%s,false> mbu=0" % cs


def residue_lens(plan, lens):
    """lens, extended so that calls with output start at every output index residue mod 8 (phase groups then start at
    every r0 = e0 mod 8 of a call)."""
    m = plan.max_in_len
    lens = list(lens)

    def starts(ls):
        c = plan.simulate(ls)
        t = np.concatenate([[0], np.cumsum(c)[:-1]])
        return {int(t[j]) % 8 for j in range(len(ls)) if c[j] > 0}, int(sum(c))
    seen, total = starts(lens)
    l0 = m // 3 + 1
    while len(seen) < 8:
        for l in range(l0, l0 + 64):
            if (total + plan.simulate(lens + [l])[-1]) % 8 not in seen:
                break
        lens += [l, m]
        seen, total = starts(lens)
        assert len(lens) < 60, "residues not reached"
    return lens


def call_lens(plan):
    """Full, empty, tiny, odd and max - 1 blocks; where the interpolator of the pair writes the call's output, also calls
    that start at every output residue."""
    m = plan.max_in_len
    lens = [m, 0, 1, 7, m, 333, m - 1, m, 2 * (m // 3) + 1]
    st = plan.stages()
    return residue_lens(plan, lens) if st[-1]["name"] == "frac_whole" and pair_stage(plan) == len(st) - 2 else lens


def run(pkg, name, monkeypatch, env=None, lens=None, seed=5, out_fmt=None, out_scale=1.0, dither_seed=None):
    """A fresh batch of N_CH channels under the entry's settings plus env, fed seeded calls.  Returns (outputs per call,
    last_variant() after each call that produced output, plan, stage, report)."""
    with monkeypatch.context() as mp:
        for k, v in dict(GEOMETRIES[name][6], **(env or {})).items():
            mp.setenv(k, v)
        plan, i, info = report(pkg, name, monkeypatch)
        b = pkg.Batch(plan, N_CH, 0)
        if dither_seed is not None:
            b.set_dither(range(N_CH), dither_seed)
        rng = np.random.default_rng(seed)
        ys, vs = [], []
        for l in lens or call_lens(plan):
            x = rng.uniform(-0.9, 0.9, size=(N_CH, l))
            y = b.process_host(x) if out_fmt is None else b.process_host_fmt(x, out_fmt=out_fmt, out_scale=out_scale)
            ys.append(y)
            if y.shape[1]:
                vs.append(b.last_variant(i))
        return ys, vs, plan, i, info


def first_diff(got, want):
    c, j = [int(v[0]) for v in np.nonzero(got != want)]
    return "channel %d first differs at output %d: %r vs %r" % (c, j, got[c, j], want[c, j])


@pytest.mark.parametrize("name", list(GEOMETRIES))
def test_reference_parity_and_instantiation(pkg, name, monkeypatch, request):
    ref = request.getfixturevalue("ref_e1" if GEOMETRIES[name][5] else "ref")
    src, dst, m, tb, at = GEOMETRIES[name][:5]
    with monkeypatch.context() as mp:
        for k, v in GEOMETRIES[name][6].items():
            mp.setenv(k, v)
        plan, i, info = report(pkg, name, monkeypatch)
        assert info["kernel"] == GEOMETRIES[name][7]
        b = pkg.Batch(plan, N_CH, 0)
        rs = [ref.Resampler(src, dst, m, tb, at) for _ in range(N_CH)]
        want = expected_variant(plan, i, info)
        rng = np.random.default_rng(17)
        got, exp, total = [[] for _ in range(N_CH)], [[] for _ in range(N_CH)], 0
        for call, l in enumerate(call_lens(plan)):
            x = rng.uniform(-1.0, 1.0, size=(N_CH, l))
            y = b.process_host(x)
            for c in range(N_CH):
                r = rs[c].process(x[c])
                assert len(r) == y.shape[1], (call, l, len(r), y.shape[1])
                got[c].append(y[c])
                exp[c].append(r)
            if y.shape[1]:
                v = b.last_variant(i)
                assert re.fullmatch(want, v), (call, v, want)
            total += y.shape[1]
    assert total > 0
    for c in range(N_CH):
        a, e = np.concatenate(got[c]), np.concatenate(exp[c])
        mx, rms = ou.parity_metrics(a, e)
        assert mx <= 32 * ou.EPS and rms <= 4 * ou.EPS, (c, mx / ou.EPS, rms / ou.EPS)


# ---- bit for bit across the exact variants -------------------------------------------------------------------------------

# name -> (settings, the kernel the report must show under them, what last_variant() must show)
VARIANTS = {
    "fma-glog0": ({"R8BGPU_F2_FLAGS": "2", "R8BGPU_F2_GLOG": "0"}, "f2-fma", r"k_up2_frac2<\d+,\w+,0,false,.*"),
    "fma-glog1": ({"R8BGPU_F2_FLAGS": "2", "R8BGPU_F2_GLOG": "1"}, "f2-fma", r"k_up2_frac2<\d+,\w+,1,false,.*"),
    "fma-glog2": ({"R8BGPU_F2_FLAGS": "2", "R8BGPU_F2_GLOG": "2"}, "f2-fma", r"k_up2_frac2<\d+,\w+,2,false,.*"),
    "fma-ir10": ({"R8BGPU_F2_FLAGS": "2", "R8BGPU_IR": "10"}, "f2-fma", r"k_up2_frac2<10,\w+,[012],false,.*"),
    "mbu2": ({"R8BGPU_F2_MBU": "2"}, "f2-tc", r"k_up2_frac2<8,\w+,0,true,.* mbu=2"),
    "mbu4": ({"R8BGPU_F2_MBU": "4"}, "f2-tc", r"k_up2_frac2<8,\w+,0,true,.* mbu=4"),
    "mbu6": ({"R8BGPU_F2_MBU": "6"}, "f2-tc", r"k_up2_frac2<8,\w+,0,true,.* mbu=6"),
    "no-bulk-copy": ({"R8BGPU_F2_FLAGS": "4"}, "f2-tc", r"k_up2_frac2<8,\w+,0,true,.*"),
}
TC_PLANS = [n for n, g in GEOMETRIES.items() if g[7] == "f2-tc" and not g[6]]
VARIANT_CASES = [(n, v) for n in TC_PLANS for v in VARIANTS]
_baseline = {}


@pytest.mark.parametrize("name,variant", VARIANT_CASES, ids=["%s-%s" % c for c in VARIANT_CASES])
def test_variant_is_bit_exact(pkg, name, variant, monkeypatch):
    env, kernel, pattern = VARIANTS[variant]
    _, _, vinfo = report(pkg, name, monkeypatch, env)
    if vinfo["kernel"] != kernel:
        pytest.skip("%s does not run %s on %s: the report gives %s (tensor bank fits %d, FMA bank fits %d)"
                    % (variant, kernel, name, vinfo["kernel"], vinfo["tc_fits"], vinfo["fma_fits"]))
    if name not in _baseline:
        _baseline[name] = run(pkg, name, monkeypatch)
    want, _, plan, _, _ = _baseline[name]
    got, vs, _, _, _ = run(pkg, name, monkeypatch, env)
    assert vs and all(re.fullmatch(pattern, v) for v in vs), (vs, pattern)
    for call, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape, (call, g.shape, w.shape)
        if g.tobytes() != w.tobytes():
            pytest.fail("%s, call %d: %s" % (variant, call, first_diff(g.view(np.int64), w.view(np.int64))))


# ---- store paths ---------------------------------------------------------------------------------------------------------

def _tc_last_pairs(pkg):
    out = []
    for n in TC_PLANS:
        plan = make_plan(pkg, n)
        if pair_stage(plan) + 2 == len(plan.stages()):
            out.append(n)
    return out


@pytest.mark.parametrize("name", TC_PLANS)
def test_float32_store_is_the_rounded_fp64_output(pkg, name, monkeypatch):
    """Planar float32 output through the tensor path's general store equals fl32 of the fp64 output, bit for bit."""
    if name not in _tc_last_pairs(pkg):
        pytest.skip("%s: the fused pair does not write the call's output" % name)
    want, _, plan, i, info = run(pkg, name, monkeypatch, seed=9)
    got, vs, _, _, _ = run(pkg, name, monkeypatch, seed=9, out_fmt=F32)
    pattern = expected_variant(plan, i, info, typed=True)
    assert vs and all(re.fullmatch(pattern, v) for v in vs), (vs, pattern)
    for call, (g, w) in enumerate(zip(got, want)):
        w32 = w.astype(np.float32)
        assert g.dtype == np.float32 and g.shape == w32.shape
        if g.tobytes() != w32.tobytes():
            pytest.fail("call %d: %s" % (call, first_diff(g.view(np.int32), w32.view(np.int32))))


@pytest.mark.parametrize("name", ["48000-44100", "180-660"])
def test_dithered_int16_store(pkg, name, monkeypatch):
    """TPDF-dithered int16 output of the fused store equals the host quantiser applied to the fp64 output."""
    scale, seed = 20000.0, 4242
    want, _, _, _, _ = run(pkg, name, monkeypatch, seed=3)
    got, vs, _, _, _ = run(pkg, name, monkeypatch, seed=3, out_fmt=S16, out_scale=scale, dither_seed=seed)
    assert vs and all(",false> mbu=" in v for v in vs), vs    # the general store, not the linear fp64 one
    state = [np.zeros(pkg.DITHER_MAX_TAPS) for _ in range(N_CH)]
    n = [0] * N_CH
    for call, (g, w) in enumerate(zip(got, want)):
        for c in range(N_CH):
            q, state[c] = pkg.dither_quantize(w[c], pkg.S16, seed, scale=scale, first_index=n[c], state=state[c])
            np.testing.assert_array_equal(g[c], q, err_msg="call %d channel %d" % (call, c))
            n[c] += len(w[c])


# ---- the persistent grid -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["44100-96000", "96000-44100"])
def test_persistent_grid(pkg, ref, name):
    """6 n_sm + 5 channels, so every half-CTA of the persistent kernel runs at least 3 tiles per call.  Channel c carries
    the input of channel c % 5 of a 5-channel twin and must equal it bit for bit; two twin channels against the
    reference."""
    import torch
    src, dst, m, tb, at = GEOMETRIES[name][:5]
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    n = 6 * n_sm + 5
    plan = make_plan(pkg, name)
    i = pair_stage(plan)
    assert plan.stages()[i]["up"] == (2 if name == "44100-96000" else 1)
    wide, twin = pkg.Batch(plan, n, 0), pkg.Batch(plan, 5, 0)
    rs = [ref.Resampler(src, dst, m, tb, at) for _ in range(2)]
    rng = np.random.default_rng(23)
    got, exp = [[], []], [[], []]
    for call, l in enumerate([m, m, m - 3, m, 1001, m]):
        x5 = rng.uniform(-1.0, 1.0, size=(5, l))
        x = np.ascontiguousarray(x5[np.arange(n) % 5])
        yw = wide.process(torch.from_numpy(x).cuda()).cpu().numpy()
        yt = twin.process_host(x5)
        assert yw.shape == (n, yt.shape[1])
        if yt.shape[1]:
            assert re.fullmatch(r"k_up2_frac2<8,\w+,0,true,.*", wide.last_variant(i)), wide.last_variant(i)
        for c in range(n):
            if yw[c].tobytes() != yt[c % 5].tobytes():
                pytest.fail("call %d: channel %d differs from twin channel %d" % (call, c, c % 5))
        for c in range(2):
            r = rs[c].process(x5[c])
            assert len(r) == yt.shape[1]
            got[c].append(yt[c])
            exp[c].append(r)
    for c in range(2):
        mx, rms = ou.parity_metrics(np.concatenate(got[c]), np.concatenate(exp[c]))
        assert mx <= 32 * ou.EPS and rms <= 4 * ou.EPS, (c, mx / ou.EPS, rms / ou.EPS)
