"""GPU: every entry of TABLE (tests/test_order2_geometry_cpu.py) on the fused order-2 path -- against the reference, with
each call's instantiation and geometry pinned, into NaN-filled buffers, and bit for bit across the settings that change
where coefficients and samples are read from.

R8BGPU_POLY_SINGLE, R8BGPU_BANK_GLOBAL, typed stores and the grid width change neither which output is computed nor
its arithmetic (fma(c2, x^2, fma(c1, x, c0)) per tap, taps ascending), so each is held to the default path's bytes, which
the first test holds to the reference (counts exact, max |d| <= 32 eps, rms <= 4 eps).  R8BGPU_POLY_V2 entries run on
k_up2_frac2<POLY>, whose tiles round differently, and are held to the reference only."""
import re

import numpy as np
import pytest

import oracle_util as ou
from test_gpu_asrc import oracle
from test_order2_geometry_cpu import TABLE, emul, emulate, entry, make_plan, pair_stage  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

N_CH = 3
F32, S16 = 1, 2


def expected_variant(c):
    """Batch.last_variant() of a k_up2_frac call whose decision the emulator recorded."""
    d = c["poly_dir"]
    return "k_up2_frac<1,8,%s,false> tiles=%d span=%d dir=%s rows=%d stride=%d chunks=%d N=%d" % (
        "true" if c["ysh"] != 31 else "false", c["n_tiles"], c["span"], "+1" if d > 0 else "-1" if d < 0 else "0",
        c["poly_rows_cap"], c["poly_row_stride"], c["poly_chunks"], c["poly_n"])


def feed(name, n_ch, seed):
    e = entry(name)
    rng = np.random.default_rng(seed)
    return [rng.uniform(-1.0, 1.0, size=(n_ch, l)) for l in e["lens"]]


def run(pkg, name, monkeypatch, env=None, n_ch=N_CH, seed=5, out_fmt=None, out_scale=1.0, xs=None):
    """A fresh batch under the entry's settings plus env, fed the entry's calls (each after its trim factor).  Returns
    (outputs per call, last_variant() per call ('' for calls without output), plan, stage)."""
    e = entry(name)
    with monkeypatch.context() as mp:
        for k, v in dict(e["env"], **(env or {})).items():
            mp.setenv(k, v)
        plan = make_plan(pkg, name)
        i = pair_stage(plan)
        b = pkg.Batch(plan, n_ch, 0)
        ys, vs = [], []
        for call, x in enumerate(xs or feed(name, n_ch, seed)):
            if e["kind"] == "asrc":
                b.set_trim(np.arange(n_ch), np.full(n_ch, e["factors"][call]))
            y = b.process_host(x) if out_fmt is None else b.process_host_fmt(x, out_fmt=out_fmt, out_scale=out_scale)
            ys.append(y)
            vs.append(b.last_variant(i) if y.shape[1] else "")
        return ys, vs, plan, i


def want_of(ref, name, plan, xs):
    """Per channel, the reference's per-call outputs: ref.Resampler for fixed ratios (built with R8B_FASTTIMING for the
    fast-timing entries), the stage-built long-double oracle for trim plans."""
    e = entry(name)
    if e["ft"]:
        if not ou.have_ref("e0_ft"):
            pytest.skip("oracle/_ref fast-timing build missing")
        ref = ou.RefOracle("e0_ft")
    out = []
    for c in range(xs[0].shape[0]):
        if e["kind"] == "asrc":
            out.append(oracle(ref, plan, e["src"], e["dst"], e["tb"], e["atten"], [x[c] for x in xs], e["factors"]))
        else:
            r = ref.Resampler(e["src"], e["dst"], e["m"], e["tb"], e["atten"])
            out.append([r.process(x[c]) for x in xs])
    return out


@pytest.mark.parametrize("name", list(TABLE))
def test_reference_parity_and_geometry(pkg, ref, emul, name, monkeypatch):  # noqa: F811
    e = entry(name)
    xs = feed(name, N_CH, 17)
    got, vs, plan, i = run(pkg, name, monkeypatch, xs=xs)
    bad, _, per_call = emulate(emul, name)
    assert bad == 0
    for call, (v, c) in enumerate(zip(vs, per_call)):
        if not c["launched"]:
            continue
        if "R8BGPU_POLY_V2" in e["env"]:
            assert re.fullmatch(r"k_up2_frac2<\d+,false,0,\w+,2,false,true,\w+,\w+> mbu=\d+", v), (call, v)
        else:
            assert v == expected_variant(c), (call, v, expected_variant(c))
    want = want_of(ref, name, plan, xs)
    for c in range(N_CH):
        assert [len(w) for w in want[c]] == [g.shape[1] for g in got], c
        a, w = np.concatenate([g[c] for g in got]), np.concatenate(want[c])
        mx, rms = ou.parity_metrics(a, w)
        assert mx <= 32 * ou.EPS and rms <= 4 * ou.EPS, (c, mx / ou.EPS, rms / ou.EPS)


SENTINEL_PLANS = ["47700-55dB", "47400-55dB", "32001-126", "96001-96", "47999-24-ft"]


@pytest.mark.parametrize("name", SENTINEL_PLANS)
def test_every_output_written_nothing_past(pkg, name, monkeypatch):
    """Device buffers filled with a NaN sentinel, row stride odd: outputs [0, n) equal the host path's bytes, every
    element past n keeps the sentinel."""
    import torch
    e = entry(name)
    xs = feed(name, N_CH, 29)
    want, _, _, _ = run(pkg, name, monkeypatch, xs=xs)
    plan = make_plan(pkg, name)
    b = pkg.Batch(plan, N_CH, 0)
    cap = b.max_out_len
    stride = cap + 3 + (cap & 1)   # odd
    sentinel = np.frombuffer(np.uint64(0x7FF8DEAD0000BEEF).tobytes(), dtype=np.float64)[0]
    for call, x in enumerate(xs):
        l = x.shape[1]
        d_in = torch.from_numpy(np.ascontiguousarray(np.pad(x, ((0, 0), (0, 1))))).cuda()  # in stride l + 1
        d_out = torch.full((N_CH, stride), sentinel, dtype=torch.float64, device="cuda")
        n = b.process_ptr(d_in.data_ptr(), l + 1, l, d_out.data_ptr(), stride, cap)
        b.sync()
        y = d_out.cpu().numpy()
        assert n == want[call].shape[1], (call, n)
        assert np.isfinite(y[:, :n]).all(), call
        assert y[:, :n].tobytes() == want[call].tobytes(), call
        tail = y[:, n:].view(np.uint64)
        assert (tail == np.uint64(0x7FF8DEAD0000BEEF)).all(), (call, "an element past n was written")
    assert e["lens"]


EXACT_PLANS = ["47700-55dB", "47400-55dB", "47999-24", "32001-126", "96001-96", "asrc-48000-55dB"]
SETTINGS = {
    "single": {"R8BGPU_POLY_SINGLE": "1"},
    "global": {"R8BGPU_BANK_GLOBAL": "1"},
    "single-global": {"R8BGPU_POLY_SINGLE": "1", "R8BGPU_BANK_GLOBAL": "1"},
}
_baseline = {}


def baseline(pkg, name, monkeypatch):
    if name not in _baseline:
        _baseline[name] = run(pkg, name, monkeypatch)
    return _baseline[name]


def first_diff(got, want):
    c, j = [int(v[0]) for v in np.nonzero(got != want)]
    return "channel %d first differs at output %d: %r vs %r" % (c, j, got[c, j], want[c, j])


@pytest.mark.parametrize("setting", list(SETTINGS))
@pytest.mark.parametrize("name", EXACT_PLANS)
def test_settings_are_bit_exact(pkg, name, setting, monkeypatch):
    want, _, _, _ = baseline(pkg, name, monkeypatch)
    got, vs, _, _ = run(pkg, name, monkeypatch, SETTINGS[setting])
    env = SETTINGS[setting]
    for call, v in enumerate(vs):
        if not v:
            continue
        if "R8BGPU_BANK_GLOBAL" in env:
            assert " dir=0 " in v and v.endswith(" N=0"), (call, v)
        else:
            assert v.startswith("k_up2_frac<1,8,false,false>") and v.endswith(" N=0"), (call, v)
    for call, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape, (call, g.shape, w.shape)
        if g.tobytes() != w.tobytes():
            pytest.fail("%s, call %d: %s" % (setting, call, first_diff(g.view(np.int64), w.view(np.int64))))


@pytest.mark.parametrize("name", ["47700-55dB", "32001-126", "asrc-48000-55dB"])
def test_typed_outputs_are_the_narrowed_fp64_output(pkg, name, monkeypatch):
    want, _, _, _ = baseline(pkg, name, monkeypatch)
    g32, _, _, _ = run(pkg, name, monkeypatch, out_fmt=F32)
    scale = 20000.0
    g16, _, _, _ = run(pkg, name, monkeypatch, out_fmt=S16, out_scale=scale)
    for call, (a, b, w) in enumerate(zip(g32, g16, want)):
        w32 = w.astype(np.float32)
        assert a.dtype == np.float32 and a.tobytes() == w32.tobytes(), call
        w16 = np.clip(np.trunc(w * scale), -32768, 32767).astype(np.int16)
        assert b.dtype == np.int16 and np.array_equal(b, w16), (call, first_diff(b, w16) if b.shape == w16.shape else "")


@pytest.mark.parametrize("name", ["47700-55dB", "asrc-48000-55dB"])
def test_wide_grid_equals_a_narrow_twin(pkg, name, monkeypatch):
    """6 n_sm + 5 channels; channel c carries the input of channel c % 5 of a 5-channel twin and equals it bit for bit."""
    import torch
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    n = 6 * n_sm + 5
    x5 = feed(name, 5, 41)
    xw = [np.ascontiguousarray(x[np.arange(n) % 5]) for x in x5]
    twin, _, _, _ = run(pkg, name, monkeypatch, n_ch=5, xs=x5)
    wide, vs, _, _ = run(pkg, name, monkeypatch, n_ch=n, xs=xw)
    assert any(vs)
    for call, (yw, yt) in enumerate(zip(wide, twin)):
        assert yw.shape == (n, yt.shape[1])
        for c in range(n):
            if yw[c].tobytes() != yt[c % 5].tobytes():
                pytest.fail("call %d: channel %d differs from twin channel %d" % (call, c, c % 5))
