"""CPU: the per-call geometry of k_up2_frac's order-2 path (a 2x BlockConvolver fused with the order-2 interpolator),
and a committed table of plans and factor sequences that reaches every class of it.

Every lock-step call of such a pair decides, from its rates (a trim factor moves dsr), its span of 2x-stream positions
and the bank's flen and fracs: the kernel (k_up2_frac, or k_up2_frac2<POLY> under R8BGPU_POLY_V2), the tiles, whether a
circular run of bank rows is staged in shared memory and in which direction (poly_dir), the staging capacity and row
stride, the number of chunks a tile pair's outputs are cut into, the outputs per thread (poly_n, poly_block4<N>) and the
y layout.  plan_poly_call (r8b_hosttab.cpp) decides all of it in one place; Plan.order2_info() reports it without a
device, restated here in closed form.

tests/cpp/order2_pairs.cpp replays each call of a table entry pair by pair with the kernel's own bookkeeping
(r8b_poly.cuh): the pairs' output ranges partition the call and each pair owns exactly the outputs whose read position
lies in its tiles; every owned window lies inside its tile buffer (PolyOut::ok, so the kernel's `if (!o.ok)` branches
never drop an output) and inside the tile's valid overlap-save samples; every staged row read is the bank row it stands
for.  tests/test_gpu_order2_geometry.py runs every entry against the reference.

The deferred-output queue (POLY_QUEUE = 1024 entries per chunk) overflows: with the 8-row bank (49-55 dB) a ratio
1-2 % off an integer changes bank row every few outputs, so a third or more of the four-output groups fall back to
the queue, and a chunk of a full tile pair holds several thousand outputs.  The emulator counts more than 2300 deferred
outputs in one chunk of 48000 -> 47700.3, and a 48000 -> 48000 drift-compensation link trimmed by 1 % overflows too;
the rest are computed in place by the queue-full branch.  The table keeps such entries, so the GPU sweep runs that
branch against the reference.

Classes no plan reaches: an odd flen (the bank has base + 2 r taps, base 8 or 6, so the odd-flen guard of the staging
decision is dead); a whole-bank staged run (n_st == fracs) whose bank is larger than 8 rows (staging needs a short run,
and every bank above 8 rows is then far longer than a chunk's run); poly_n 0 with staging except through
R8BGPU_POLY_SINGLE (a staged call has a ratio within a few per cent of 1, 2 or 3, and the planner fuses no ratio near 4:
the 2x BlockConvolver makes the interpolator's ratio at most about 2 before decimation stages take over)."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "r8brain-free-src_b200", "csrc")

ATTEN_24 = 180.15
FRACWIN2_ATTEN = [55.5446, 81.4191, 96.3392, 111.1315, 125.4653, 139.7379, 154.0532, 168.2101, 182.1076, 195.5668,
                  209.0610, 222.5010]
# one requested attenuation per R8B_FRACWIN2 row (the row is the first whose attenuation reaches the request)
ROW_ATTENS = [49.0] + [a + 0.01 for a in FRACWIN2_ATTEN[:-1]]
M = 65536

# name -> dict(kind: "plan" | "asrc", src, dst, tb, atten, m, lens, factors (asrc: one per call), max_trim, ft, env)
_FULL = [M] * 3
TABLE = {
    # N = 2, rows ascending: 1.3 % off 2 at 55 dB -- two chunks, queue overflow, ragged spans, odd tile counts
    "47700-55dB": dict(kind="plan", src=48000.0, dst=47700.3, atten=49.0, lens=[M, 1000, 333, M, 5000, 17, M]),
    # three and four chunks at 55 dB, queue overflow
    "47550-55dB": dict(kind="plan", src=48000.0, dst=47550.3, atten=49.0, lens=[M, M]),
    "47400-55dB": dict(kind="plan", src=48000.0, dst=47400.3, atten=49.0, lens=_FULL),
    # N = 2 at 24 bit: the chains the suite ran before, now with their geometry pinned
    "47999-24": dict(kind="plan", src=48000.0, dst=47999.0, atten=ATTEN_24, lens=[M, 40000, 9, M]),
    "48001-24": dict(kind="plan", src=48000.0, dst=48001.0, atten=ATTEN_24, lens=[M, 40000, M]),      # N = 2, rows descending
    "47995-126": dict(kind="plan", src=48000.0, dst=47995.0, atten=126.0, lens=_FULL),               # two chunks
    "95999-96": dict(kind="plan", src=48000.0, dst=95999.0, atten=96.0, lens=_FULL),                 # N = 1, ascending
    "96001-96": dict(kind="plan", src=48000.0, dst=96001.0, atten=96.0, lens=_FULL),                 # N = 1, descending
    "31999-126": dict(kind="plan", src=48000.0, dst=31999.0, atten=126.0, lens=_FULL),               # N = 3, ascending
    "32001-126": dict(kind="plan", src=48000.0, dst=32001.0, atten=126.0, lens=_FULL),               # N = 3, descending
    "48001.3-24": dict(kind="plan", src=44100.0, dst=48001.3, atten=ATTEN_24, lens=[M, 20000, M]),   # unstaged: > 4 chunks
    "47999-218": dict(kind="plan", src=48000.0, dst=47999.0, atten=218.0, lens=[M, 7, M]),           # 222 dB row, unstaged
    "47999-24-ft": dict(kind="plan", src=48000.0, dst=47999.0, atten=ATTEN_24, ft=1, lens=[M, 3001, M]),  # R8B_FASTTIMING
    "47999-24-global": dict(kind="plan", src=48000.0, dst=47999.0, atten=ATTEN_24, lens=[M, 3001, M],
                            env={"R8BGPU_BANK_GLOBAL": "1"}),
    "47999-24-single": dict(kind="plan", src=48000.0, dst=47999.0, atten=ATTEN_24, lens=[M, 3001, M],
                            env={"R8BGPU_POLY_SINGLE": "1"}),
    "47999-24-v2": dict(kind="plan", src=48000.0, dst=47999.0, atten=ATTEN_24, lens=[M, 3001, M],
                        env={"R8BGPU_POLY_V2": "1"}),
    # drift compensation at 48000 -> 48000: f = 1 exactly (ratio 2, every output on row 0), then factors crossing 1 both
    # ways by up to 1 % (direction flips, four chunks, queue overflow at 55 dB)
    "asrc-48000-55dB": dict(kind="asrc", src=48000.0, dst=48000.0, atten=49.0, max_trim=0.01,
                            lens=[M, M, M, M, M, 3000, M], factors=[1.0, 1.01, 0.99, 1.005, 0.995, 1.0, 1.0 + 1.7e-4]),
    # the whole 8-row bank staged (n_st == fracs): small drifts at 55 dB
    "asrc-48000-55dB-small": dict(kind="asrc", src=48000.0, dst=48000.0, atten=49.0, max_trim=0.01,
                                  lens=[M, M, 20000, M], factors=[1.0 + 3e-4, 1.0 - 3e-4, 1.0 + 2e-3, 1.0 - 6e-4]),
    # 44100 -> 352800: the pair writes the ring of the 2x BlockConvolver behind it
    "asrc-352800-24": dict(kind="asrc", src=44100.0, dst=352800.0, atten=ATTEN_24, max_trim=0.001, m=16384,
                           lens=[16384] * 4, factors=[1.0, 1.0001, 0.9999, 1.0]),
}

STATS = ("calls pairs outputs bad_own not_ok bad_row not_valid max_queue overflow row_fracs max_nst whole_bank wrap_up "
         "wrap_dn max_chunks fast odd_tiles dir_up dir_dn dir_none staged_reads ft_calls row0_wrap dir_flips "
         "v2_calls").split()
PER_CALL = ("range", "n_tiles", "span", "poly_dir", "poly_rows_cap", "poly_row_stride", "poly_chunks", "poly_n", "ysh",
            "queue", "launched", "v2", "row0_wrap", "max_row")

# every class some entry must reach
CLASSES = (["N=%d dir=%+d" % (n, d) for n in (1, 2, 3) for d in (1, -1)] +
           ["chunks=%d" % c for c in (1, 2, 3, 4)] +
           ["N=0 staged", "unstaged by chunk count", "unstaged by BANK_GLOBAL", "exact integer ratio",
            "run wraps ascending", "run wraps descending", "whole bank staged", "stride padded", "stride unpadded",
            "odd tile count", "pair writes a ring", "dir flip", "fast timing", "POLY_V2", "queue overflow",
            "span of a few outputs"])


def _cuda_include():
    for d in (os.environ.get("CUDA_HOME"), "/usr/local/cuda"):
        if d and os.path.exists(os.path.join(d, "include", "cuda_runtime.h")):
            return os.path.join(d, "include")
    return None


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    inc = _cuda_include()
    if inc is None:
        pytest.skip("CUDA headers not found")
    so = str(tmp_path_factory.mktemp("o2pairs") / "libo2pairs.so")
    srcs = [os.path.join(HERE, "cpp", "order2_pairs.cpp")] + [os.path.join(CSRC, f) for f in
                                                              ("r8b_plan.cpp", "r8b_design.cpp", "r8b_hosttab.cpp")]
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-I" + inc, "-o", so] + srcs,
                   check=True)
    L = C.CDLL(so)
    L.o2pairs_run.restype = C.c_int
    L.o2pairs_run.argtypes = [C.c_int, C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_int, C.c_double,
                              C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.o2first_k.restype = C.c_longlong
    L.o2first_k.argtypes = [C.c_double, C.c_double, C.c_double, C.c_int, C.c_int, C.c_longlong, C.c_longlong,
                            C.c_longlong, C.POINTER(C.c_longlong)]
    return L


def entry(name):
    e = dict(tb=2.0, m=M, ft=0, max_trim=0.0, env={}, factors=None)
    e.update(TABLE[name])
    if e["factors"] is None:
        e["factors"] = [1.0] * len(e["lens"])
    return e


def make_plan(pkg, name):
    e = entry(name)
    if e["kind"] == "asrc":
        return pkg.Plan.asrc(e["src"], e["dst"], e["m"], e["tb"], e["atten"], e["max_trim"])
    return pkg.Plan(e["src"], e["dst"], e["m"], e["tb"], e["atten"], fasttiming=e["ft"])


def pair_stage(plan):
    """The BlockConvolver fused with the order-2 interpolator behind it."""
    st = plan.stages()
    return next(i for i in range(len(st) - 1) if st[i]["name"] == "blockconv" and st[i + 1]["name"] == "frac_poly")


def emulate(emul, name):
    """(failures, stats dict, per-call list of dicts) of the entry's stream under its settings."""
    e = entry(name)
    lens = np.asarray(e["lens"], dtype=np.int32)
    fs = np.asarray(e["factors"], dtype=np.float64)
    st = np.zeros(len(STATS), dtype=np.int64)
    pc = np.zeros((len(lens), len(PER_CALL)), dtype=np.int64)
    kind = 2 if e["kind"] == "asrc" else 0
    bad = emul.o2pairs_run(kind, e["src"], e["dst"], e["m"], e["tb"], e["atten"], e["ft"], e["max_trim"],
                           lens.ctypes.data, fs.ctypes.data, len(lens), int("R8BGPU_BANK_GLOBAL" in e["env"]),
                           int("R8BGPU_POLY_SINGLE" in e["env"]), int("R8BGPU_POLY_V2" in e["env"]), st.ctypes.data,
                           pc.ctypes.data)
    return bad, dict(zip(STATS, st.tolist())), [dict(zip(PER_CALL, r)) for r in pc.tolist()]


def reports(pkg, name, monkeypatch, per_call):
    """Plan.order2_info at each launching call's factor and span, under the entry's settings."""
    e = entry(name)
    with monkeypatch.context() as mp:
        for k, v in e["env"].items():
            mp.setenv(k, v)
        plan = make_plan(pkg, name)
        i = pair_stage(plan)
        return plan, i, [plan.order2_info(i, f, c["range"]) if c["launched"] else None
                         for f, c in zip(e["factors"], per_call)]


def classes_of(name, plan, i, stats, infos, per_call):
    e = entry(name)
    out = set()
    for info, c in zip(infos, per_call):
        if info is None:
            continue
        if info["poly_v2"]:
            out.add("POLY_V2")
            continue
        n, d = info["poly_n"], info["poly_dir"]
        if d and n:
            out.add("N=%d dir=%+d" % (n, d))
        if d and not n:
            out.add("N=0 staged")
        if d:
            out.add("chunks=%d" % info["poly_chunks"])
            out.add("stride padded" if info["poly_row_stride"] != 3 * info["flen"] else "stride unpadded")
        elif "R8BGPU_BANK_GLOBAL" in e["env"]:
            out.add("unstaged by BANK_GLOBAL")
        else:
            out.add("unstaged by chunk count")
        if info["n_tiles"] & 1:
            out.add("odd tile count")
        if info["span"] <= 64:
            out.add("span of a few outputs")
        # f = 1 exactly: every output reads row 0 and the staged run starts at row fracs - 1
        if info["ratio"] == round(info["ratio"]) and d and c["max_row"] == 0 and c["row0_wrap"] > 0:
            out.add("exact integer ratio")
    if stats["wrap_up"]:
        out.add("run wraps ascending")
    if stats["wrap_dn"]:
        out.add("run wraps descending")
    if stats["whole_bank"]:
        out.add("whole bank staged")
    if stats["dir_flips"]:
        out.add("dir flip")
    if stats["ft_calls"]:
        out.add("fast timing")
    if stats["overflow"]:
        out.add("queue overflow")
    # launch_call writes the pair's outputs into the ring of the stage behind the interpolator whenever the interpolator
    # is not the plan's last stage (else into the caller's buffer)
    if i + 2 < len(plan.stages()) and stats["calls"] > 0:
        out.add("pair writes a ring")
    return out


# ---- the emulator ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(TABLE))
def test_every_pair_owns_its_outputs(emul, name):
    e = entry(name)
    bad, st, _ = emulate(emul, name)
    assert bad >= 0, "%s has no fused order-2 pair" % name
    assert bad == 0, (name, {k: st[k] for k in ("bad_own", "not_ok", "bad_row", "not_valid")})
    if "R8BGPU_POLY_V2" in e["env"]:
        assert st["v2_calls"] > 0  # (calls on k_up2_frac2 are counted, not replayed)
    else:
        assert st["calls"] > 0 and st["outputs"] > 0 and st["v2_calls"] == 0
    if "R8BGPU_POLY_V2" not in e["env"] and "R8BGPU_BANK_GLOBAL" not in e["env"]:
        # a staged call reads staged rows for most of its outputs
        if st["dir_up"] + st["dir_dn"]:
            assert st["staged_reads"] > 0


@pytest.mark.parametrize("name", list(TABLE))
def test_each_call_is_reported(pkg, emul, name, monkeypatch):
    """The emulator's per-call decision (plan_poly_call with the call's own rates and span) equals the report at that
    call's factor and span."""
    _, _, per_call = emulate(emul, name)
    _, _, infos = reports(pkg, name, monkeypatch, per_call)
    for call, (c, info) in enumerate(zip(per_call, infos)):
        if info is None:
            continue
        assert info["poly_v2"] == c["v2"], (name, call)
        if c["v2"]:
            continue  # (the emulator replays k_up2_frac only; k_up2_frac2's tiles are checked by test_fused2_tiles_cpu)
        for f in ("n_tiles", "span", "poly_dir", "poly_rows_cap", "poly_row_stride", "poly_chunks", "poly_n", "ysh"):
            assert info[f] == c[f], (name, call, f, info[f], c[f])


def test_table_reaches_every_class(pkg, emul, monkeypatch):
    seen = {}
    for name in TABLE:
        _, st, per_call = emulate(emul, name)
        plan, i, infos = reports(pkg, name, monkeypatch, per_call)
        for c in classes_of(name, plan, i, st, infos, per_call):
            seen.setdefault(c, []).append(name)
    missing = [c for c in CLASSES if c not in seen]
    assert not missing, missing


def test_queue_overflow_is_reachable(emul):
    """The deferred-output queue of one chunk holds POLY_QUEUE = 1024 outputs; these streams defer more."""
    for name in ("47700-55dB", "47400-55dB", "asrc-48000-55dB"):
        _, st, _ = emulate(emul, name)
        assert st["max_queue"] > 1024 and st["overflow"] > 0, (name, st["max_queue"])
    _, st, _ = emulate(emul, "47999-24")
    assert 0 < st["max_queue"] <= 1024


# ---- the report, restated ----------------------------------------------------------------------------------------------

FPL = 4096 + 4096 // 16
BASE_SMEM = 2 * FPL * 16 + 512 * 16   # k_up2_frac's tile buffers and twiddle tables
QUEUE_BYTES = 1024 * 4


def restated(info, bank_global=False, single=False):
    """Every order2_info field of k_up2_frac from flen, fracs, the ratio and the call's span."""
    flen, fracs, ratio, smax = info["flen"], info["fracs"], info["ratio"], info["span_max"]
    rng = info["_range"]
    nt = -(-rng // smax)
    if nt > 1 and nt & 1:
        nt += 1
    span = ((rng + nt - 1) // nt + 1) & ~1
    r = dict(poly_v2=0, n_tiles=nt, span=span, poly_dir=0, poly_rows_cap=0, poly_row_stride=0, poly_chunks=1, poly_n=0,
             ysh=31, smem_bytes=BASE_SMEM)
    if flen % 2 == 0 and not bank_global:
        fr = ratio - math.floor(ratio)
        outs = 2.0 * span / ratio + 4.0
        stride = 3 * flen + (0 if (6 * flen) % 8 == 4 else 2)
        cap = (224 * 1024 - BASE_SMEM - QUEUE_BYTES) // (stride * 8)
        up, dn = fr * fracs * outs + 4.0, (1.0 - fr) * fracs * outs + 4.0
        chunks = math.ceil(min(up, dn) / cap)
        r["poly_row_stride"] = stride
        if cap >= 8 and chunks <= 4:
            r.update(poly_dir=1 if up < dn else -1, poly_rows_cap=cap, poly_chunks=max(1, chunks),
                     smem_bytes=BASE_SMEM + cap * stride * 8 + QUEUE_BYTES)
            nn = round(ratio)
            if 1 <= nn <= 3 and not single:
                r.update(poly_n=nn, ysh=4)
    return r


SWEEP_PAIRS = [(48000.0, 47999.0), (48000.0, 48001.0), (48000.0, 47700.3), (44100.0, 48001.3), (48000.0, 31999.0),
               (48000.0, 95999.0), (48000.0, 72001.0), (44100.0, 44099.5)]


def _sweep_plans(pkg):
    for at in ROW_ATTENS + [218.0]:
        for s, d in SWEEP_PAIRS:
            for ft in (0, 1):
                yield "%g->%g at %g ft %d" % (s, d, at, ft), pkg.Plan(s, d, 4096, 2.0, at, fasttiming=ft), [1.0]
        for s, d, mt in ((48000.0, 48000.0, 0.01), (44100.0, 88200.0, 0.002), (44100.0, 352800.0, 0.001)):
            fs = [1.0, 1.0 + mt, 1.0 - mt, 1.0 + mt / 3, 1.0 - mt / 7, 1.0 + 1e-6]
            yield "asrc %g->%g at %g" % (s, d, at), pkg.Plan.asrc(s, d, 4096, 2.0, at, mt), fs


@pytest.mark.parametrize("setting", [None, "R8BGPU_BANK_GLOBAL", "R8BGPU_POLY_SINGLE"])
def test_report_is_the_closed_form(pkg, monkeypatch, setting):
    """Attenuation over every R8B_FRACWIN2 row, near-integer and other ratios, trim factors across max_trim on both sides
    of 1 and exactly 1, R8B_FASTTIMING, and spans from a full tile pair down to a few positions."""
    rows, n = set(), 0
    with monkeypatch.context() as mp:
        if setting:
            mp.setenv(setting, "1")
        for what, plan, fs in _sweep_plans(pkg):
            try:
                i = pair_stage(plan)
            except StopIteration:
                continue
            if plan.fused_info(i)["kernel"] != "order2":
                continue
            for f in fs:
                for span in (0, 1, 2, 37, 1000, 5001, 30000, 100001):
                    info = plan.order2_info(i, f, span)
                    info["_range"] = span if span else 2 * info["span_max"]
                    want = restated(info, setting == "R8BGPU_BANK_GLOBAL", setting == "R8BGPU_POLY_SINGLE")
                    got = {k: info[k] for k in want}
                    assert got == want, (what, f, span, got, want)
                    rows.add((info["flen"], info["fracs"]))
                    n += 1
    # every row of the window table (flen 8 .. 30) reached, the 8-row and the 3869-row banks at the two ends
    assert {fl for fl, _ in rows} == set(range(8, 31, 2)), sorted(rows)
    assert (8, 8) in rows and (30, 3869) in rows
    assert n > 1000


def test_poly_v2_setting(pkg, monkeypatch):
    """R8BGPU_POLY_V2 moves calls within 1e-3 of an integer ratio to k_up2_frac2 (k_up2_frac's fields unset), and no
    other call."""
    with monkeypatch.context() as mp:
        mp.setenv("R8BGPU_POLY_V2", "1")
        near = pkg.Plan(48000.0, 47999.0, 4096, 2.0, ATTEN_24)
        far = pkg.Plan(48000.0, 47700.3, 4096, 2.0, ATTEN_24)
        a, b = near.order2_info(pair_stage(near)), far.order2_info(pair_stage(far))
    assert a["poly_v2"] == 1 and a["poly_n"] == 2 and a["poly_dir"] == 0 and a["ysh"] == 31 and a["smem_bytes"] == 0
    assert b["poly_v2"] == 0
    assert near.order2_info(pair_stage(near))["poly_v2"] == 0   # the setting is read when asked


def test_report_refusals(pkg):
    plan = pkg.Plan(48000.0, 47999.0, 4096, 2.0, ATTEN_24)
    i = pair_stage(plan)
    with pytest.raises(pkg.R8bGpuError, match="factor"):
        plan.order2_info(i, 1.0001)
    with pytest.raises(pkg.R8bGpuError, match="order-2"):
        plan.order2_info(i + 1)
    whole = pkg.Plan(44100.0, 96000.0, 4096, 2.0, ATTEN_24)
    with pytest.raises(pkg.R8bGpuError, match="order-2"):
        whole.order2_info(0)
    ap = pkg.Plan.asrc(48000.0, 48000.0, 4096, 2.0, ATTEN_24, 0.001)
    j = pair_stage(ap)
    ap.order2_info(j, 1.001)
    with pytest.raises(pkg.R8bGpuError, match="factor"):
        ap.order2_info(j, 1.0011)
    with pytest.raises(pkg.R8bGpuError, match="span"):
        ap.order2_info(j, 1.0, -1)


# ---- the closed-form inverse of poly_first_k --------------------------------------------------------------------------

# Timing states whose closed-form inverse lands one output off the exact first output, found by searching shifts a few
# ulps around an integer boundary: (ssr, dsr, in_pos_shift (hex), in_counter0, lim, estimate, exact).  They are states a
# stream can be in: the counter re-bases once past 1000 (so a call starts at most there), the shift is a re-based
# fraction in [0, 2), and the first output lies some 10^4 outputs into one call.  The table's streams happen not to land
# within a few ulps of such a boundary.  Without the settle loops of poly_first_k a tile pair would own an output whose
# read position lies in the next pair's tiles (estimate > exact) or leave one to the previous pair (estimate < exact).
FIRST_K_MISSES = [
    (48000.0, 47999.0, "0x1.6604189368000p-1", 930, 62436, 61504, 61505),
    (192000.0, 48001.0, "0x1.194dd2f1a6000p-1", 734, 249489, 61640, 61639),
    (88200.0, 31999.0, "0x1.a6d165c5df600p-1", 43, 108963, 39488, 39489),
    (96000.0, 31999.0, "0x1.499af72014000p-1", 687, 66199, 21378, 21379),
    (192000.0, 31999.0, "0x1.1c66666662400p-1", 582, 85350, 13643, 13642),
    (88200.0, 31999.0, "0x1.b76a178b7b000p-1", 273, 103704, 37350, 37351),
]


def estimate(ssr, dsr, shift, c0, int0, p0, lim, nk):
    """poly_first_k's closed-form estimate alone, the same IEEE operations in the same order."""
    e = math.ceil(float(lim - p0 + int0) * dsr / ssr - shift - float(c0))
    return 0 if e < 0 else min(int(e), nk)


@pytest.mark.parametrize("case", FIRST_K_MISSES, ids=["%g-%g-%d" % (c[0], c[1], c[3]) for c in FIRST_K_MISSES])
def test_first_output_settles_where_the_estimate_misses(emul, case):
    ssr, dsr, shift, c0, lim, est, exact = case
    shift = float.fromhex(shift)
    nk = exact + 50
    assert estimate(ssr, dsr, shift, c0, 0, 0, lim, nk) == est != exact
    scan = C.c_longlong()
    assert emul.o2first_k(ssr, dsr, shift, c0, 0, 0, lim, nk, C.byref(scan)) == scan.value == exact


def test_first_output_is_exact_near_boundaries(emul):
    """Seeded timing states with the shift a few ulps around the value that puts an output exactly on lim, across the
    table's ratios, counters up to 1000 and outputs up to 20000 into a call: poly_first_k equals the scan every time, and the estimate alone misses in both
    directions somewhere in the sweep."""
    rng = np.random.default_rng(11)
    low = high = n = 0
    scan = C.c_longlong()
    for _ in range(400):
        ssr = float(rng.choice([96000.0, 88200.0, 95999.0, 48000.0, 192000.0]))
        dsr = float(rng.choice([47999.0, 48001.0, 47700.3, 96001.0, 31999.0, 44100.0, 48000.0 * (1 + rng.uniform(-0.01, 0.01))]))
        c0 = int(rng.integers(0, 1001))
        k = int(rng.integers(1, 20000))
        lim = int(((float(c0 + k) + 0.5) * ssr) / dsr) + 1
        base = lim * dsr / ssr - c0 - k
        for d in range(-6, 7):
            shift = base + d * math.ulp(float(c0))
            if not 0.0 <= shift < 2.0:
                continue
            nk = k + 50
            got = emul.o2first_k(ssr, dsr, shift, c0, 0, 0, lim, nk, C.byref(scan))
            assert got == scan.value, (ssr, dsr, shift.hex(), c0, lim, got, scan.value)
            e = estimate(ssr, dsr, shift, c0, 0, 0, lim, nk)
            low += e < scan.value
            high += e > scan.value
            n += 1
    assert n > 2000 and low > 0 and high > 0, (n, low, high)
