"""CPU: the geometry space of the unfused BlockConvolvers and the stand-alone interpolators, and a committed table of
plans that covers it.

A BlockConvolver that is not fused with the interpolator behind it runs on k_blockconv<M, UP> (M = 64 .. 8192 for UP 1,
1024 .. 4096 for UP 2, one CTA per tile pair) or, when its filter is too long for those tiles, on the large-tile trio
k_bcl_gather<R0> / k_bcl_conv / k_bcl_scatter<R0> (M = 16384, 32768, 65536; R0 = M / 4096).  The tile follows from the
stage alone: its up-factor (3x runs as a 1x convolution over the zero-stuffed source, src_up 3), its kernel length, and
for power-of-two decimation (block-exact: the tile is the reference's own block, whose Nyquist bin M / (2 D) carries one
real value) the reference's block length.  An interpolator that is not fused runs on k_frac<POLY>, one CTA per `tile`
consecutive outputs, which stages the input window of its outputs in FRAC_CAP doubles of shared memory.  The host
decides all of it in one place each, which Plan.blockconv_info() and Plan.frac_info() report without a device.

walk() plans every pair of RATES (standard and odd rates) at transition bands from 0.5 to 45 % and attenuations from 49
to 218 dB across the design-table rows, with R8B_EXTFFT 0 and 1, plus trim plans at their max_trim.  Every report is
restated here in closed form from StageInfo.  BLOCKCONVS names plans that together reach every class the walk reaches;
tests/test_gpu_blockconv_geometry.py runs each of them against the reference and bit for bit across the exact variants.
If a planner change moves a plan out of a class, test_every_class_is_reached fails here, on a machine without a GPU.

k_frac's window: the kernel traps when a tile's window exceeds FRAC_CAP.  The tile used to stop halving at 32, so a
single stage at more than about 47 input samples per output (Plan.single_stage, for example 4800000 -> 48000, 100:1)
could trap; the tile now goes down to 1 (window = flen).  test_walk_reports_match_restatement and
test_frac_window_fits_single_stages prove the bound on exact positions for every interpolator of the walk and for single
stages up to 1000:1.  With the old floor they fail like this:

    AssertionError: single 100:1 whole lock-step: tile 32 stages up to 3110 samples > FRAC_CAP 1536
    test_frac_tile_at_100_to_1: assert (32 == 8)   (4800000 -> 48000 at 180.15 dB, 24 taps)

What the walk showed when the table was made (about 17000 plans): k_blockconv<64, 1> is reached only below 109 dB (for
example 32000 -> 48000 at 45 % and 49 dB); UP 2 with down 1 only at M = 4096 (shorter 2x kernels run on the fused copy
kernel), and at 1024 and 2048 under R8BGPU_NO_FUSION or R8BGPU_FUSED_V1.  The 3/4 stages (src_up 3, trunc 4) reach
M = 128 .. 8192 and the large path.  Every compiled k_blockconv and k_bcl instantiation is reached.  k_frac runs filter
lengths 8 .. 30 in steps of 2, whole and order-2, and 6 order-2 (third-band, 49 dB).  Behind chains its tile is 1024,
512 or 256 (at most about 6 input samples per output); only single stages reach the smaller tiles, down to 1."""
import math
import os
from fractions import Fraction

import pytest

ATTEN_16IR, ATTEN_16, ATTEN_24, ATTEN_DEF = 109.56, 136.45, 180.15, 206.91
FRAC_CAP = 1536
SMEM_OPT_IN = 227 * 1024                    # per CTA on sm_90; k_blockconv's static shared memory is one double2
BCL_SCRATCH_DEFAULT = 256 << 20

RATES = [7999.0, 8000.0, 11025.0, 16000.0, 22050.0, 32000.0, 44100.0, 44101.0, 47999.0, 48000.0, 64000.0, 88200.0,
         96000.0, 96001.0, 176400.0, 192000.0]
TBS = [0.5, 2.0, 10.0, 30.0, 45.0]
ATTENS = [49.0, 80.0, ATTEN_16IR, ATTEN_16, ATTEN_24, ATTEN_DEF, 218.0]
# the first attenuation of each row of the interpolator design table (filter lengths 8, 10, ..., 30)
ROW_ATTENS = [49.0, 56.0, 82.0, 97.0, 112.0, 126.0, 140.0, 155.0, 169.0, 183.0, 196.0, 210.0, 218.0]
ROW_PAIRS = [(44100.0, 48000.0), (48000.0, 44101.0), (44100.0, 7999.0), (96000.0, 44100.0), (8000.0, 47999.0),
             (192000.0, 47999.0), (32000.0, 11025.0)]

# name -> (src, dst, MaxInLen, TransBand, atten, R8B_EXTFFT, settings); "trim:" names a trim plan at max_trim 0.01;
# "single:" names a one-stage plan: (kind, params, MaxInLen, R8B_EXTFFT, settings), kind 0 BlockConvolver, 1 interpolator
BLOCKCONVS = {
    "16000-7999-45-49": (16000.0, 7999.0, 16384, 45.0, 49.0, 0, {}),            # M 1024; k_frac<true> flen 8
    "32000-48000-45-49": (32000.0, 48000.0, 16384, 45.0, 49.0, 0, {}),          # 3/2 block-exact, M 64
    "64000-48000-45-49": (64000.0, 48000.0, 16384, 45.0, 49.0, 0, {}),          # 3/4 block-exact, M 128
    "32000-48000-30-80": (32000.0, 48000.0, 16384, 30.0, 80.0, 0, {}),          # 3/2 block-exact, M 256
    "16000-8000-10-80": (16000.0, 8000.0, 16384, 10.0, 80.0, 0, {}),            # 1/2 block-exact, M 512
    "64000-48000-0.5-80": (64000.0, 48000.0, 16384, 0.5, 80.0, 0, {}),          # 3/4 block-exact on k_bcl R0 4
    "16000-8000-0.5-16": (16000.0, 8000.0, 16384, 0.5, ATTEN_16, 0, {}),        # 1/2 block-exact on k_bcl R0 4
    "32000-48000-0.5-24": (32000.0, 48000.0, 16384, 0.5, ATTEN_24, 0, {}),      # 3/2 block-exact on k_bcl R0 8
    "8000-48000-0.5-24": (8000.0, 48000.0, 16384, 0.5, ATTEN_24, 0, {}),        # 3x on k_bcl R0 16
    "16000-11025-0.5-24": (16000.0, 11025.0, 16384, 0.5, ATTEN_24, 0, {}),      # 2x on k_bcl R0 16 (zero-stuffed view)
    "47999-8000-0.5-24": (47999.0, 8000.0, 16384, 0.5, ATTEN_24, 0, {}),        # 1x on k_bcl R0 16; k_frac<true> flen 24
    "176400-48000-0.5-default": (176400.0, 48000.0, 16384, 0.5, ATTEN_DEF, 0, {}),  # 1x on k_bcl; k_frac<false> flen 22
    "48000-32000-45-49": (48000.0, 32000.0, 16384, 45.0, 49.0, 0, {}),          # 2/3, UP 2 M 1024
    "48000-32000-10-24": (48000.0, 32000.0, 16384, 10.0, ATTEN_24, 0, {}),      # 2/3, UP 2 M 2048
    "48000-32000-2-80": (48000.0, 32000.0, 16384, 2.0, 80.0, 0, {}),            # 2/3, UP 2 M 4096
    "16000-11025-0.5-16": (16000.0, 11025.0, 16384, 0.5, ATTEN_16, 0, {}),      # 2/1, UP 2 M 4096; k_frac<false> flen 18
    "16000-7999-10-16IR": (16000.0, 7999.0, 16384, 10.0, ATTEN_16IR, 0, {}),    # M 2048; flen 14
    "176400-47999-10-16IR": (176400.0, 47999.0, 16384, 10.0, ATTEN_16IR, 0, {}),  # M 4096; flen 12
    "176400-47999-10-default": (176400.0, 47999.0, 16384, 10.0, ATTEN_DEF, 0, {}),  # M 8192; flen 22
    "176400-48000-0.5-16IR": (176400.0, 48000.0, 16384, 0.5, ATTEN_16IR, 0, {}),  # M 8192; k_frac<false> flen 12
    "7999-11025-45-49": (7999.0, 11025.0, 16384, 45.0, 49.0, 0, {}),            # k_frac tile 1024
    "44100-7999": (44100.0, 7999.0, 8192, 2.0, ATTEN_24, 0, {}),               # the issue's example: 1x, then k_frac<true>
    "47999-7999-45-49": (47999.0, 7999.0, 16384, 45.0, 49.0, 0, {}),            # k_frac<true> flen 6, tile 256
    "16000-7999-45-80": (16000.0, 7999.0, 16384, 45.0, 80.0, 0, {}),            # flen 10
    "16000-7999-45-16": (16000.0, 7999.0, 16384, 45.0, ATTEN_16, 0, {}),        # flen 18
    "16000-7999-45-default": (16000.0, 7999.0, 16384, 45.0, ATTEN_DEF, 0, {}),  # flen 28
    "16000-7999-45-218": (16000.0, 7999.0, 16384, 45.0, 218.0, 0, {}),          # flen 30
    "192000-47999-2-112": (192000.0, 47999.0, 16384, 2.0, 112.0, 0, {}),        # k_frac<true> flen 16
    "192000-47999-2-140": (192000.0, 47999.0, 16384, 2.0, 140.0, 0, {}),        # flen 20
    "192000-47999-2-183": (192000.0, 47999.0, 16384, 2.0, 183.0, 0, {}),        # flen 26
    "32000-11025-45-49": (32000.0, 11025.0, 16384, 45.0, 49.0, 0, {}),          # k_frac<false> flen 8
    "32000-11025-45-80": (32000.0, 11025.0, 16384, 45.0, 80.0, 0, {}),          # flen 10
    "32000-11025-45-16IR": (32000.0, 11025.0, 16384, 45.0, ATTEN_16IR, 0, {}),  # flen 14
    "32000-11025-45-112": (32000.0, 11025.0, 16384, 45.0, 112.0, 0, {}),        # flen 16
    "32000-11025-45-140": (32000.0, 11025.0, 16384, 45.0, 140.0, 0, {}),        # flen 20
    "32000-11025-45-24": (32000.0, 11025.0, 16384, 45.0, ATTEN_24, 0, {}),      # flen 24
    "32000-11025-45-183": (32000.0, 11025.0, 16384, 45.0, 183.0, 0, {}),        # flen 26
    "32000-11025-45-default": (32000.0, 11025.0, 16384, 45.0, ATTEN_DEF, 0, {}),  # flen 28
    "32000-11025-45-218": (32000.0, 11025.0, 16384, 45.0, 218.0, 0, {}),        # flen 30
    "44100-88200-45-nofusion": (44100.0, 88200.0, 16384, 45.0, 49.0, 0, {"R8BGPU_NO_FUSION": "1"}),  # 2/1, UP 2 M 1024
    "44100-88200-2-nofusion": (44100.0, 88200.0, 16384, 2.0, 49.0, 0, {"R8BGPU_NO_FUSION": "1"}),   # 2/1, UP 2 M 2048
    "16000-7999-e1": (16000.0, 7999.0, 16384, 10.0, ATTEN_24, 1, {}),           # R8B_EXTFFT 1
    "trim:44100-7999": (44100.0, 7999.0, 16384, 2.0, ATTEN_24, 0, {}),          # trim plan: ragged tile at 1 - max_trim
    "single:1000-order2": (1, [48000000.0, 48000.0, ATTEN_24, 0], 65536, 0, {}),  # k_frac tile 1
}


def _fft_len(lg, lo, hi, forced=None):
    """choose_fft_log2: the b in [lo, hi] minimising b 2^b / (2^b - 2 lg) with at least 64 valid positions."""
    if forced is not None and lo <= forced <= hi and (1 << forced) - 2 * lg >= 64:
        return forced
    best, cost = -1, 0.0
    for b in range(lo, hi + 1):
        valid = (1 << b) - 2 * lg
        if valid < 64:
            continue
        c = b * (1 << b) / valid
        if best < 0 or c < cost:
            best, cost = b, c
    return best


def is_pow2(n):
    return n > 0 and n & (n - 1) == 0


def restate_bc(s, n_ch=1, forced=None, scratch_cap=BCL_SCRATCH_DEFAULT):
    """The report of an unfused BlockConvolver (k_blockconv or k_bcl) from StageInfo: kernel_len, block_len_bits,
    ref_input_len, up, down and max_out_len."""
    K, up, down = s["kernel_len"], s["up"], s["down"]
    L = (K - 1) // 2
    b2 = 2 << s["block_len_bits"]
    exact = down > 1 and is_pow2(down)
    virt, tup = (up, 1) if up > 2 else (1, up)
    lg = (L + tup - 1) // tup
    large = False
    if exact:
        lg = b2 - s["ref_input_len"] - L           # the reference's PrevInputLen - L
        f = s["block_len_bits"] + 1
        if not ((6 if tup == 1 else 10) <= f <= 13 - (tup - 1)):
            large = True
            assert tup == 1 and 14 <= f <= 16, s
    else:
        f = _fft_len(lg, 10, 13 if tup == 1 else 12, forced)
        if f < 0:
            large = True
            if tup == 2:
                virt, tup, lg = 2, 1, L
            f = _fft_len(lg, 14, 16, forced)
            assert f >= 0, s
    M = 1 << f
    out = dict(kernel="k_bcl" if large else "k_blockconv", fft_log2=f, up=tup, src_up=virt, down=down,
               block_exact=int(exact), trunc=down if exact else 0, nyq_bin=M // (2 * down) if exact else 0, lg=lg,
               adv=s["ref_input_len"] if exact else M - 2 * lg,
               smem_bytes=(4096 + 256 if large else (M + M // 16) * (2 if tup == 2 else 1)) * 16,
               r0=0, scratch_tiles=0, scratch_bytes_per_ch=0, group_ch=0)
    if large:
        span = (s["max_out_len"] + 2) * down + 2
        nt = span // s["ref_input_len"] + 2 if exact else -(-span // (M - 2 * lg))
        nt += nt & 1
        per = nt // 2 * M * 16
        out.update(r0=M // 4096, scratch_tiles=nt, scratch_bytes_per_ch=per, group_ch=max(1, min(n_ch, scratch_cap // per)))
    return out


def stage_rates(plan, src, dst):
    """(input rate, output rate) of every stage: the chain's rate after each stage's up / down."""
    out, r = [], Fraction(src)
    for s in plan.stages():
        up, down = {"hbup": (2, 1), "hbdown": (1, 2)}.get(s["name"], (s["up"], s["down"]))
        if s["name"].startswith("frac"):
            nxt = Fraction(dst)
            for t in plan.stages()[len(out) + 1:]:
                u, d = {"hbup": (2, 1), "hbdown": (1, 2)}.get(t["name"], (t["up"], t["down"]))
                nxt = nxt * d / u
            out.append((r, nxt))
            r = nxt
        else:
            out.append((r, r * up / down))
            r = r * up / down
    return out


def window_bound(s, ssr, dsr, tile):
    """The most input samples a k_frac tile of `tile` outputs stages, on exact positions.  Whole stepping: output j sits
    at floor(j InStep / OutStep), so the max over k0 of floor((k0 + tile - 1) a / b) - floor(k0 a / b) is
    floor(((tile - 1) a + b - gcd(a, b)) / b).  Order 2: the position is ((counter + shift) ssr) / dsr rounded in fp64;
    its integer parts differ by at most floor((tile - 1) ssr / dsr + rounding) + 1 (positions below 2^31 * ratio)."""
    if s["name"] == "frac_whole":
        a, b = s["in_step"], s["out_step"]
        return ((tile - 1) * a + b - math.gcd(a, b)) // b
    r = Fraction(ssr) / Fraction(dsr)
    slack = r * Fraction(1, 1 << 19)
    return math.floor((tile - 1) * r + slack) + 1


def frac_tile(r, flen):
    tile = 1024
    while tile > 1 and tile * r + flen + 4 > FRAC_CAP:
        tile >>= 1
    return tile


def frac_window(tile, r, flen):
    return math.floor((tile - 1) * r) + 2 + flen


def make_plan(pkg, name, entry=None):
    e = BLOCKCONVS[name] if entry is None else entry
    if name.startswith("single:"):
        kind, params, m, ext, _ = e
        return pkg.Plan.single_stage(kind, params, m, extfft=ext)
    src, dst, m, tb, at, ext, _ = e
    if name.startswith("trim:"):
        return pkg.Plan.trim(src, dst, m, tb, at, 0.01, extfft=ext)
    return pkg.Plan(src, dst, m, tb, at, extfft=ext)


def rates_of(name, plan):
    """(src, dst) of the chain; for a single stage its own rates (the interpolator's params), or 1, 1."""
    e = BLOCKCONVS[name]
    if name.startswith("single:"):
        return (e[1][0], e[1][1]) if e[0] == 1 else (1.0, 1.0)
    return e[0], e[1]


def settings_of(name):
    return BLOCKCONVS[name][-1]


# ---- the walk --------------------------------------------------------------------------------------------------------

def _walk_entries():
    for ext in (0, 1):
        for src in RATES:
            for dst in RATES:
                if src == dst:
                    continue
                for tb in TBS:
                    for at in ATTENS:
                        yield ("%g-%g tb%g a%g e%d" % (src, dst, tb, at, ext), (src, dst, 4096, tb, at, ext, {}))
    for src, dst in ROW_PAIRS:
        for at in ROW_ATTENS:
            yield ("%g-%g tb2 a%g e0" % (src, dst, at), (src, dst, 4096, 2.0, at, 0, {}))
            yield ("trim:%g-%g a%g" % (src, dst, at), (src, dst, 4096, 2.0, at, 0, {}))


_WALK = None


def walk(pkg):
    """[(name, plan, entry)] of every plan of the walk the planner accepts."""
    global _WALK
    if _WALK is None:
        _WALK = []
        for name, e in _walk_entries():
            src, dst, m, tb, at, ext, _ = e
            try:
                plan = (pkg.Plan.trim(src, dst, m, tb, at, 0.01, extfft=ext) if name.startswith("trim:")
                        else pkg.Plan(src, dst, m, tb, at, extfft=ext))
            except pkg.R8bGpuError:
                continue
            _WALK.append((name, plan, e))
    return _WALK


def classes_of(plan, n_ch=1):
    """The classes a plan's unfused BlockConvolvers and interpolators reach."""
    out = set()
    st = plan.stages()
    for i, s in enumerate(st):
        if s["name"] == "blockconv":
            info = plan.blockconv_info(i, n_ch)
            if info["kernel"] == "k_blockconv":
                out.add("k_blockconv M=%d up=%d" % (1 << info["fft_log2"], info["up"]))
                out.add("src_up %d" % info["src_up"])
                out.add("down %d" % info["down"])
                out.add("trunc %d" % info["trunc"])
                if info["up"] == 2:
                    out.add("k_blockconv M=%d up=2 down=%d" % (1 << info["fft_log2"], info["down"]))
            elif info["kernel"] == "k_bcl":
                out.add("k_bcl R0=%d" % info["r0"])
                out.add("k_bcl src_up=%d %s" % (info["src_up"], "block-exact" if info["block_exact"] else "plain"))
                out.add("down %d" % info["down"])
                out.add("trunc %d" % info["trunc"])
        elif s["name"].startswith("frac"):
            info = plan.frac_info(i)
            poly = int(s["name"] == "frac_poly")
            if info["kernel"] != "fused":
                out.add("k_frac poly=%d flen=%d" % (poly, info["flen"]))
            out.add("k_frac tile %d" % info["tile"])
            out.add("k_frac tile %d" % info["tile_ragged"])
    return out


# every class BLOCKCONVS must reach (the walk reaches each; test_walk_reaches_the_classes checks that it still does)
CLASSES = (["k_blockconv M=%d up=1" % (1 << b) for b in range(6, 14)] +
           ["k_blockconv M=%d up=2" % (1 << b) for b in range(10, 13)] +
           ["k_blockconv M=%d up=2 down=%d" % (1 << b, d) for b in range(10, 13) for d in (1, 3)] +
           ["src_up 1", "src_up 3", "down 1", "down 2", "down 3", "down 4", "trunc 0", "trunc 2", "trunc 4"] +
           ["k_bcl R0=%d" % r for r in (4, 8, 16)] +
           ["k_bcl src_up=%d %s" % (v, k) for v in (1, 2, 3) for k in ("plain", "block-exact") if (v, k) != (2, "block-exact")] +
           ["k_frac poly=%d flen=%d" % (p, f) for p in (0, 1) for f in range(8, 32, 2)] + ["k_frac poly=1 flen=6"] +
           ["k_frac tile 1024", "k_frac tile 1"])
# reached only through R8BGPU_NO_FUSION / R8BGPU_FUSED_V1 (shorter 2x kernels run on the fused copy kernel) or a single
# stage (the walk's chains read at most about 6 input samples per output)
BY_SETTINGS = {"k_blockconv M=1024 up=2 down=1", "k_blockconv M=2048 up=2 down=1", "k_frac tile 1"}


@pytest.fixture(scope="module")
def reports(pkg):
    out = {}
    for name in BLOCKCONVS:
        with pytest.MonkeyPatch.context() as mp:
            for k, v in settings_of(name).items():
                mp.setenv(k, v)
            plan = make_plan(pkg, name)
            out[name] = (plan, classes_of(plan, 3))
    return out


def test_every_class_is_reached(reports):
    reached = {}
    for name, (_, cls) in reports.items():
        for c in cls:
            reached.setdefault(c, []).append(name)
    print("\nclass -> plans")
    for c in CLASSES:
        print("  %-34s %s" % (c, ", ".join(reached.get(c, ["-"]))[:100]))
    missing = [c for c in CLASSES if c not in reached]
    assert not missing, missing


def test_walk_reaches_the_classes(pkg):
    """The classes are the walk's (plus the settings and single stages the table uses for the few it cannot reach): a
    class no plan of the walk reaches any more, or a new one it reaches, shows here."""
    reached = set()
    for _, plan, _ in walk(pkg):
        reached |= classes_of(plan)
    known = set(CLASSES)
    new = sorted(c for c in reached - known if not c.startswith("k_frac tile"))
    assert not new, "classes the walk reaches that CLASSES does not list: %s" % new
    assert not reached & BY_SETTINGS, sorted(reached & BY_SETTINGS)
    lost = sorted(known - reached - BY_SETTINGS)
    print("\n%d walked plans; k_frac tiles %s; reached only through settings or single stages: %s" % (
        len(walk(pkg)), sorted(c for c in reached if c.startswith("k_frac tile")), sorted(known - reached)))
    assert not lost, lost


@pytest.mark.parametrize("name", list(BLOCKCONVS))
def test_table_report_matches_restatement(pkg, reports, name):
    plan, _ = reports[name]
    with pytest.MonkeyPatch.context() as mp:
        for k, v in settings_of(name).items():
            mp.setenv(k, v)
        check_plan(pkg, plan, rates_of(name, plan), n_ch=3)


def check_plan(pkg, plan, rates, n_ch=1, forced=None, scratch_cap=BCL_SCRATCH_DEFAULT):
    """Every unfused BlockConvolver report equals its restatement; every interpolator's tiles fit FRAC_CAP on exact
    positions.  Returns the number of stages checked."""
    st = plan.stages()
    sr = stage_rates(plan, *rates) if rates[0] != 1.0 or len(st) > 1 else None
    n = 0
    for i, s in enumerate(st):
        if s["name"] == "blockconv":
            info = plan.blockconv_info(i, n_ch)
            if info["kernel"] in ("fused", "f2-copy"):
                assert info["fft_log2"] == 12, info
                continue
            want = restate_bc(s, n_ch, forced, scratch_cap)
            got = {k: info[k] for k in want}
            assert got == want, (i, s, got, want)
            assert info["smem_bytes"] + 16 <= SMEM_OPT_IN
            n += 1
        elif s["name"].startswith("frac"):
            check_frac(plan, i, s, sr[i] if sr else None)
            n += 1
    return n


def check_frac(plan, i, s, rates, what=""):
    info = plan.frac_info(i)
    flen = info["flen"]
    assert info["frac_cap"] == FRAC_CAP and info["fll"] == flen // 2 - 1
    assert info["fracs"] == (s["fracs"] if s["name"] == "frac_poly" else 0)
    if s["name"] == "frac_whole":
        r = Fraction(s["in_step"], s["out_step"])
        ssr, dsr = r, 1
    else:
        ssr, dsr = rates
        r = Fraction(ssr) / Fraction(dsr)
    trim = plan.max_trim
    # a trim plan's ragged calls read at most ssr / (dsr (1 - max_trim)) input samples per output (its lock-step calls,
    # at one common factor, at most as many)
    r_rag = r / (1 - Fraction(trim)) if trim else r
    for tile, window, ratio, kind in ((info["tile"], info["window"], r, "lock-step"),
                                      (info["tile_ragged"], info["window_ragged"], r_rag, "ragged")):
        assert is_pow2(tile) and tile <= 1024
        exact = window_bound(s, ssr, dsr if kind == "lock-step" or not trim else Fraction(dsr) * (1 - Fraction(trim)), tile)
        assert exact + flen <= window, (what, kind, tile, exact, window)
        assert window <= FRAC_CAP, "%s %s: tile %d stages up to %d samples > FRAC_CAP %d" % (what, kind, tile, window, FRAC_CAP)
        if "R8BGPU_FRAC_TILE" not in os.environ:
            assert tile == frac_tile(float(ratio), flen), (what, kind, tile, float(ratio))
    if trim:
        assert info["tile_ragged"] <= info["tile"]


def test_walk_reports_match_restatement(pkg):
    n = 0
    for name, plan, e in walk(pkg):
        n += check_plan(pkg, plan, (e[0], e[1]))
    print("\n%d stages restated" % n)
    assert n > 1000


SINGLE_RATIOS = [2, 3, 4, 7.5, 10, 16, 32, 47, 48, 64, 100, 128, 250, 500, 750, 754, 1000]


@pytest.mark.parametrize("ratio", SINGLE_RATIOS)
def test_frac_window_fits_single_stages(pkg, ratio):
    """Single-stage interpolators up to 1000:1, whole-stepping and order-2, at each attenuation: the window of both
    tiles fits FRAC_CAP on exact positions."""
    n = 0
    for at in (49.0, ATTEN_16IR, ATTEN_24, 218.0):
        for src, dst in ((48000.0 * ratio, 48000.0), (48000.0 * ratio + 7.0, 48000.0)):
            plan = pkg.Plan.single_stage(1, [src, dst, at, 0], 1024)
            s = plan.stages()[0]
            check_frac(plan, 0, s, (src, dst), "single %g:1 %s" % (src / dst, s["name"][5:]))
            n += 1
    assert n == 8


def test_frac_tile_at_100_to_1(pkg):
    """The configuration that used to trap: 4800000 -> 48000 whole-stepping (in_step 100, out_step 1, 24 taps)."""
    plan = pkg.Plan.single_stage(1, [4800000.0, 48000.0, ATTEN_24, 0], 1024)
    s = plan.stages()[0]
    assert (s["name"], s["in_step"], s["out_step"], s["kernel_len"]) == ("frac_whole", 100, 1, 24), s
    info = plan.frac_info(0)
    assert (info["flen"], info["tile"], info["tile_ragged"]) == (24, 8, 8) and info["window"] <= FRAC_CAP, info


# ---- settings ----------------------------------------------------------------------------------------------------------

def _unfused_bcs(pkg):
    for name, plan, e in walk(pkg):
        for i, s in enumerate(plan.stages()):
            if s["name"] == "blockconv" and plan.blockconv_info(i)["kernel"] in ("k_blockconv", "k_bcl"):
                yield name, plan, i, s


def test_fft_log2_setting_moves_only_the_tile(pkg, monkeypatch):
    """R8BGPU_FFT_LOG2 = b takes b where it is in the stage's range with 64 valid positions, and changes nothing else."""
    seen = {}
    for name, plan, i, s in _unfused_bcs(pkg):
        d = plan.blockconv_info(i)
        if d["block_exact"]:
            continue
        key = (d["kernel"], d["up"], d["lg"])
        if key in seen:
            continue
        seen[key] = 1
        for b in range(6, 18):
            monkeypatch.setenv("R8BGPU_FFT_LOG2", str(b))
            got = plan.blockconv_info(i)
            monkeypatch.delenv("R8BGPU_FFT_LOG2")
            want = restate_bc(s, 1, b)
            assert {k: got[k] for k in want} == want, (name, b, got, want)
            lo, hi = (10, 13 if d["up"] == 1 else 12) if d["kernel"] == "k_blockconv" else (14, 16)
            assert (got["fft_log2"] == b) == (lo <= b <= hi and (1 << b) - 2 * d["lg"] >= 64), (name, b, got)
    assert len(seen) > 20


def test_block_exact_ignores_fft_log2(pkg, monkeypatch):
    for name, plan, i, s in _unfused_bcs(pkg):
        d = plan.blockconv_info(i)
        if d["block_exact"]:
            monkeypatch.setenv("R8BGPU_FFT_LOG2", "11")
            assert plan.blockconv_info(i) == d, name
            monkeypatch.delenv("R8BGPU_FFT_LOG2")


def test_fusion_settings(pkg, monkeypatch):
    """R8BGPU_NO_FUSION and R8BGPU_FUSED_V1 move fused and copy stages to k_blockconv with their own tile; R8BGPU_NO_FUSION
    also leaves each interpolator on k_frac."""
    moved = {"NO_FUSION": 0, "FUSED_V1": 0}
    for name, plan, e in walk(pkg)[::7]:
        st = plan.stages()
        base = {i: plan.blockconv_info(i) for i, s in enumerate(st) if s["name"] == "blockconv"}
        for key in moved:
            monkeypatch.setenv("R8BGPU_" + key, "1")
            for i, d in base.items():
                got = plan.blockconv_info(i)
                if d["kernel"] in ("k_blockconv", "k_bcl"):
                    assert got == d, (name, key)
                elif key == "NO_FUSION" or d["kernel"] == "f2-copy" or got["kernel"] != "fused":
                    assert got["kernel"] in ("k_blockconv", "k_bcl"), (name, key, got)
                    want = restate_bc(st[i], 1)
                    assert {k: got[k] for k in want} == want, (name, key)
                    moved[key] += 1
                if key == "NO_FUSION" and i + 1 < len(st) and st[i + 1]["name"].startswith("frac"):
                    assert plan.frac_info(i + 1)["kernel"] != "fused"
            monkeypatch.delenv("R8BGPU_" + key)
    assert moved["NO_FUSION"] > 0 and moved["FUSED_V1"] > 0, moved


def test_bcl_scratch_setting(pkg, monkeypatch):
    """R8BGPU_BCL_SCRATCH_MB sets the channels per launch group: as many as the cap holds, at least one."""
    n = 0
    for name, plan, i, s in _unfused_bcs(pkg):
        d = plan.blockconv_info(i, 1000)
        if d["kernel"] != "k_bcl":
            continue
        assert d["group_ch"] == max(1, min(1000, BCL_SCRATCH_DEFAULT // d["scratch_bytes_per_ch"]))
        for mb in (1, 64, 4096):
            monkeypatch.setenv("R8BGPU_BCL_SCRATCH_MB", str(mb))
            got = plan.blockconv_info(i, 1000)
            monkeypatch.delenv("R8BGPU_BCL_SCRATCH_MB")
            assert got == dict(d, group_ch=max(1, min(1000, (mb << 20) // d["scratch_bytes_per_ch"])))
            n += 1
        assert plan.blockconv_info(i, 3)["group_ch"] == min(3, d["group_ch"]) or d["group_ch"] < 3
    assert n > 0


def test_frac_tile_setting(pkg, monkeypatch):
    """R8BGPU_FRAC_TILE: every power of two whose worst window fits is taken for both kinds of call; a larger one, or a
    value that is not a power of two from 1 to 1024, is refused with a message."""
    plan = pkg.Plan.single_stage(1, [4800000.0, 48000.0, ATTEN_24, 0], 1024)
    flen = plan.frac_info(0)["flen"]
    for t in [1 << k for k in range(11)]:
        monkeypatch.setenv("R8BGPU_FRAC_TILE", str(t))
        if frac_window(t, 100.0, flen) <= FRAC_CAP:
            info = plan.frac_info(0)
            assert info["tile"] == info["tile_ragged"] == t and info["window"] <= FRAC_CAP
        else:
            with pytest.raises(pkg.R8bGpuError, match="R8BGPU_FRAC_TILE=%d: stage 0" % t):
                plan.frac_info(0)
    for bad in ("0", "3", "2048", "-4"):
        monkeypatch.setenv("R8BGPU_FRAC_TILE", bad)
        with pytest.raises(pkg.R8bGpuError, match="power of two from 1 to 1024"):
            plan.frac_info(0)
