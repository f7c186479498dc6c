"""CPU: the geometry space of the half-band cascades, and a committed table of plans that covers it.

Whole power-of-two up and down chains run their half-band stages in k_hbup_cascade / k_hbdown_cascade: up to 6
consecutive stages of one direction in one kernel, every intermediate rate in shared memory.  Each stage takes its taps
from one of the steepness families of the plain or third-band table (an up cascade's stage k from family k, a down
cascade's from families c-1 .. 0), and the attenuation picks the row.  The tap vector decides everything else: the
instantiation of each stage pass (hb_stage<T>, T = 1 .. 14, or hb_stage_last2<T1, T2> for the last two stages of an up
cascade, T1 <= 6, T2 <= 4), the halos, the number of shared-memory buffers and the tile width.  The host decides all of
it in one place, which Plan.cascade_info() reports without a device.

walk() steps the attenuation from 49 dB across every row boundary the planner selects (the next one is just above the
smallest selected-row attenuation the plan's stage info reports) up to 218 dB, for chains of 2 .. 7 half-band stages,
plain and third-band, up and down.  That reaches 518 distinct tap vectors.  CASCADES names plans that together reach
every class below; tests/test_gpu_hb_geometry.py runs each of them against the reference, and every walked vector bit
for bit against one kernel per stage.  If a planner change moves a plan out of a class, test_every_class_is_reached
fails here, on a machine without a GPU, instead of the coverage vanishing.

What the walk showed when the table was made: the up cascades reach hb_stage<T> on a non-last stage for every T from 1
to 14, an unfused last stage for T = 4 .. 8, and 13 of the 24 instantiated hb_stage_last2 pairs.  No plan reaches the
other 11: <1,2> <1,3> <1,4> <2,3> <2,4> <3,1> <3,4> <4,1> <5,1> <6,1> <6,2>.  The default budget gives down cascades a tile width of 1024, 256, 128 and 64 outputs for 2 .. 5 stages and 32, 16 or 8 for 6."""
import pytest

ATTEN_16, ATTEN_24 = 136.45, 180.15
BASE = 44100.0
UP_SMEM_OPT_IN, DOWN_SMEM_OPT_IN = 220 * 1024, 227 * 1024     # what the launchers opt the two kernels in to
UP_BUDGET, DOWN_BUDGET = 7000, 6400                           # doubles per CTA when no setting is given
HB = ("hbup", "hbdown")


def chain_rates(direction, third, c):
    """(src, dst) of the whole chain with c half-band stages: up 2^c (or 3 * 2^c) behind a 2x (3x) BlockConvolver, down c
    half-band stages in front of a 1/2 (1/3) BlockConvolver."""
    f = (3 if third else 2) << c
    return (BASE, BASE * f) if direction == "up" else (BASE * f, BASE)


def max_in(direction, c):
    return 1024 if direction == "up" else 1024 << c


SHAPES = [(d, t, c) for d in ("up", "down") for t in (0, 1) for c in range(2, 8)]

# name -> (src, dst, MaxInLen, atten); the comments give the half-band taps in chain order
CASCADES = {
    "single-hbup": (BASE, 4 * BASE, 4096, ATTEN_24),                 # 11: one k_hbup
    "single-hbdown": (4 * BASE, BASE, 4096, ATTEN_24),               # 11: one k_hbdown
    "44100-2822400": (BASE, 64 * BASE, 1024, ATTEN_24),              # 11/6/5/4/3
    "2822400-44100": (64 * BASE, BASE, 32768, ATTEN_24),             # 3/4/5/6/11
    "48000-2822400": (48000.0, 2822400.0, 1024, ATTEN_24),           # 11/6/5/4/3 behind the interpolator
    "11025-2822400": (BASE / 4, 64 * BASE, 1024, ATTEN_24),          # 11/6/5/4/3/3 + 2: the cascade writes a ring
    "11289600-44100": (256 * BASE, BASE, 131072, ATTEN_24),          # 2/3/3/4/5/6 + 11: feeding k_hbdown
    "up2-49": (BASE, 8 * BASE, 1024, 49.0),                          # 4/2
    "up2-54.52": (BASE, 8 * BASE, 1024, 54.52),                      # 5/2
    "up2-56.61": (BASE, 8 * BASE, 1024, 56.61),                      # 5/3
    "up2-66.31": (BASE, 8 * BASE, 1024, 66.31),                      # 6/3
    "up2-83.03": (BASE, 8 * BASE, 1024, 83.03),                      # 6/4
    "up2-121.01": (BASE, 8 * BASE, 1024, 121.01),                    # 9/4: unfused last stage
    "up2-152.45": (BASE, 8 * BASE, 1024, 152.45),                    # 11/6
    "up2-181.26": (BASE, 8 * BASE, 1024, 181.26),                    # 11/7
    "up2-215.14": (BASE, 8 * BASE, 1024, 215.14),                    # 14/8
    "up3-56.61": (BASE, 16 * BASE, 1024, 56.61),                     # 5/3/2
    "up3-183.8": (BASE, 16 * BASE, 1024, 183.8),                     # 12/7/5
    "up4-49": (BASE, 32 * BASE, 1024, 49.0),                         # 4/2/2/1
    "up4-113.22": (BASE, 32 * BASE, 1024, 113.22),                   # 8/4/3/3
    "up4-136.7": (BASE, 32 * BASE, 1024, 136.7),                     # 10/5/4/3
    "up5-209.95": (BASE, 64 * BASE, 1024, 209.95),                   # 13/8/5/4/4
    "up6-49": (BASE, 128 * BASE, 1024, 49.0),                        # 4/2/2/1/1/1
    "up-third2-24": (BASE, 12 * BASE, 1024, ATTEN_24),              # 8/5
    "up-third4-24": (BASE, 48 * BASE, 1024, ATTEN_24),              # 8/5/4/3
    "up-third7-115.78": (BASE, 384 * BASE, 1024, 115.78),            # 5/4/3/2/2/2 + 2
    "down3-49": (16 * BASE, BASE, 8192, 49.0),                       # 2/2/4
    "down4-49": (32 * BASE, BASE, 16384, 49.0),                      # 1/2/2/4
    "down5-49": (64 * BASE, BASE, 32768, 49.0),                      # 1/1/2/2/4
    "down6-105.29": (128 * BASE, BASE, 65536, 105.29),               # 2/2/2/3/4/8
    "down6-209.95": (128 * BASE, BASE, 65536, 209.95),               # 3/4/4/5/8/13
    "down7-49": (256 * BASE, BASE, 131072, 49.0),                    # 1/1/1/1/2/2 + 4
    "down-third2-49": (12 * BASE, BASE, 4096, 49.0),                 # 2/3
    "down-third4-24": (48 * BASE, BASE, 32768, ATTEN_24),           # 3/4/5/8
    "down-third6-24": (192 * BASE, BASE, 131072, ATTEN_24),          # 3/3/3/4/5/8
}


def hb_stages(plan):
    return [i for i, s in enumerate(plan.stages()) if s["name"] in HB]


def walk(pkg, src, dst, m):
    """{tap vector of the plan's half-band stages: (atten, plan)} over the attenuations 49 .. 218 dB, stepping just past
    the smallest selected-row attenuation at or above the current one."""
    out, a = {}, 49.0
    while True:
        plan = pkg.Plan(src, dst, m, 2.0, a)
        st = plan.stages()
        hb = [s for s in st if s["name"] in HB]
        out.setdefault(tuple(s["kernel_len"] for s in hb), (a, plan))
        nxt = [s["atten"] for s in hb if s["atten"] >= a]
        if not nxt or min(nxt) + 1e-6 > 218.0:
            return out
        a = min(nxt) + 1e-6


@pytest.fixture(scope="session")
def walked(pkg):
    """[(direction, third, c, taps, atten, plan)] over SHAPES."""
    out = []
    for d, t, c in SHAPES:
        src, dst = chain_rates(d, t, c)
        for taps, (a, plan) in walk(pkg, src, dst, max_in(d, c)).items():
            out.append((d, t, c, taps, a, plan))
    return out


def runs(plan):
    """[(first stage, Plan.cascade_info)] of every kernel that runs half-band stages, and the reports of the stages
    inside cascades."""
    out, inside = [], []
    for i in hb_stages(plan):
        info = plan.cascade_info(i)
        (inside if info["kind"] == "inside" else out).append((i, info))
    return out, inside


# ---- the report's numbers, restated from the stage taps --------------------------------------------------------------

def up_halos(taps):
    """Stream k of an up-cascade tile covering input [A, A + w) spans [2^k A - lo[k], 2^k (A + w) + hi[k]): what stage k's
    taps need to produce stream k + 1's span, from the last stage backwards (s_{k+1}[2n+1] reads s_k[n-T+1 .. n+T])."""
    c = len(taps)
    lo, hi = [0] * (c + 1), [0] * (c + 1)
    for k in range(c - 1, -1, -1):
        lo[k] = -(-lo[k + 1] // 2) + taps[k] - 1
        hi[k] = (hi[k + 1] - 1) // 2 + taps[k] + 1
    return tuple(lo), tuple(hi)


def last2_ok(t1, t2):
    return 1 <= t1 <= 6 and 1 <= t2 <= 4


def up_plan(taps, budget=UP_BUDGET, last2=True):
    """(fuse_last2, n_buffers, w, smem bytes) of an up cascade: w is the widest multiple of 32 (32 .. 1024) whose
    buffers -- 5/4-skewed, w 2^k samples plus halos and 8 of slack each -- fit 4/5 of the budget."""
    c = len(taps)
    lo, hi = up_halos(taps)
    fuse = int(last2 and last2_ok(taps[-2], taps[-1]))
    nbuf = c - fuse
    halo = sum(lo[k] + hi[k] + 8 for k in range(nbuf))
    w = int((budget * 4 // 5 - halo) / ((1 << nbuf) - 1)) & ~31
    w = min(max(w, 32), 1024)
    off = 0
    for k in range(nbuf):
        off += (((w << k) + lo[k] + hi[k] + 8) * 5 + 3) // 4 + 2
        off = (off + 1) & ~1
    return fuse, nbuf, w, 8 * off


def down_back(taps):
    """Stream s of a down cascade reaches back[s] samples either side of 2^(n-s) m for final output m:
    out[m] = x[2m] + sum_k f[k] (x[2m+1+2k] + x[2m-1-2k]) reaches 2T - 1."""
    n = len(taps)
    b = [0] * (n + 1)
    for s in range(n - 1, -1, -1):
        b[s] = 2 * b[s + 1] + 2 * taps[s] - 1
    return tuple(b)


def down_plan(taps, budget=DOWN_BUDGET):
    """(w, smem bytes) of a down cascade: the widest power of two 8 .. 1024 whose split even/odd buffers fit the budget;
    (0, 0) when none does."""
    n, b = len(taps), down_back(taps)

    def doubles(w):
        return sum(2 * ((((w - 1) << (n - s)) + 2 * b[s] + 1) // 2 + 2) for s in range(n))
    fit = [w for w in (8 << j for j in range(8)) if doubles(w) <= budget]
    return (fit[-1], 8 * doubles(fit[-1])) if fit else (0, 0)


def check_run(plan, i, info, up_budget=UP_BUDGET, down_budget=DOWN_BUDGET, last2=True):
    st = plan.stages()
    taps = info["ntaps"]
    c = info["n_stages"]
    assert info["first"] == i and taps == tuple(st[i + k]["kernel_len"] for k in range(c)), info
    assert all(st[i + k]["name"] == st[i]["name"] for k in range(c))
    assert info["writes_ring"] == (i + c < len(st))
    if info["kind"] == "single":
        assert c == 1 and info["w"] == 0 and info["smem_bytes"] == 0
        return
    if info["kind"] == "up-cascade":
        assert (info["lo_off"], info["hi_off"]) == up_halos(taps), info
        assert (info["fuse_last2"], info["n_buffers"], info["w"], info["smem_bytes"]) == up_plan(taps, up_budget, last2)
        assert info["back"] == (0,) * (c + 1)
    else:
        assert info["kind"] == "down-cascade"
        assert info["back"] == down_back(taps) and (info["w"], info["smem_bytes"]) == down_plan(taps, down_budget)
        assert info["n_buffers"] == c and not info["fuse_last2"]
        assert info["lo_off"] == info["hi_off"] == (0,) * (c + 1)


def expected_runs(plan):
    """[(first stage, n_stages)]: runs of half-band stages of one direction, cut into kernels of at most 6."""
    st, out = plan.stages(), []
    i = 0
    while i < len(st):
        if st[i]["name"] not in HB:
            i += 1
            continue
        c = 1
        while i + c < len(st) and st[i + c]["name"] == st[i]["name"] and c < 6:
            c += 1
        out.append((i, c))
        i += c
    return out


# ---- classes ------------------------------------------------------------------------------------------------------------

def classes_of(plan):
    st = plan.stages()
    table = "third" if "third=1" in plan.describe() else "plain"     # (the HBUp / HBDown lines)
    out = set()
    for i, info in runs(plan)[0]:
        taps, c = info["ntaps"], info["n_stages"]
        if info["kind"] == "single":
            out.add("single k_%s" % st[i]["name"])
            continue
        if info["kind"] == "up-cascade":
            out.add("up, %d stages" % c)
            out.add("up, %s table" % table)
            for t in taps[:c - 1 - info["fuse_last2"]]:
                out.add("up, hb_stage<%d> on a non-last stage" % t)
            if info["fuse_last2"]:
                out.add("up, last2 <%d,%d>" % taps[-2:])
            else:
                out.add("up, unfused last stage T=%d" % taps[-1])
            if info["writes_ring"]:
                out.add("up, cascade writes a ring")
            if any(s["name"].startswith("frac") for s in st[:i]):
                out.add("up, cascade behind the interpolator")
        else:
            out.add("down, %d stages" % c)
            out.add("down, %s table" % table)
            out.add("down, w=%d" % info["w"])
            if c == 6 and st[i + 6]["name"] == "hbdown":
                out.add("down, 6-stage cascade feeding k_hbdown")
    return out


def expected_classes(walked_plans):
    """Every class the walk reaches, plus the path-3 one (the walk's chains have no interpolator)."""
    out = {"up, cascade behind the interpolator", "single k_hbup", "single k_hbdown"}
    for plan in walked_plans:
        out |= classes_of(plan)
    return out


def make_plan(pkg, name):
    src, dst, m, a = CASCADES[name]
    return pkg.Plan(src, dst, m, 2.0, a)


# ---- tests ----------------------------------------------------------------------------------------------------------------

def test_walk_reaches_the_space(pkg, walked):
    """The space itself: 518 tap vectors, every hb_stage<T>, the unfused last stages and the last2 pairs the docstring
    names, 2 .. 6-stage cascades of both tables and directions, and the down tile widths."""
    assert len({(d, t, taps) for d, t, c, taps, a, p in walked}) == 518
    cls = expected_classes([w[-1] for w in walked])
    assert {"up, hb_stage<%d> on a non-last stage" % t for t in range(1, 15)} <= cls
    assert {x for x in cls if x.startswith("up, unfused")} == {"up, unfused last stage T=%d" % t for t in range(4, 9)}
    pairs = {x for x in cls if x.startswith("up, last2")}
    unreached = {(1, 2), (1, 3), (1, 4), (2, 3), (2, 4), (3, 1), (3, 4), (4, 1), (5, 1), (6, 1), (6, 2)}
    assert pairs == {"up, last2 <%d,%d>" % (a, b) for a in range(1, 7) for b in range(1, 5) if (a, b) not in unreached}
    assert {x for x in cls if x.startswith("down, w=")} == {"down, w=%d" % w for w in (8, 16, 32, 64, 128, 256, 1024)}
    for d in ("up", "down"):
        assert {"%s, %d stages" % (d, c) for c in range(2, 7)} | {"%s, plain table" % d, "%s, third table" % d} <= cls


def test_every_class_is_reached(pkg, walked):
    want = expected_classes([w[-1] for w in walked])
    reached = {}
    for name in CASCADES:
        for c in classes_of(make_plan(pkg, name)):
            reached.setdefault(c, []).append(name)
    print("\nclass -> plans")
    for c in sorted(want):
        print("  %-44s %s" % (c, ", ".join(reached.get(c, ["-"]))))
    missing = sorted(c for c in want if c not in reached)
    assert not missing, missing


def test_report_restated_for_every_walked_vector(pkg, walked):
    """Every field of every report, from the stage taps; the bytes fit each kernel's opt-in limit; every down run of 2 or
    more stages gets a cascade; a stage inside a cascade names its first stage."""
    for d, t, c, taps, a, plan in walked:
        got, inside = runs(plan)
        assert [(i, info["n_stages"]) for i, info in got] == expected_runs(plan), (d, t, taps)
        for i, info in got:
            check_run(plan, i, info)
            assert info["kind"] == ("single" if info["n_stages"] == 1 else "%s-cascade" % d), (d, t, taps, info)
            lim = UP_SMEM_OPT_IN if d == "up" else DOWN_SMEM_OPT_IN
            assert info["smem_bytes"] <= lim, (taps, info)
        firsts = {i: info["n_stages"] for i, info in got}
        for j, info in inside:
            assert info["first"] in firsts and info["first"] < j < info["first"] + firsts[info["first"]]
            assert info["n_stages"] == 0 and info["w"] == 0


@pytest.mark.parametrize("env", [{"R8BGPU_NO_HB_CASCADE": "1"}, {"R8BGPU_NO_FUSION": "1"}])
def test_no_cascade_settings(pkg, walked, monkeypatch, env):
    """One k_hbup / k_hbdown per stage."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    for d, t, c, taps, a, plan in walked[::7]:
        got, inside = runs(plan)
        assert not inside and len(got) == c
        for i, info in got:
            check_run(plan, i, info)
            assert info["kind"] == "single"


def test_settings_move_the_tile_plans(pkg, walked, monkeypatch):
    """R8BGPU_HB_NO_LAST2 unfuses the last two stages; the two budgets move w (and only w, buffers and bytes) as the
    closed forms say; a down budget too small for any tile falls back to one kernel per stage."""
    moved = {"last2": 0, "up w": 0, "down w": 0}
    for env, kw in (({"R8BGPU_HB_NO_LAST2": "1"}, {"last2": False}),
                    ({"R8BGPU_HB_SMEM_DOUBLES": "3500"}, {"up_budget": 3500}),
                    ({"R8BGPU_HBD_SMEM_DOUBLES": "3200"}, {"down_budget": 3200})):
        with monkeypatch.context() as mp:
            for k, v in env.items():
                mp.setenv(k, v)
            for d, t, c, taps, a, plan in walked:
                for i, info in runs(plan)[0]:
                    check_run(plan, i, info, **kw)
                    if info["kind"] == "single":
                        continue
                    base = up_plan(info["ntaps"]) if d == "up" else down_plan(info["ntaps"])
                    if "last2" in kw and base[0]:
                        moved["last2"] += 1
                        assert not info["fuse_last2"] and info["n_buffers"] == info["n_stages"]
                    elif "up_budget" in kw and d == "up" and base[2] != info["w"]:
                        moved["up w"] += 1
                    elif "down_budget" in kw and d == "down" and base[0] != info["w"]:
                        moved["down w"] += 1
    assert all(moved.values()), moved
    with monkeypatch.context() as mp:
        mp.setenv("R8BGPU_HBD_SMEM_DOUBLES", "100")
        plan = make_plan(pkg, "2822400-44100")
        got, inside = runs(plan)
        assert not inside and all(info["kind"] == "single" for _, info in got) and len(got) == 5


def test_report_refuses_other_stages(pkg):
    plan = make_plan(pkg, "44100-2822400")
    assert plan.stages()[0]["name"] == "blockconv"
    with pytest.raises(pkg.R8bGpuError):
        plan.cascade_info(0)
    with pytest.raises(pkg.R8bGpuError):
        plan.cascade_info(len(plan.stages()))
