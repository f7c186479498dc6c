"""CPU: the geometry space of the whole-stepping fused kernels, and a committed table of plans that covers it.

A 2x or 1x BlockConvolver fused with the whole-stepping interpolator runs on k_up2_frac2 (tensor-path or FMA
interpolation) or on the round-1 k_up2_frac (bank in shared or global memory).  Which one, and with which geometry
(phase groups, padded window smaxp, y layout, spectrum table), follows from a few numbers of the plan.  The host decides
all of it in one place, which Plan.fused_info() reports without a device.

GEOMETRIES names plans that together reach every class below; tests/test_gpu_fused_geometry.py runs each of them against
the reference and bit for bit across the kernel's exact variants.  If a planner change moves a plan to another class,
test_every_class_is_reached fails here, on a machine without a GPU, instead of the coverage vanishing.

Rates need not be standard.  A 2x pair with interpolator steps (InStep, OutStep) coprime is src = InStep k / 2,
dst = OutStep k (here k = 60); a 1x pair is src = InStep k, dst = OutStep k with 2 <= InStep / OutStep < 4.

What the report showed when the table was made: with the default settings a whole-stepping pair never reaches the FMA
interpolation of k_up2_frac2 or k_up2_frac with its bank in shared memory (k_up2_frac2 holds any bank k_up2_frac could,
and an FMA bank is never smaller than the tensor-path one), so those classes are reached through the settings a user
may give (R8BGPU_F2_FLAGS, R8BGPU_FUSED_V1).  Every OutStep above 320 at 24-bit attenuation, such as the 441 and 640
pairs of 32000->22050 or 8000->11025, runs on k_up2_frac with its bank in global memory."""
import pytest

ATTEN_16IR, ATTEN_16, ATTEN_24, ATTEN_DEF = 109.56, 136.45, 180.15, 206.91
ATTENS = {"16IR": ATTEN_16IR, "16": ATTEN_16, "24": ATTEN_24, "default": ATTEN_DEF}

# name -> (src, dst, MaxInLen, TransBand, atten, R8B_EXTFFT, settings, kernel of the pair as the report names it)
GEOMETRIES = {
    "44100-96000": (44100.0, 96000.0, 16384, 2.0, ATTEN_24, 0, {}, "f2-tc"),
    "480-540": (480.0, 540.0, 16384, 2.0, ATTEN_24, 0, {}, "f2-tc"),                 # 16/9: padded y, OutStep % 8 = 1
    "390-600": (390.0, 600.0, 16384, 2.0, ATTEN_16IR, 0, {}, "f2-tc"),              # 13/10
    "180-660": (180.0, 660.0, 16384, 2.0, ATTEN_24, 0, {}, "f2-tc"),                # 6/11
    "48000-44100": (48000.0, 44100.0, 16384, 2.0, ATTEN_24, 0, {}, "f2-tc"),        # 320/147: no spectrum table
    "570-720": (570.0, 720.0, 16384, 2.0, ATTEN_16, 0, {}, "f2-tc"),                # 19/12
    "330-780": (330.0, 780.0, 16384, 3.0, ATTEN_DEF, 0, {}, "f2-tc"),               # 11/13
    "510-840": (510.0, 840.0, 16384, 2.0, ATTEN_24, 0, {}, "f2-tc"),                # 17/14
    "510-900": (510.0, 900.0, 16384, 2.0, ATTEN_16IR, 0, {}, "f2-tc"),              # 17/15
    "150-210": (150.0, 210.0, 16384, 2.0, ATTEN_24, 0, {}, "f2-tc"),                # 10/7: OutStep below 8
    "96000-44100": (96000.0, 44100.0, 16384, 2.0, ATTEN_24, 0, {}, "f2-tc"),        # 1x pair, 320/147
    "350-150": (350.0, 150.0, 16384, 2.0, ATTEN_16, 0, {}, "f2-tc"),                # 1x pair, 7/3
    "44100-192000": (44100.0, 192000.0, 8192, 2.0, ATTEN_24, 1, {}, "f2-tc"),       # the pair writes a ring
    "10530-19200": (10530.0, 19200.0, 16384, 2.0, ATTEN_24, 0, {}, "f2-tc"),        # 351/320: the largest that fits
    "10560-19260": (10560.0, 19260.0, 16384, 2.0, ATTEN_24, 0, {}, "v1-global"),    # 352/321: the smallest that does not
    "49470-90000": (49470.0, 90000.0, 16384, 2.0, ATTEN_24, 0, {}, "v1-global"),    # 1649/1500: OutStep 1500, 188 groups
    "44100-96000-fma": (44100.0, 96000.0, 16384, 2.0, ATTEN_24, 0, {"R8BGPU_F2_FLAGS": "2"}, "f2-fma"),
    "48000-44100-fma": (48000.0, 44100.0, 16384, 2.0, ATTEN_24, 0, {"R8BGPU_F2_FLAGS": "2"}, "f2-fma"),
    "44100-96000-v1": (44100.0, 96000.0, 16384, 2.0, ATTEN_24, 0, {"R8BGPU_FUSED_V1": "1"}, "v1-smem"),
    "44100-88200": (44100.0, 88200.0, 16384, 2.0, ATTEN_24, 0, {}, "f2-copy"),
}

# every class some entry must reach
CLASSES = (["tensor path, OutStep %% 8 = %d" % r for r in range(8)] +
           ["tensor path, smaxp %% 16 = %d" % r for r in (0, 4, 8, 12)] +
           ["padded y", "plain y", "up 1", "up 2", "copy", "spectrum table", "no spectrum table", "OutStep below 8",
            "largest tensor bank at 24-bit", "smallest bank past the tensor path at 24-bit", "n_groups next to 192",
            "OutStep 1500", "FMA bank, IR 8", "FMA bank, IR 10", "k_up2_frac, bank in shared memory",
            "k_up2_frac, bank in global memory", "fused pair writes a ring"] +
           ["attenuation %s" % a for a in ATTENS])

F2 = ("f2-tc", "f2-fma")


def make_plan(pkg, name):
    src, dst, m, tb, at, ext = GEOMETRIES[name][:6]
    return pkg.Plan(src, dst, m, tb, at, extfft=ext)


def pair_stage(plan):
    """Index of the BlockConvolver the fused kernel runs on: the first one followed by a whole-stepping interpolator, or
    (a plan without one) the first 2x BlockConvolver."""
    st = plan.stages()
    for i in range(len(st) - 1):
        if st[i]["name"] == "blockconv" and st[i + 1]["name"] == "frac_whole":
            return i
    return next(i for i, s in enumerate(st) if s["name"] == "blockconv" and s["up"] == 2)


def report(pkg, name, monkeypatch, extra=None):
    """(plan, stage, Plan.fused_info) under the entry's settings plus `extra`."""
    with monkeypatch.context() as m:
        for k, v in dict(GEOMETRIES[name][6], **(extra or {})).items():
            m.setenv(k, v)
        plan = make_plan(pkg, name)
        i = pair_stage(plan)
        return plan, i, plan.fused_info(i)


# ---- the report's numbers, restated from the interpolator's StageInfo -------------------------------------------------

def restated_bank(in_step, out_step, flen, ir):
    """(groups, smaxp) of a grouped bank of ir phases: phase pr >= out_step continues in the next stepping cycle."""
    off = [(r * in_step) // out_step for r in range(out_step)]

    def offx(pr):
        return off[pr % out_step] + (pr // out_step) * in_step
    dmax = max(offx(r0 + ir - 1) - offx(r0) for r0 in range(out_step))
    return -(-out_step // ir), (flen + dmax + 3) & ~3


def restated_ir(out_step):
    """8 or 10 phases per FMA group: 10 where it spreads the groups more evenly and out_step % 8 != 0."""
    g8, g10 = -(-out_step // 8), -(-out_step // 10)
    return 10 if out_step % 8 != 0 and ((g10 + 15) // 16) * 10 < ((g8 + 15) // 16) * 8 else 8


def restated_ysh(in_step):
    """The padded y layout's shift for an even in_step (31: plain)."""
    if in_step & 1:
        return 31
    sh = 0
    while not (in_step >> sh) & 1:
        sh += 1
    sh = max(sh, 4)
    return 31 if ((in_step + (in_step >> sh)) & 1) == 0 else sh


def classes_of(name, plan, i, info):
    st = plan.stages()
    k = info["kernel"]
    out = set()
    if k == "f2-tc":
        out.add("tensor path, OutStep %% 8 = %d" % (info["out_step"] % 8))
        out.add("tensor path, smaxp %% 16 = %d" % (info["tc_smaxp"] % 16))
    if k in F2 or k.startswith("v1"):
        out.add("padded y" if info["pad"] else "plain y")
        out.add("up %d" % info["up"])
        if info["out_step"] < 8:
            out.add("OutStep below 8")
        if info["out_step"] == 1500:
            out.add("OutStep 1500")
        if info["tc_n_groups"] >= 185:
            out.add("n_groups next to 192")
        if i + 2 < len(st):
            out.add("fused pair writes a ring")
        out.add("attenuation %s" % next(a for a, v in ATTENS.items() if v == GEOMETRIES[name][4]))
    if k == "f2-copy":
        out.add("copy")
    if k in F2 and info["up"] == 2 or k == "f2-copy":
        out.add("spectrum table" if info["cs"] else "no spectrum table")
    if k == "f2-fma":
        out.add("FMA bank, IR %d" % info["ir"])
    if k == "v1-smem":
        out.add("k_up2_frac, bank in shared memory")
    if k == "v1-global":
        out.add("k_up2_frac, bank in global memory")
    return out


def boundary_classes(reports):
    """The pair of entries at the tensor bank's edge: same attenuation and smaxp, consecutive OutStep, the first fits."""
    out = set()
    for a, (pa, _, ia) in reports.items():
        for b, (pb, _, ib) in reports.items():
            if (GEOMETRIES[a][4] == GEOMETRIES[b][4] == ATTEN_24 and not GEOMETRIES[a][6] and not GEOMETRIES[b][6] and
                    ia["tc_fits"] and not ib["tc_fits"] and ib["out_step"] == ia["out_step"] + 1 and
                    ia["tc_smaxp"] == ib["tc_smaxp"] and ia["kernel"] == "f2-tc" and ib["kernel"] == "v1-global"):
                out |= {"largest tensor bank at 24-bit", "smallest bank past the tensor path at 24-bit"}
    return out


@pytest.fixture(scope="module")
def reports(pkg):
    mp = pytest.MonkeyPatch()
    try:
        return {name: report(pkg, name, mp) for name in GEOMETRIES}
    finally:
        mp.undo()


def test_every_class_is_reached(pkg, reports):
    reached = {}
    for name, (plan, i, info) in reports.items():
        for c in classes_of(name, plan, i, info):
            reached.setdefault(c, []).append(name)
    for c in boundary_classes(reports):
        reached.setdefault(c, []).append("(pair)")
    print("\nclass -> plans")
    for c in CLASSES:
        print("  %-46s %s" % (c, ", ".join(reached.get(c, ["-"]))))
    missing = [c for c in CLASSES if c not in reached]
    assert not missing, missing


@pytest.mark.parametrize("name", list(GEOMETRIES))
def test_report_matches_the_plan(pkg, reports, name):
    """The kernel the table names, the chain shape, and the report's numbers restated from StageInfo."""
    plan, i, info = reports[name]
    st = plan.stages()
    assert info["kernel"] == GEOMETRIES[name][7], info
    bc = st[i]
    assert bc["name"] == "blockconv" and bc["down"] == 1
    if info["kernel"] == "f2-copy":
        assert info["up"] == 2 and info["copy"] == 1 and info["out_step"] == 0
        assert i + 1 == len(st) or st[i + 1]["name"] != "frac_whole"
        return
    f = st[i + 1]
    assert f["name"] == "frac_whole" and info["up"] == bc["up"] and not info["copy"]
    assert (info["in_step"], info["out_step"]) == (f["in_step"], f["out_step"])
    a, b = f["in_step"], f["out_step"]
    if len(st) == 2:    # the interpolator runs from the BlockConvolver's output rate to dst
        src, dst = GEOMETRIES[name][:2]
        assert src * bc["up"] * b == dst * a
    assert (info["tc_n_groups"], info["tc_smaxp"]) == restated_bank(a, b, f["kernel_len"], 8)
    assert info["ir"] == restated_ir(b)
    assert (info["fma_n_groups"], info["fma_smaxp"]) == restated_bank(a, b, f["kernel_len"], info["ir"])
    assert info["tc_smaxp"] % 4 == 0 and info["tc_n_groups"] == -(-b // 8)
    assert info["ysh"] == restated_ysh(a) and info["pad"] == (info["ysh"] != 31)
    assert info["kernel"] in F2 or not (info["tc_fits"] and GEOMETRIES[name][6] == {})


def test_settings_move_the_report(pkg, monkeypatch):
    """The report honours the settings a batch reads: no fusion, the round-1 kernel, no tensor path, IR 10."""
    _, _, base = report(pkg, "44100-96000", monkeypatch)
    assert base["kernel"] == "f2-tc" and base["ir"] == 8
    assert report(pkg, "44100-96000", monkeypatch, {"R8BGPU_NO_FUSION": "1"})[2]["kernel"] == "none"
    assert report(pkg, "44100-96000", monkeypatch, {"R8BGPU_FUSED_V1": "1"})[2]["kernel"] == "v1-smem"
    fma = report(pkg, "44100-96000", monkeypatch, {"R8BGPU_F2_FLAGS": "2", "R8BGPU_IR": "10"})[2]
    assert fma["kernel"] == "f2-fma" and fma["ir"] == 10
    # the 1x pair exists only on the tensor path: without it the two stages run unfused
    assert report(pkg, "96000-44100", monkeypatch, {"R8BGPU_F2_FLAGS": "2"})[2]["kernel"] == "none"
    assert report(pkg, "44100-88200", monkeypatch, {"R8BGPU_FUSED_V1": "1"})[2]["kernel"] == "none"


def test_report_refuses_other_stages(pkg):
    plan = make_plan(pkg, "44100-96000")
    with pytest.raises(pkg.R8bGpuError):
        plan.fused_info(1)      # the interpolator
    with pytest.raises(pkg.R8bGpuError):
        plan.fused_info(2)
