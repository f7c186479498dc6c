"""CPU: the segment layout of long clips (r8bgpu_plan_simulate_oneshot through Plan.simulate_oneshot) over the chain kinds
and seeded clip sets.  For every clip the kept output ranges tile [0, oplen) exactly, each range ends where the twin run
(the clip fed in blocks of MaxInLen from sample 0, r8bgpu_plan_simulate) has produced that many outputs, no round holds more
lanes than the batch has, and the call count is the policy's: the fewest blocks per segment that fit the clips into
ceil(m / n_lanes) rounds of n_lanes lanes, segments dealt out longest first."""
import numpy as np
import pytest

from __graft_entry__ import load_package

pkg = load_package()

CHAINS = [
    (44100.0, 96000.0, 2.0),    # 2x BlockConvolver -> whole stepping
    (48000.0, 44100.0, 2.0),
    (48000.0, 47999.0, 2.0),    # order-2 bank
    (192000.0, 44100.0, 2.0),   # half-band down cascade
    (44100.0, 176400.0, 2.0),   # half-band up
    (48000.0, 16000.0, 2.0),    # 1/3 BlockConvolver
    (48000.0, 16000.0, 0.5),    # large-tile path
    (96000.0, 48000.0, 2.0),
    (2822400.0, 88200.0, 2.0),  # DSD64 -> 88200
    (48000.0, 48000.0, 2.0),    # passthrough
]
MAX_IN = 4096


def plan_of(src, dst, tb, max_in=MAX_IN):
    return pkg.Plan(src, dst, max_in, tb, pkg.ATTEN_24)


def clip_sets(seed, B):
    rng = np.random.default_rng(seed)
    lens = [0, 1, B - 1, B, 3 * B, 5 * B + 17, int(rng.integers(1, 40 * B)), int(rng.integers(1, 200 * B))]
    return np.array(lens, dtype=np.int64)


def twin_totals(plan, length, B):
    """The twin's output total after each block boundary k * B (k = 0 .. ceil(length / B)); passthrough: the input."""
    nb = -(-length // B)
    blocks = [min(B, length - k * B) for k in range(nb)]
    if plan.passthrough:
        return np.concatenate([[0], np.cumsum(blocks)]).astype(np.int64)
    return np.concatenate([[0], np.cumsum(plan.simulate(blocks))]).astype(np.int64) if nb else np.zeros(1, np.int64)


def expected_calls(plan, n_lanes, lens, oplens, B):
    """The policy restated: returns (segments that run, n_calls)."""
    W = plan.oneshot_warmup
    wb = W // B
    nb = [-(-int(v) // B) for v in lens]
    act = [r for r in range(len(lens)) if oplens[r] > 0]
    lanes = max(1, -(-len(act) // n_lanes)) * n_lanes

    def count(L):
        return sum(max(1, -(-nb[r] // L)) for r in act)

    lo, hi = 0, max([1] + nb)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if count(mid) <= lanes:
            hi = mid
        else:
            lo = mid
    L = hi
    costs = []
    for r in act:
        E = twin_totals(plan, int(lens[r]), B)
        K = max(1, -(-nb[r] // L))
        for k in range(K):
            p0, p1 = k * L * B, min((k + 1) * L * B, int(lens[r]))
            e0 = min(int(E[min(k * L, nb[r])]), int(oplens[r]))
            e1 = int(oplens[r]) if k + 1 == K else min(int(E[(k + 1) * L]), int(oplens[r]))
            if e1 > e0:
                costs.append((-(-(p1 - max(0, p0 - wb * B)) // B), k + 1 == K))
    costs.sort(key=lambda t: -t[0])
    n_calls = 0
    for i in range(0, len(costs), n_lanes):
        rd = costs[i:i + n_lanes]
        n_calls += max(c for c, _ in rd) + (1 if any(f for _, f in rd) else 0)
    return len(costs), n_calls


@pytest.mark.parametrize("src,dst,tb", CHAINS)
@pytest.mark.parametrize("n_lanes", [1, 7, 64])
@pytest.mark.parametrize("seed", [3, 11])
def test_layout_tiles_outputs(src, dst, tb, n_lanes, seed):
    plan = plan_of(src, dst, tb)
    B = MAX_IN
    W = plan.oneshot_warmup
    assert W % MAX_IN == 0
    if not plan.passthrough:
        assert W >= int(plan.state_windows()[0]) and W > 0
    lens = clip_sets(seed, B)
    rng = np.random.default_rng(seed + 100)
    default = np.array([plan.default_target(int(v)) for v in lens], dtype=np.int64)
    for oplens in (None, default, np.maximum(default - rng.integers(0, 300, len(lens)), 0),
                   default + rng.integers(0, 3000, len(lens))):
        op = default if oplens is None else oplens
        segs, n_calls = plan.simulate_oneshot(n_lanes, lens, oplens)
        n_segs, want_calls = expected_calls(plan, n_lanes, lens, op, B)
        assert len(segs) == n_segs and n_calls == want_calls
        for s in segs:
            assert s["p0"] % B == 0 and s["start"] % B == 0
            assert s["start"] == max(0, s["p0"] - W)
            assert 0 <= s["lane"] < n_lanes
        for rd in np.unique(segs["round"]):
            lanes = segs["lane"][segs["round"] == rd]
            assert len(lanes) == len(set(lanes.tolist())) <= n_lanes
        for r in range(len(lens)):
            mine = np.sort(segs[segs["clip"] == r], order="e0")
            if op[r] == 0:
                assert len(mine) == 0
                continue
            assert mine["e0"][0] == 0 and mine["e1"][-1] == op[r]
            assert np.all(mine["e1"][:-1] == mine["e0"][1:]) and np.all(mine["e1"] > mine["e0"])
            E = twin_totals(plan, int(lens[r]), B)
            for s in mine:
                assert s["e0"] == min(E[s["p0"] // B], op[r])
                if s["p1"] < lens[r]:
                    assert s["p1"] % B == 0 and s["e1"] == min(E[s["p1"] // B], op[r])
            # the clip's last segment runs unless its whole output lies in the blocks before it
            assert mine["p1"][-1] == lens[r] or E[mine["p1"][-1] // B] >= op[r]


def test_clip_past_2_31():
    """A DSD64 clip of an hour: lengths past 2^31 are the point of 64-bit lengths."""
    plan = plan_of(2822400.0, 88200.0, 2.0, 65536)
    n = 2822400 * 3600 // 8 * 8
    assert n > 2 ** 31
    segs, n_calls = plan.simulate_oneshot(1024, [n])
    segs = np.sort(segs, order="e0")
    assert segs["e0"][0] == 0 and segs["e1"][-1] == plan.default_target(n)
    assert np.all(segs["e1"][:-1] == segs["e0"][1:]) and len(segs) <= 1024
    nb = -(-n // 65536)
    L = -(-nb // 1024)  # the fewest blocks per segment that fit 1024 lanes
    assert n_calls == plan.oneshot_warmup // 65536 + L + 1


def test_refusals():
    tr = pkg.Plan.trim(48000.0, 44100.0, MAX_IN, 2.0, pkg.ATTEN_24, 0.001)
    with pytest.raises(pkg.R8bGpuError, match="trim plans"):
        tr.simulate_oneshot(4, [1000])
    ft = pkg.Plan(48000.0, 47999.0, MAX_IN, 2.0, pkg.ATTEN_24, fasttiming=1)
    with pytest.raises(pkg.R8bGpuError, match="R8B_FASTTIMING"):
        ft.simulate_oneshot(4, [1000])
    p = plan_of(44100.0, 96000.0, 2.0)
    with pytest.raises(pkg.R8bGpuError, match="negative length"):
        p.simulate_oneshot(4, [1000, -1])
    with pytest.raises(pkg.R8bGpuError, match="negative length"):
        p.simulate_oneshot(4, [1000, 10], [5, -3])
    with pytest.raises(pkg.R8bGpuError, match="bad arguments"):
        p.simulate_oneshot(0, [1000])
