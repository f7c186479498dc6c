"""End of stream on the host scheduler (r8bgpu_plan_simulate_flush, behind r8bgpu_batch_flush): the samples a flush
returns and the silence it feeds, against the compiled reference fed the same chunks and then silence, as
CDSPResampler::oneshot() feeds it (CDSPResampler.h:592-651).  No GPU needed."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from test_host_cpu import RATES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_IN = 4096


def ref_tail(r, lens, target, max_in, zeros=None):
    """Feed a fresh reference object the chunks lens (any values: counts do not depend on them), then silence in blocks
    of max_in until its output reaches target (or exactly `zeros` samples of silence).  Returns (outputs before the
    silence, outputs after it, silence fed)."""
    x = np.zeros(max_in)
    got = sum(len(r.process(x[:l])) for l in lens)
    before, fed = got, 0
    while (got < target) if zeros is None else (fed < zeros):
        l = max_in if zeros is None else min(max_in, zeros - fed)
        got += len(r.process(x[:l]))
        fed += l
    r.clear()
    return before, got, fed


def check_against_ref(pkg, ref, src, dst, lens, max_in, target=None, extfft=0):
    plan = pkg.Plan(src, dst, max_in, 2.0, pkg.ATTEN_24, extfft=extfft)
    zeros, count = plan.simulate_flush(lens, target)
    T = plan.default_target(int(np.sum(lens))) if target is None else target
    r = ref.Resampler(src, dst, max_in, 2.0, pkg.ATTEN_24)
    before, after, _ = ref_tail(r, lens, T, max_in)
    assert count == max(0, T - before), (src, dst, list(lens), T)
    if count == 0:
        assert zeros == 0
        return plan, count
    # the silence is the shortest that reaches the target: z samples do, z - 1 do not
    _, got, _ = ref_tail(r, lens, T, max_in, zeros)
    assert got >= T
    _, got, _ = ref_tail(r, lens, T, max_in, zeros - 1)
    assert got < T
    return plan, count


@pytest.mark.parametrize("src,dst", RATES)
def test_default_target_counts_equal_reference(pkg, ref, src, dst):
    rng = np.random.default_rng(int(src * 5 + dst))
    for n_calls in (0, 1, 3, 6):
        lens = rng.integers(0, MAX_IN + 1, n_calls)
        check_against_ref(pkg, ref, src, dst, lens, MAX_IN)


@pytest.mark.parametrize("src,dst", [(44100.0, 96000.0), (48000.0, 44100.0), (48000.0, 47999.0), (2822400.0, 44100.0),
                                     (44100.0, 176400.0), (44100.0, 132300.0), (11025.0, 96000.0)])
def test_explicit_targets(pkg, ref, src, dst):
    rng = np.random.default_rng(int(src + 3 * dst))
    lens = rng.integers(1, MAX_IN + 1, 4)
    plan = pkg.Plan(src, dst, MAX_IN, 2.0, pkg.ATTEN_24)
    produced = sum(plan.simulate(lens))
    T = plan.default_target(int(lens.sum()))
    for target in (0, produced // 2, produced, produced + 1, T, T + 1, T + 5 * MAX_IN + 7):
        check_against_ref(pkg, ref, src, dst, lens, MAX_IN, target=target)


def test_target_already_reached_returns_nothing(pkg):
    plan = pkg.Plan(44100.0, 96000.0, MAX_IN, 2.0, pkg.ATTEN_24)
    lens = [MAX_IN] * 3
    produced = sum(plan.simulate(lens))
    assert produced > 0
    for target in (0, 1, produced):
        assert plan.simulate_flush(lens, target) == (0, 0)


def test_flush_right_after_clear(pkg, ref):
    for src, dst in [(44100.0, 96000.0), (48000.0, 44100.0), (2822400.0, 44100.0)]:
        plan = pkg.Plan(src, dst, MAX_IN, 2.0, pkg.ATTEN_24)
        assert plan.simulate_flush([]) == (0, 0)  # N = 0: the default target is 0
        check_against_ref(pkg, ref, src, dst, [], MAX_IN, target=1000)


@pytest.mark.parametrize("src,dst", [(44100.0, 96000.0), (48000.0, 47999.0), (2822400.0, 44100.0),
                                     (44100.0, 2822400.0)])
def test_silence_spans_several_sub_steps(pkg, ref, src, dst):
    """A MaxInLen far below the chain's latency: the silence goes in as many MaxInLen sub-steps and a shorter last one."""
    max_in = 64
    _, count = check_against_ref(pkg, ref, src, dst, [64, 17, 64, 1], max_in)
    zeros, _ = pkg.Plan(src, dst, max_in, 2.0, pkg.ATTEN_24).simulate_flush([64, 17, 64, 1])
    assert zeros > 4 * max_in and count > 0


def test_extfft(pkg, ref_e1):
    rng = np.random.default_rng(11)
    for src, dst in [(44100.0, 96000.0), (48000.0, 44100.0), (44100.0, 2822400.0), (192000.0, 44100.0)]:
        lens = rng.integers(0, 2049, 4)
        check_against_ref(pkg, ref_e1, src, dst, lens, 2048, extfft=1)
        check_against_ref(pkg, ref_e1, src, dst, lens, 2048, target=int(lens.sum()) * 3, extfft=1)


def test_passthrough(pkg):
    plan = pkg.Plan(44100.0, 44100.0, MAX_IN)
    assert plan.flush_max_out_len == 0
    assert plan.simulate_flush([100, 5]) == (0, 0)
    assert plan.simulate_flush([100, 5], 200) == (95, 95)  # T - E zeros


@pytest.mark.parametrize("src,dst", RATES)
def test_flush_max_out_len_bounds_every_tail(pkg, src, dst):
    """The bound holds over seeded random histories (every chunking, totals far past one block) and is not loose."""
    plan = pkg.Plan(src, dst, MAX_IN, 2.0, pkg.ATTEN_24)
    bound = plan.flush_max_out_len
    rng = np.random.default_rng(int(src + dst * 13))
    worst = 0
    for trial in range(48):
        n_calls = int(rng.integers(0, 12))
        if trial % 3 == 0:
            lens = rng.integers(0, 40, n_calls)
        elif trial % 3 == 1:
            lens = rng.integers(0, MAX_IN + 1, n_calls)
        else:  # far past the chain's latency (the half-band cascades buffer several blocks)
            lens = np.concatenate([np.full(80, MAX_IN), rng.integers(0, MAX_IN + 1, n_calls)])
        worst = max(worst, plan.simulate_flush(lens)[1])
    assert worst <= bound, (worst, bound)
    if not plan.passthrough:
        assert bound <= 2 * worst + 64, (worst, bound)


def test_default_target_is_exact(pkg):
    plan = pkg.Plan(44100.0, 96000.0, MAX_IN)
    for n in (1, 441, 44100, 10 ** 12 + 7, 2 ** 62 // 3):
        want = -((-n * 96000) // 44100)
        assert plan.default_target(n) == want
    plan = pkg.Plan(44100.0, 22050.5, MAX_IN)  # a rate with a fraction: still exact on the binary values
    assert plan.default_target(44100) == -((-44100 * 44101) // 88200)
    # the C++ scheduler uses the same rule: a stream of N samples flushed by default ends at the default target
    for n in (1, 1000, 4096 * 3 + 5):
        lens = [MAX_IN] * (n // MAX_IN) + [n % MAX_IN]
        zeros, count = plan.simulate_flush(lens)
        assert sum(plan.simulate(lens)) + count == plan.default_target(n)


def test_errors(pkg):
    plan = pkg.Plan(44100.0, 96000.0, 64)
    with pytest.raises(pkg.R8bGpuError):
        plan.simulate_flush([65])
    with pytest.raises(pkg.R8bGpuError, match="FASTTIMING"):
        pkg.Plan(48000.0, 47999.0, 1024, 2.0, pkg.ATTEN_24, fasttiming=1).simulate_flush([10])


def test_cpp_header_declares_flush_calls():
    """The r8b:: header's batch class compiles with the flush calls and the batched oneshot (syntax only)."""
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    src = ('#include "r8b/CDSPResampler.h"\n'
           "int f(r8b::CDSPResamplerBatch& b, const double* ip, double* op, const int* lens, int* counts) {\n"
           "    int ch[1] = {0};\n"
           "    long long t[1] = {100};\n"
           "    r8bgpu_buffer o = {op, R8BGPU_S16, 1, 2, 1.0};\n"
           "    return b.flushChannels(ch, 1, t, op, 256, 256, counts) | b.flushChannels(ch, 1, NULL, o, 256, counts) |\n"
           "           b.flushChannelsDevice(ch, 1, NULL, op, 256, 256, counts) |\n"
           "           b.flushChannelsDevice(ch, 1, t, o, 256, counts) | b.oneshot(ip, 64, lens, op, 256, lens);\n"
           "}\n")
    r = subprocess.run([cxx, "-std=c++11", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), "-x", "c++", "-"],
                       input=src, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
