"""Independent streams on the host: the per-channel schedules behind r8bgpu_batch_process_ragged and
r8bgpu_batch_clear_channels, checked against running each channel through the single-stream scheduler
(Plan.simulate) with its own length sequence.  No GPU needed."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from test_host_cpu import RATES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_IN = 4096


def ragged_lens(rng, n_calls, n_ch, max_in=MAX_IN):
    """Seeded ragged block lengths that include 0, 1 and MaxInLen on every channel."""
    lens = rng.integers(0, max_in + 1, size=(n_calls, n_ch))
    for c in range(n_ch):
        rows = rng.choice(n_calls, 3, replace=False)
        lens[rows, c] = (0, 1, max_in)
    return lens.astype(np.int32)


def per_channel_expected(plan, lens, clear):
    """Counts of each channel fed on its own, restarted (a fresh scheduler) wherever it was cleared."""
    n_calls, n_ch = lens.shape
    want = np.empty_like(lens)
    for c in range(n_ch):
        start = 0
        for i in range(n_calls + 1):
            if i == n_calls or (i > start and clear[i, c]):
                want[start:i, c] = plan.simulate(lens[start:i, c])
                start = i
    return want


@pytest.mark.parametrize("src,dst", RATES)
def test_ragged_counts_equal_per_channel_scheduler(pkg, src, dst):
    rng = np.random.default_rng(int(src * 3 + dst))
    plan = pkg.Plan(src, dst, MAX_IN, 2.0, pkg.ATTEN_24)
    lens = ragged_lens(rng, 14, 6)
    counts, groups = plan.simulate_ragged(lens)
    assert np.array_equal(counts, per_channel_expected(plan, lens, np.zeros_like(lens)))
    # distinct schedules never exceed the distinct length histories
    for i in range(len(lens)):
        assert 1 <= groups[i] <= len({tuple(lens[:i + 1, c]) for c in range(lens.shape[1])})


@pytest.mark.parametrize("src,dst", RATES)
def test_clear_channels_restarts_only_the_named_channels(pkg, src, dst):
    rng = np.random.default_rng(int(src + dst * 7))
    plan = pkg.Plan(src, dst, MAX_IN, 2.0, pkg.ATTEN_24)
    lens = ragged_lens(rng, 16, 5)
    clear = (rng.random(lens.shape) < 0.15).astype(np.int32)
    clear[0] = 0
    counts, _ = plan.simulate_ragged(lens, clear)
    assert np.array_equal(counts, per_channel_expected(plan, lens, clear))


def test_lockstep_lengths_keep_one_group(pkg):
    """Equal lengths on every channel leave one schedule, and the counts are the lock-step scheduler's."""
    plan = pkg.Plan(44100.0, 96000.0, MAX_IN, 2.0, pkg.ATTEN_24)
    seq = [4096, 1000, 0, 1, 4096, 17]
    counts, groups = plan.simulate_ragged(np.repeat(np.array(seq, dtype=np.int32)[:, None], 8, axis=1))
    assert list(groups) == [1] * len(seq)
    assert all(list(counts[:, c]) == plan.simulate(seq) for c in range(8))


def test_channels_reconverge(pkg):
    """Channels that diverged share one schedule again once they are in the same state: after equal totals on the
    integer-only chains, and when every diverged channel is cleared."""
    plan = pkg.Plan(48000.0, 44100.0, MAX_IN, 2.0, pkg.ATTEN_24)
    lens = np.array([[100, 200], [200, 100], [0, 0]], dtype=np.int32)
    _, groups = plan.simulate_ragged(lens)
    assert list(groups) == [2, 1, 1]  # BlockConv + whole-step interpolator: the state is the totals
    lens = np.array([[4096, 4096, 10], [4096, 4096, 4096], [5, 5, 5]], dtype=np.int32)
    clear = np.array([[0, 0, 0], [0, 0, 0], [1, 1, 1]], dtype=np.int32)
    counts, groups = plan.simulate_ragged(lens, clear)
    assert list(groups) == [2, 2, 1]
    assert list(counts[2]) == [plan.simulate([5])[0]] * 3


def test_order2_state_depends_on_chunking(pkg):
    """The order-2 interpolator resets its counter once per call (CDSPFracInterpolator.h:907-919): channels with equal
    totals but different block lengths keep separate schedules, and each still counts like its own scheduler."""
    plan = pkg.Plan(48000.0, 47999.0, MAX_IN, 2.0, pkg.ATTEN_24)
    seq_a, seq_b = [4096] * 6, [2048] * 12
    lens = np.zeros((12, 2), dtype=np.int32)
    lens[:6, 0] = seq_a
    lens[:, 1] = seq_b
    counts, _ = plan.simulate_ragged(lens)
    assert list(counts[:, 0]) == plan.simulate(list(lens[:, 0]))
    assert list(counts[:, 1]) == plan.simulate(seq_b)


def test_ragged_errors(pkg):
    plan = pkg.Plan(44100.0, 96000.0, 64)
    with pytest.raises(pkg.R8bGpuError):
        plan.simulate_ragged(np.array([[64, 65]], dtype=np.int32))
    with pytest.raises(pkg.R8bGpuError):
        plan.simulate_ragged(np.array([[-1, 3]], dtype=np.int32))


def test_cpp_header_declares_ragged_calls():
    """The r8b:: header's batch class compiles with the ragged calls (syntax only: no CUDA needed)."""
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    src = ('#include "r8b/CDSPResampler.h"\n'
           "int f(r8b::CDSPResamplerBatch& b, const double* ip, double* op, const int* lens, int* counts) {\n"
           "    int ch[1] = {0};\n"
           "    return b.processRagged(ip, 64, lens, op, 256, 256, counts) |\n"
           "           b.processRaggedDevice(ip, 64, lens, op, 256, 256, counts) | b.clearChannels(ch, 1);\n"
           "}\n")
    r = subprocess.run([cxx, "-std=c++11", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), "-x", "c++", "-"],
                       input=src, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
