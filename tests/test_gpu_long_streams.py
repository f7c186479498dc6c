"""GPU: streams past 2^31 and 2^32 samples.

Every stage is a pure function of absolutely indexed streams, so a live stream's indices only grow; an always-on 48 kHz
stream passes 2^32 after about a day, a DSD64 input after 25 minutes.  One absolute index truncated to 32 bits would give
correct output for hours and garbage afterwards.  Two ways to get there:

(a) Real long runs.  A device buffer of silence is fed call after call past 2^32 input samples (or 2^31 output samples),
    then a few calls of noise.  The reference's state is bounded and its InCounter resets every call, so it is fed a
    prefix of silence of R = (N mod P) + k P samples instead, P a period of the chain's input: per-call counts must be
    equal and values within the parity bar of test_gpu_parity.py.

(b) Seeking through the state blob.  A channel's exported stream is shifted by whole periods of every stage -- n_in,
    n_out, the order-2 read position p and the dither count m -- and imported again.  Each kernel is translation-invariant
    under such shifts, so a seeked channel must produce the same counts and the same bits as an unshifted twin fed the
    same calls (dithered outputs: the host quantiser at the shifted output index).
"""
from fractions import Fraction
from math import gcd

import numpy as np
import pytest

import oracle_util as ou
from test_gpu_mixed import assert_bits
from test_long_streams_cpu import _chain_ratios, chain_total, emitted

pytestmark = pytest.mark.gpu

A24 = 180.15
M16 = 2 ** 16


def _lcm(a, b):
    return a * b // gcd(a, b)


# ---- (b) seeking ------------------------------------------------------------------------------------------------------------

def period(plan, src, dst):
    """An input shift Q whose induced shift at every stage input and output is a multiple of every absolute period that
    stage has.  The periods the operators themselves define are exact: whole-step InStep on the input and OutStep on the
    output (the phase of output j is j * InStep mod OutStep), BlockConv U and D, the block length (InputLen) of block-exact
    decimation, half-band parity.  On top of those, every stage other than block-exact decimation takes a margin factor
    that is not derived from the kernels: 2^16 at its input and output (2^8 / 2^7 for a half-band decimator, whose
    cascade gathers DSD bytes), and 8 on the output of an interpolator (the fused kernels' 8-phase groups).  The 2^16
    margin is an upper bound chosen to exceed every tile size of the kernels (at most 2^16 samples), not derived from any
    anchor found in them: a tile anchored to an absolute index would be covered by it rather than exposed.  So Q is a
    bound, not the smallest such shift.  Returns (Q, [(ratio at the stage input, ratio of the stage)])."""
    stages = plan.stages()
    ratios = _chain_ratios(stages, Fraction(src), Fraction(dst))
    q, r = 1, Fraction(1)
    out = []
    for st, ri in zip(stages, ratios):
        k = st["name"]
        exact = k == "blockconv" and st["down"] > 1 and st["down"] & (st["down"] - 1) == 0
        if exact:
            m_in, m_out = st["ref_input_len"], st["ref_input_len"] // st["down"]
        elif k == "blockconv":
            m_in, m_out = _lcm(M16, _lcm(st["up"], st["down"])), M16
        elif k == "frac_whole":
            m_in, m_out = _lcm(M16, st["in_step"]), _lcm(M16, 8 * st["out_step"])
        elif k == "frac_poly":
            m_in, m_out = M16, 8
        elif k == "hbdown":
            m_in, m_out = 2 ** 8, 2 ** 7
        else:
            m_in, m_out = M16, 2 * M16
        for m, x in ((m_in, r), (m_out, r * ri)):  # Q * x must be a multiple of m
            mq = m * x.denominator
            q = _lcm(q, mq // gcd(mq, x.numerator))
        out.append((r, ri))
        r *= ri
    return q, out


def shifts(plan, src, dst, d0):
    """Per stage (input shift, output shift) for an input shift d0 (a multiple of period())."""
    q, rs = period(plan, src, dst)
    assert d0 % q == 0
    res = []
    for r, ri in rs:
        a, b = d0 * r, d0 * r * ri
        assert a.denominator == 1 and b.denominator == 1
        res.append((int(a), int(b)))
    return res


_MASK = 2 ** 64 - 1


def _term(w, i):
    z = (w ^ (i * 0x9E3779B97F4A7C15)) & _MASK
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _MASK
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _MASK
    return z ^ (z >> 31)


def seek_blob(blob, plan, src, dst, d0, dm=None):
    """The blob of the same stream d0 input samples later (r8b_capi.cu StateHeader / StateStage): every stage's n_in and
    n_out and the order-2 read position move by that stage's shifts, the dither count m by the chain's output shift (or
    dm), and word 1 (the checksum: the sum of state_word_term(w_i, i) over i != 1, mod 2^64) follows."""
    w = np.frombuffer(blob, dtype=np.uint64).copy()
    v = w.view(np.int64)
    stages = plan.stages()
    sh = shifts(plan, src, dst, d0)
    changes = {}

    def add(i, d):
        changes.setdefault(i, int(w[i]))
        v[i] += d

    for j, (st, (di, do)) in enumerate(zip(stages, sh)):
        base = 32 + 8 * j
        if st["name"] != "frac_poly":  # past its start-up, a stage's count moves with its input: n_out = emitted(n_in)
            n_in, n_out = int(v[base]), int(v[base + 1])
            assert emitted(st, n_in) == n_out and emitted(st, n_in + di) == n_out + do, ("stage %d in its start-up" % j)
        add(base + 0, di)
        add(base + 1, do)
        if st["name"] == "frac_poly":
            add(base + 5, di)
    add(31, sh[-1][1] if dm is None else dm)
    s = int(w[1])
    for i, old in changes.items():
        s = (s - _term(old, i) + _term(int(w[i]), i)) & _MASK
    w[1] = np.uint64(s)
    return w.tobytes()


def seek(batch, channels, plan, src, dst, d0):
    """Moves the named channels of batch d0 input samples ahead (all by the same shift)."""
    blobs = batch.export_channels(channels)
    batch.import_channels(channels, [seek_blob(b, plan, src, dst, d0) for b in blobs])


def shift_to(plan, src, dst, n_in, target, below=False):
    """A multiple of period() that moves a stream at n_in inputs to target or just past it (below: just below it)."""
    q, _ = period(plan, src, dst)
    assert q < 2 ** 30, q
    return (target - n_in) // q * q if below else -((n_in - target) // q) * q


STRADDLE, PAST_2_32, AT_2_40 = 2 ** 31, 2 ** 32 + 12345, 2 ** 40
POSITIONS = [STRADDLE, PAST_2_32, AT_2_40]
# Input positions whose chain OUTPUT index lies in [2^31, 2^32): an index cast to int there turns negative.  For chains
# whose period is a power of two (the half-band cascades) a 32-bit truncation is otherwise a shift by a multiple of 2^32,
# which the bit-identity oracle cannot see; a sign change it can.
OUT_3_2_30 = -1


# lock-step, every channel seeked by the same shift: the fused / cascade kernels at large indices
LOCKSTEP = [
    (44100.0, 96000.0, 0),     # k_up2_frac2, UP = 2
    (96000.0, 44100.0, 0),     # the 1x fused pair
    (192000.0, 44100.0, 0),    # k_hbdown + fused pair
    (48000.0, 16000.0, 0),     # k_blockconv 1/3
    (48000.0, 47999.0, 0),     # order-2 interpolator
    (2822400.0, 44100.0, 0),   # half-band decimator cascade
    (44100.0, 2822400.0, 1),   # half-band upsampler cascade
]


@pytest.mark.parametrize("target", POSITIONS + [OUT_3_2_30], ids=["straddle_2_31", "past_2_32", "at_2_40", "out_3_2_30"])
@pytest.mark.parametrize("src,dst,ext", LOCKSTEP)
def test_seek_lockstep_is_bit_identical(pkg, src, dst, ext, target):
    L = 2 ** 18 if src > 10 ** 6 else 2 ** 16 if dst / src < 8 else 2 ** 13
    out_case = target == OUT_3_2_30
    if out_case:
        target = int(3 * 2 ** 30 * Fraction(src) / Fraction(dst)) + 1
    plan = pkg.Plan(src, dst, L, 2.0, A24, extfft=ext)
    S, T = pkg.Batch(plan, 2, 0), pkg.Batch(plan, 2, 0)
    rng = np.random.default_rng(int(src + dst))
    x = ou.white_noise(2, L * 4, seed=int(dst))
    for k in range(4):  # past every stage's start-up
        xa = x[:, k * L:(k + 1) * L]
        assert_bits(S.process_host(xa), T.process_host(xa), "warm-up")
    n_in = int(S.channel_totals()[0][0])
    d0 = shift_to(plan, src, dst, n_in, target - L // 2, below=True) if target == STRADDLE else \
        shift_to(plan, src, dst, n_in, target)
    seek(S, [0, 1], plan, src, dst, d0)
    assert S.channel_groups == 1
    assert list(S.channel_totals()[0]) == [n_in + d0] * 2
    # up to the straddling call in whole blocks of L, then blocks of L / 2 .. L
    n_calls = 3 if target != STRADDLE else 3 + (STRADDLE - (n_in + d0)) // L
    for k in range(n_calls):
        xa = ou.white_noise(2, L if k + 3 < n_calls else int(rng.integers(L // 2, L + 1)), seed=100 + k)
        ys, yt = S.process_host(xa), T.process_host(xa)
        assert_bits(ys, yt, "call %d at input %d" % (k, int(S.channel_totals()[0][0])))
    assert S.channel_totals()[0][0] > target
    tot_s, tot_t = S.channel_totals(), T.channel_totals()
    if out_case:
        assert 3 * 2 ** 30 <= tot_s[1][0] < 2 ** 32
    assert tot_s[0][0] - tot_t[0][0] == d0
    assert tot_s[1][0] - tot_t[1][0] == shifts(plan, src, dst, d0)[-1][1]
    # the flush's default target moves with the stream (d0 * dst / src outputs): the same tail
    fs, ns = S.flush([0, 1])
    ft, nt = T.flush([0, 1])
    assert list(ns) == list(nt) and ns[0] > 0
    assert_bits(fs, ft, "flushed tails")


def _ragged_states(pkg, plan, src, dst, n_ch, seed):
    """A twin pair of batches whose channels hold diverged streams (ragged warm-up)."""
    S, T = pkg.Batch(plan, n_ch, 0), pkg.Batch(plan, n_ch, 0)
    rng = np.random.default_rng(seed)
    M = plan.max_in_len
    for k in range(4):
        lens = rng.integers(M // 2, M + 1, n_ch)
        xs = [ou.white_noise(1, int(l), seed=seed * 10 + k * n_ch + c)[0] for c, l in enumerate(lens)]
        ys, yt = S.process_ragged(xs), T.process_ragged(xs)
        for c in range(n_ch):
            assert_bits(ys[c], yt[c], "warm-up")
    return S, T, rng


@pytest.mark.parametrize("src,dst", [(44100.0, 96000.0), (48000.0, 47999.0), (192000.0, 44100.0)])
def test_seek_ragged_channels_at_different_positions(pkg, src, dst):
    M = 2 ** 16
    plan = pkg.Plan(src, dst, M, 2.0, A24)
    S, T, rng = _ragged_states(pkg, plan, src, dst, 5, 7)
    n_in = S.channel_totals()[0]
    S.clear_channels([2])  # a fresh channel next to the far ones
    T.clear_channels([2])
    for c, target in zip((0, 1, 3), POSITIONS):
        seek(S, [c], plan, src, dst, shift_to(plan, src, dst, int(n_in[c]), target))
    assert S.channel_groups == 5
    for k in range(4):
        lens = rng.integers(0, M + 1, 5)
        xs = [ou.white_noise(1, int(l), seed=500 + k * 5 + c)[0] for c, l in enumerate(lens)]
        ys, yt = S.process_ragged(xs), T.process_ragged(xs)
        for c in range(5):
            assert_bits(ys[c], yt[c], "call %d channel %d" % (k, c))
    assert S.channel_totals()[0][0] > STRADDLE
    # explicit flush targets: the twin's target moved by the channel's output shift returns the same tail
    tt = T.channel_totals()[1][[0, 1, 3]] + np.array([1000, 7, 4096])
    ts = tt + (S.channel_totals()[1][[0, 1, 3]] - T.channel_totals()[1][[0, 1, 3]])
    fs, ns = S.flush([0, 1, 3], targets=ts)
    ft, nt = T.flush([0, 1, 3], targets=tt)
    assert list(ns) == list(nt)
    for c in (0, 1, 3):
        assert_bits(fs[c, :ns[c]], ft[c, :nt[c]], "flushed tail, channel %d" % c)


# typed inputs and outputs: int16 planar and interleaved, mu-law, DSD
@pytest.mark.parametrize("case", ["s16_planar", "s16_interleaved", "ulaw", "dsd"])
def test_seek_typed_buffers(pkg, case):
    src, dst = (2822400.0, 44100.0) if case == "dsd" else (48000.0, 44100.0)
    M = 2 ** 20 if case == "dsd" else 2 ** 17
    plan = pkg.Plan(src, dst, M, 2.0, A24)
    S, T = pkg.Batch(plan, 3, 0), pkg.Batch(plan, 3, 0)
    rng = np.random.default_rng(11)
    inter = case == "s16_interleaved"

    def block(lens):
        w = int(max(lens))
        if case == "dsd":
            return rng.integers(0, 256, (3, (w + 7) // 8), dtype=np.uint8), dict(fmt=pkg.DSD_LSB, in_scale=0.5)
        if case == "ulaw":
            return rng.integers(0, 256, (3, w), dtype=np.uint8), dict(fmt=pkg.ULAW, out_fmt=pkg.ULAW, in_scale=1 / 32768,
                                                                       out_scale=32768.0)
        x = rng.integers(-20000, 20000, (w, 3) if inter else (3, w), dtype=np.int16)
        return x, dict(interleaved=inter)

    def call(lens):
        x, kw = block(lens)
        ys, cs = S.process_ragged_fmt(x, lens, **kw)
        yt, ct = T.process_ragged_fmt(x, lens, **kw)
        assert list(cs) == list(ct)
        assert_bits(ys, yt, "%s call" % case)

    step = 8 if case == "dsd" else 1
    for _ in range(3):
        call((rng.integers(M // 2, M + 1, 3) // step * step).astype(np.int32))
    n_in = S.channel_totals()[0]
    for c, target in zip(range(3), POSITIONS):
        seek(S, [c], plan, src, dst, shift_to(plan, src, dst, int(n_in[c]), target))
    for _ in range(3):
        call((rng.integers(0, M + 1, 3) // step * step).astype(np.int32))


def test_seek_mixed_batch_with_three_parts(pkg):
    M = 2 ** 15
    specs = [(44100.0, 96000.0), (48000.0, 47999.0), (96000.0, 44100.0)]
    plans = [pkg.Plan(s, d, M, 2.0, A24) for s, d in specs]
    plan_of = np.array([0, 1, 2, 1, 0, 2], np.int32)
    S, T = pkg.Batch.mixed(plans, plan_of, 0), pkg.Batch.mixed(plans, plan_of, 0)
    rng = np.random.default_rng(5)

    def call():
        lens = rng.integers(M // 2, M + 1, 6)
        xs = [ou.white_noise(1, int(l), seed=int(rng.integers(1 << 30)))[0] for l in lens]
        ys, yt = S.process_ragged(xs), T.process_ragged(xs)
        for c in range(6):
            assert_bits(ys[c], yt[c], "channel %d" % c)

    for _ in range(4):
        call()
    n_in = S.channel_totals()[0]
    for c in range(6):
        p = plan_of[c]
        seek(S, [c], plans[p], specs[p][0], specs[p][1],
             shift_to(plans[p], specs[p][0], specs[p][1], int(n_in[c]), POSITIONS[c % 3]))
    for _ in range(3):
        call()


def test_seek_trim_channel_with_a_new_factor_every_call(pkg):
    src, dst, M = 44100.0, 48000.0, 2 ** 16
    plan = pkg.Plan.trim(src, dst, M, 2.0, A24, 0.01)
    S, T, rng = _ragged_states(pkg, plan, src, dst, 2, 9)
    n_in = S.channel_totals()[0]
    seek(S, [0], plan, src, dst, shift_to(plan, src, dst, int(n_in[0]), PAST_2_32))
    seek(S, [1], plan, src, dst, shift_to(plan, src, dst, int(n_in[1]), STRADDLE))
    for k in range(4):
        f = 1.0 + float(rng.uniform(-0.01, 0.01))
        S.set_trim([0, 1], [f, 2.0 - f])
        T.set_trim([0, 1], [f, 2.0 - f])
        lens = rng.integers(0, M + 1, 2)
        xs = [ou.white_noise(1, int(l), seed=900 + 2 * k + c)[0] for c, l in enumerate(lens)]
        ys, yt = S.process_ragged(xs), T.process_ragged(xs)
        for c in range(2):
            assert_bits(ys[c], yt[c], "trim call %d channel %d" % (k, c))


@pytest.mark.parametrize("taps", [None, [1.2, -0.9, 0.6, -0.4, 0.25]], ids=["flat", "shaped"])
def test_seek_dithered_int16(pkg, taps):
    """TPDF noise is indexed by the absolute output number: a seeked dithered stream equals the host quantiser, at the
    shifted output index, of its twin's fp64 output.  (The dither count m indexes the error-history ring, so it moves by
    the output shift, a multiple of 16.)"""
    src, dst, M = 48000.0, 44100.0, 2 ** 15
    plan = pkg.Plan(src, dst, M, 2.0, A24)
    A, T = pkg.Batch(plan, 1, 0), pkg.Batch(plan, 1, 0)
    A.set_dither([0], 4242, taps)
    rng = np.random.default_rng(3)
    scale = 30000.0
    hist = np.zeros(16)

    def twin_call(x, first):
        nonlocal hist
        y, nt = T.process_ragged_fmt(x, [x.shape[1]])
        want, hist = pkg.dither_quantize(y[0, :nt[0]], pkg.S16, 4242, taps, scale=scale, first_index=first, state=hist)
        return want

    for _ in range(3):  # the quantiser restates the exporter from its clear on
        x = ou.white_noise(1, int(rng.integers(M // 2, M + 1)), seed=int(rng.integers(1 << 30)))
        first = int(T.channel_totals()[1][0])
        q, n = A.process_ragged_fmt(x, [x.shape[1]], out_dtype=np.int16, out_scale=scale)
        assert_bits(q[0, :n[0]], twin_call(x, first), "dithered int16 before the seek")
    n_in = int(A.channel_totals()[0][0])
    d0 = shift_to(plan, src, dst, n_in, 2 * PAST_2_32)  # outputs past 2^32
    d_out = shifts(plan, src, dst, d0)[-1][1]
    assert d_out % 16 == 0
    S = pkg.Batch(plan, 1, 0)
    S.import_channels([0], [seek_blob(A.export_channels([0])[0], plan, src, dst, d0)])
    for _ in range(3):
        x = ou.white_noise(1, int(rng.integers(0, M + 1)), seed=int(rng.integers(1 << 30)))
        first = int(T.channel_totals()[1][0]) + d_out
        assert first == int(S.channel_totals()[1][0]) > 2 ** 32
        q, n = S.process_ragged_fmt(x, [x.shape[1]], out_dtype=np.int16, out_scale=scale)
        assert_bits(q[0, :n[0]], twin_call(x, first), "dithered int16 past 2^32")


def test_reexport_seeked_stream_into_a_second_batch(pkg):
    src, dst, M = 44100.0, 96000.0, 2 ** 16
    plan = pkg.Plan(src, dst, M, 2.0, A24)
    S, T, rng = _ragged_states(pkg, plan, src, dst, 2, 13)
    seek(S, [1], plan, src, dst, shift_to(plan, src, dst, int(S.channel_totals()[0][1]), AT_2_40))
    B = pkg.Batch(plan, 3, 0)
    B.import_channels([2], S.export_channels([1]))
    assert B.channel_totals()[0][2] == S.channel_totals()[0][1] > AT_2_40 - 2 ** 30
    for k in range(3):
        x = ou.white_noise(1, int(rng.integers(0, M + 1)), seed=1300 + k)[0]
        yb = B.process_ragged([np.zeros(0), np.zeros(0), x])[2]
        yt = T.process_ragged([np.zeros(0), x])[1]
        assert_bits(yb, yt, "re-exported stream, call %d" % k)


# ---- (a) real long runs ---------------------------------------------------------------------------------------------------

def _silence_run(call, n_target, l):
    """call(l) feeds l samples of the device buffer of silence; calls it until n_target inputs have gone in.  Returns (inputs
    fed, the calls' counts)."""
    counts, done = [], 0
    while done < n_target:
        counts.append(call(l))
        done += l
    return done, counts


def _noise_calls(blocks, load, call, d_out):
    """Loads each block into the device input buffer (load(block)), runs one call of its length and copies the output out."""
    got = []
    for b in blocks:
        load(b)
        n = call(len(b))
        got.append(d_out[:n].cpu().numpy())
    return got


def _assert_meets_reference(r, fill, n_prefix, blocks, got):
    """Feeds the reference object r n_prefix samples of fill (one period of the silence, tiled), in calls of at most MaxInLen
    = len(fill), then the blocks: per call the same count as got, values within the parity bar."""
    while n_prefix > 0:
        k = min(len(fill), n_prefix)
        r.process(fill[:k])
        n_prefix -= k
    for k, (b, y) in enumerate(zip(blocks, got)):
        want = r.process(b)
        assert len(want) == len(y), (k, len(want), len(y))
        mx, rms = ou.parity_metrics(y, want)
        assert mx <= 32 * ou.EPS and rms <= 4 * ou.EPS, (k, mx / ou.EPS, rms / ou.EPS)


def _prefix_len(n, q, least):
    """A silence prefix the reference can take instead of n inputs: n mod q plus whole periods q, past its start-up."""
    return n % q + q * max(1, -(-least // q))


def _f64_real_run(pkg, src, dst, ext, L, n_target, blocks):
    """One fp64 channel fed silence through process_ptr until n_target inputs, then the blocks.  Returns (plan, inputs
    before the blocks, the silence calls' counts, the blocks' outputs)."""
    import torch
    plan = pkg.Plan(src, dst, L, 2.0, A24, extfft=ext)
    B = pkg.Batch(plan, 1, 0)
    cap = plan.max_out_len
    d_in = torch.zeros(L, dtype=torch.float64, device="cuda:0")
    d_out = torch.empty(cap, dtype=torch.float64, device="cuda:0")
    B.set_stream(0)

    def call(l):
        return B.process_ptr(d_in.data_ptr(), L, l, d_out.data_ptr(), cap, cap)

    N, counts = _silence_run(call, n_target, L)
    assert B.channel_totals()[0][0] == N
    assert B.channel_totals()[1][0] == chain_total(plan.stages(), N) == sum(counts)
    got = _noise_calls(blocks, lambda b: d_in[:len(b)].copy_(torch.from_numpy(b)), call, d_out)
    del d_in, d_out
    torch.cuda.empty_cache()
    return plan, N, counts, got


REAL = [(44100.0, 96000.0), (96000.0, 44100.0), (192000.0, 44100.0), (48000.0, 16000.0)]


@pytest.mark.parametrize("src,dst", REAL)
def test_real_run_past_2_32_meets_the_reference(pkg, ref, src, dst):
    L = 2 ** 22
    x = ou.white_noise(1, 2 * L + L // 3, seed=17)[0]
    blocks = [x[:L], x[L:2 * L], x[2 * L:]]  # the last one short
    plan, N, _, got = _f64_real_run(pkg, src, dst, 0, L, 2 ** 32, blocks)
    q, _ = period(plan, src, dst)
    _assert_meets_reference(ref.Resampler(src, dst, L, 2.0, A24), np.zeros(L), _prefix_len(N, q, 2 ** 20), blocks, got)


def test_real_run_upsampler_cascade_past_2_31_outputs(pkg, ref_e1):
    """44100 -> 2822400 (R8B_EXTFFT): the half-band upsampler cascade writes output indices past 2^31."""
    src, dst, L = 44100.0, 2822400.0, 2 ** 20
    x = ou.white_noise(1, L + L // 2 + 3, seed=19)[0]
    blocks = [x[:L], x[L:]]
    plan, N, counts, got = _f64_real_run(pkg, src, dst, 1, L, 2 ** 31 // 64 + L, blocks)
    assert sum(counts) > 2 ** 31
    q, _ = period(plan, src, dst)
    _assert_meets_reference(ref_e1.Resampler(src, dst, L, 2.0, A24), np.zeros(L), _prefix_len(N, q, 2 ** 18), blocks, got)


def _dsd_values(raw):
    """DSF (LSB-first) bytes as the samples the reference takes: bit 1 -> +0.5, bit 0 -> -0.5."""
    return np.unpackbits(raw, bitorder="little").astype(np.float64) - 0.5


def test_real_run_dsd_past_2_32_bits(pkg, ref):
    """2822400 -> 44100 from planar DSD bytes: the decimator cascade's bit gather past 2^32 input bits (idle pattern 0x69,
    then random bits)."""
    import torch
    src, dst, L = 2822400.0, 44100.0, 2 ** 22
    plan = pkg.Plan(src, dst, L, 2.0, A24)
    B = pkg.Batch(plan, 1, 0)
    cap = plan.max_out_len
    d_in = torch.full((L // 8,), 0x69, dtype=torch.uint8, device="cuda:0")
    d_out = torch.empty(cap, dtype=torch.float64, device="cuda:0")
    B.set_stream(0)
    bi = pkg.Buffer.make(d_in.data_ptr(), pkg.DSD_LSB, False, L // 8, 0.5)
    bo = pkg.Buffer.make(d_out.data_ptr(), pkg.F64, False, cap, 1.0)

    def call(l):
        return B.process_fmt(bi, l, bo, cap, host=False)

    N, counts = _silence_run(call, 2 ** 32, L)
    assert B.channel_totals()[1][0] == chain_total(plan.stages(), N) == sum(counts)
    rng = np.random.default_rng(23)
    raws = [rng.integers(0, 256, L // 8, dtype=np.uint8), rng.integers(0, 256, L // 16, dtype=np.uint8)]
    got = _noise_calls(raws, lambda b: d_in[:len(b)].copy_(torch.from_numpy(b)), lambda nb: call(8 * nb), d_out)
    del d_in, d_out
    torch.cuda.empty_cache()
    q, _ = period(plan, src, dst)
    q = _lcm(q, 8)  # and whole bytes of the idle pattern
    idle = np.tile(_dsd_values(np.array([0x69], np.uint8)), L // 8)
    _assert_meets_reference(ref.Resampler(src, dst, L, 2.0, A24), idle, _prefix_len(N, q, 2 ** 20),
                            [_dsd_values(r) for r in raws], got)


def test_real_run_order2_past_2_32_seeks_back(pkg):
    """48000 -> 47999 runs for real past 2^32 inputs; its exported stream, imported as it is into one fresh batch and
    seeked back down by whole periods into another, continues bit for bit alike in both."""
    import torch
    src, dst, L = 48000.0, 47999.0, 2 ** 22
    plan = pkg.Plan(src, dst, L, 2.0, A24)
    A = pkg.Batch(plan, 1, 0)
    cap = plan.max_out_len
    d_in = torch.zeros(L, dtype=torch.float64, device="cuda:0")
    d_out = torch.empty(cap, dtype=torch.float64, device="cuda:0")
    A.set_stream(0)
    _silence_run(lambda l: A.process_ptr(d_in.data_ptr(), L, l, d_out.data_ptr(), cap, cap), 2 ** 32, L)
    del d_in, d_out
    torch.cuda.empty_cache()
    x = ou.white_noise(1, L, seed=29)[0]
    A.process_ragged([x[:L // 2]])
    blob = A.export_channels([0])[0]
    n_in = int(A.channel_totals()[0][0])
    d0 = shift_to(plan, src, dst, n_in, 2 ** 25)  # back down to about 2^25
    assert d0 < 0 and n_in + d0 > 2 ** 24
    X, Y = pkg.Batch(plan, 2, 0), pkg.Batch(plan, 2, 0)
    X.import_channels([1], [blob])
    Y.import_channels([1], [seek_blob(blob, plan, src, dst, d0, dm=0)])  # (no dither: m stays 0)
    assert Y.channel_totals()[0][1] == n_in + d0
    rng = np.random.default_rng(31)
    for k in range(3):
        xk = ou.white_noise(1, int(rng.integers(0, L + 1)), seed=3100 + k)[0]
        yx = X.process_ragged([np.zeros(0), xk])[1]
        yy = Y.process_ragged([np.zeros(0), xk])[1]
        assert_bits(yx, yy, "real 2^32 stream vs its seeked-back copy, call %d" % k)


# ---- (c) caller buffers past 2^31 elements ------------------------------------------------------------------------------

def _device_buffer(n, fill, dtype=None):
    """A device tensor of n elements set to fill, or a skip when the shared device has no room for it."""
    import torch
    try:
        return torch.full((n,), fill, dtype=dtype or torch.uint8, device="cuda:0")
    except torch.cuda.OutOfMemoryError:
        torch.cuda.empty_cache()
        pytest.skip("no room on the device for a %.1f GB buffer" % (n / 1e9))


def _view(buf, n_ch, n, stride, interleaved):
    """Channel-major [n_ch, n] view of the typed buffer layout: channel c's sample i at c * stride + i (planar) or
    i * stride + c (interleaved)."""
    import torch
    return torch.as_strided(buf, (n_ch, n), (1, stride) if interleaved else (stride, 1))


@pytest.mark.parametrize("interleaved", [False, True], ids=["planar", "interleaved"])
def test_u8_call_with_element_offsets_past_2_31(pkg, interleaved):
    """One-byte samples keep a caller buffer of more than 2^31 elements near 2 GB.  Input and output both put samples past
    element 2^31 (planar: channel 1 starts there; interleaved: a frame stride of 2^19 + 1 puts frames >= 4096 there), and
    every call must be bit-identical to the same channels run on compact buffers in a twin batch."""
    import torch
    src, dst, L, n_ch = 44100.0, 48000.0, 4200, 2
    plan = pkg.Plan(src, dst, L, 2.0, A24)
    cap = plan.max_out_len
    si = so = 2 ** 19 + 1 if interleaved else 2 ** 31 + 64
    n_in = (L - 1) * si + n_ch if interleaved else si + L
    n_out = (cap - 1) * so + n_ch if interleaved else so + cap
    big_in = _device_buffer(n_in, 128)
    big_out = _device_buffer(n_out, 0)
    S, T = pkg.Batch(plan, n_ch, 0), pkg.Batch(plan, n_ch, 0)
    small_in = torch.empty((L, n_ch) if interleaved else (n_ch, L), dtype=torch.uint8, device="cuda:0")
    small_out = torch.zeros((cap, n_ch) if interleaved else (n_ch, cap), dtype=torch.uint8, device="cuda:0")
    rng = np.random.default_rng(41)
    past = False
    for k in range(3):
        x = torch.from_numpy(rng.integers(0, 256, (n_ch, L), dtype=np.uint8)).cuda()
        _view(big_in, n_ch, L, si, interleaved).copy_(x)
        (small_in.T if interleaved else small_in).copy_(x)
        n = S.process_fmt(pkg.Buffer.make(big_in.data_ptr(), pkg.U8, interleaved, si, 1.0 / 128),
                          L, pkg.Buffer.make(big_out.data_ptr(), pkg.U8, interleaved, so, 128.0), cap, host=False)
        nt = T.process_fmt(pkg.Buffer.make(small_in.data_ptr(), pkg.U8, interleaved, n_ch if interleaved else L, 1.0 / 128),
                           L, pkg.Buffer.make(small_out.data_ptr(), pkg.U8, interleaved, n_ch if interleaved else cap, 128.0),
                           cap, host=False)
        assert n == nt
        ys = _view(big_out, n_ch, n, so, interleaved).cpu().numpy()
        yt = (small_out[:n].T if interleaved else small_out[:, :n]).cpu().numpy()
        for c in range(n_ch):
            assert_bits(ys[c], yt[c], "call %d channel %d" % (k, c))
        past = past or (n - 1) * so + n_ch - 1 >= 2 ** 31
    assert past and n_in - 1 >= 2 ** 31
    del big_in, big_out
    torch.cuda.empty_cache()


def test_dsd_call_of_2_31_bits(pkg):
    """One DSD64 call of R8BGPU_MAX_LEN = 2^31 - 2^16 bits (256 MB) through 2822400 -> 44100 at that MaxInLen, against the
    same bits fed in 2^20-bit calls on a twin batch: equal totals, values within the parity bar."""
    import torch
    src, dst = 2822400.0, 44100.0
    M, m = 2 ** 31 - 2 ** 16, 2 ** 20
    plan, small = pkg.Plan(src, dst, M, 2.0, A24), pkg.Plan(src, dst, m, 2.0, A24)
    cap, cap_s = plan.max_out_len, small.max_out_len
    g = torch.Generator(device="cuda:0").manual_seed(43)
    try:
        B = pkg.Batch(plan, 1, 0)
        bits = torch.randint(0, 256, (M // 8,), dtype=torch.uint8, device="cuda:0", generator=g)
        y = torch.empty(cap, dtype=torch.float64, device="cuda:0")
        yt = torch.empty(cap + cap_s, dtype=torch.float64, device="cuda:0")
    except (torch.cuda.OutOfMemoryError, pkg.R8bGpuError) as e:
        if "memory" not in str(e):
            raise
        torch.cuda.empty_cache()
        pytest.skip("no room on the device: %s" % e)
    T = pkg.Batch(small, 1, 0)
    y_s = torch.empty(cap_s, dtype=torch.float64, device="cuda:0")
    B.set_stream(0)
    T.set_stream(0)
    n = B.process_fmt(pkg.Buffer.make(bits.data_ptr(), pkg.DSD_LSB, False, M // 8, 0.5), M,
                      pkg.Buffer.make(y.data_ptr(), pkg.F64, False, cap, 1.0), cap, host=False)
    got = 0
    bo = pkg.Buffer.make(y_s.data_ptr(), pkg.F64, False, cap_s, 1.0)
    for off in range(0, M, m):
        l = min(m, M - off)
        k = T.process_fmt(pkg.Buffer.make(bits.data_ptr() + off // 8, pkg.DSD_LSB, False, m // 8, 0.5), l, bo, cap_s,
                          host=False)
        yt[got:got + k].copy_(y_s[:k])
        got += k
    assert n == got == chain_total(plan.stages(), M) > 2 ** 24
    assert list(B.channel_totals()[1]) == list(T.channel_totals()[1]) == [n]
    mx, rms = ou.parity_metrics(y[:n].cpu().numpy(), yt[:n].cpu().numpy())
    assert mx <= 32 * ou.EPS and rms <= 4 * ou.EPS, (mx / ou.EPS, rms / ou.EPS)
    del bits, y, yt, y_s, B
    torch.cuda.empty_cache()
