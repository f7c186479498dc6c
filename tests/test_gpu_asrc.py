"""GPU: trim plans for every rate pair (Plan.asrc) -- drift compensation on same-rate and integer-ratio links.

Yardsticks:
  - a constant factor per channel equals the reference at (src, fl(dst * f)) where the ordinary planner builds the
    forced chain's stages with the same data (counts equal, max|d| <= 32 eps, rms <= 4 eps);
  - every forced chain, at f = 1 exactly, at a constant f and under a factor that changes every call, matches an oracle
    built from the reference's own stage classes around a long-double restatement of convolve2 at the restated timing;
  - lock-step calls equal ragged calls bit for bit (fp64 and int16 output) where both run the same unfused stages,
    and meet the stage oracle wherever the fused kernels run;
  - on pairs Plan.trim accepts, an asrc batch is a trim batch, bytes and state blobs alike;
  - a 48000 -> 48000 stream moves between slots and batches bit for bit, and a passthrough batch refuses its blob;
  - the ordinary parts of a mixed batch are unaffected by an asrc part of the same rates;
  - R8BGPU_DEVICE_ALL routes per-channel factors to the shards and gives a single-device batch's bytes;
  - a flush to an explicit target equals the oracle's output up to the target, and the channel restarts."""
import numpy as np
import pytest

import oracle_util as ou
from test_asrc_cpu import FORCED, PAIRS, restate_chain
from test_gpu_trim import blocks, parity
from test_trim_cpu import A16, A24, random_walk

pytestmark = pytest.mark.gpu


# ---- the stage-built oracle --------------------------------------------------------------------------------------------

def stage_objects(ref, plan, src, dst, tb, atten):
    """The reference's stage classes for the stages before and after the interpolator (CDSPResampler.h:218-393 with
    the forced interpolator), and the interpolator's bank."""
    st = plan.stages()
    k = next(i for i, s in enumerate(st) if s["name"] == "frac_poly")
    n_down = sum(s["name"] == "hbdown" for s in st)
    third = dst * (1 << n_down) * 3.0 <= src  # the decimating branch's IsThird (NormFreq * 3 <= 1)
    pre, post = [], []
    for i, s in enumerate(st):
        if s["name"] == "hbdown":
            pre.append(ref.stage_hbdown(atten, n_down - 1 - i, third))
        elif s["name"] == "blockconv" and i < k:
            if s["up"] == 2:
                pre.append(ref.stage_blockconv(0.5 if dst >= src else 0.5 * dst / src, tb, atten, 2.0, 2, 1))
            else:
                pre.append(ref.stage_blockconv(dst * (1 << n_down) / src, tb, atten, 0.5 ** n_down, 1, 1))
        elif s["name"] == "blockconv":  # behind the interpolator: 2x, transition band from the intermediate rate
            div = (FORCED[(src, dst, tb)][1][0] / 2.0) / src
            post.append(ref.stage_blockconv(0.5, min(45.0, (1.0 - src * div / dst) / 0.0175), atten, 2.0, 2, 1))
        elif s["name"] == "hbup":
            post.append(ref.stage_hbup(atten, i - k - 2, False))
    bank = ref.fracbank(-1, 3, 8, atten, third)
    assert bank["filter_len"] == st[k]["kernel_len"]
    return pre, post, bank


def convolve2(bank, z, outs):
    """The order-2 interpolation (CDSPFracInterpolator.h:1069-1179) in long double at read positions outs."""
    flen = bank["filter_len"]
    tab = bank["table"].astype(np.longdouble)
    P = np.array([p for p, _ in outs], dtype=np.int64)
    F = np.array([f for _, f in outs], dtype=np.float64)
    xf = F * bank["fracs"]
    fti = xf.astype(np.int64)
    xr = (xf - fti).astype(np.longdouble)
    fll = flen // 2 - 1
    zp = np.concatenate([np.zeros(flen), z, np.zeros(flen)]).astype(np.longdouble)
    y = np.empty(len(P), dtype=np.longdouble)
    for a in range(0, len(P), 8192):
        s = slice(a, a + 8192)
        rows = tab[fti[s]]
        coef = rows[..., 0] + rows[..., 1] * xr[s, None] + rows[..., 2] * (xr[s, None] * xr[s, None])
        idx = (P[s, None] - fll + np.arange(flen)[None, :]) + flen
        y[s] = np.sum(coef * zp[idx], axis=1)
    return y.astype(np.float64)


def oracle(ref, plan, src, dst, tb, atten, xs, factors):
    """Per-call outputs of one channel fed blocks xs[i] after factor factors[i] was set."""
    pre, post, bank = stage_objects(ref, plan, src, dst, tb, atten)
    z = []
    for x in xs:
        for s in pre:
            x = s.process(x)
        z.append(x)
    z = np.concatenate(z)
    outs, fc = [], []
    counts, _, _ = restate_chain(plan, dst, [len(x) for x in xs], factors, outs, fc)
    y = convolve2(bank, z, outs)
    got, a = [], 0
    for n in fc:
        v = y[a:a + n]
        a += n
        for s in post:
            v = s.process(v)
        got.append(v)
    assert [len(v) for v in got] == counts
    return got


def feed(rng, n_calls, n_ch, M, seed):
    lens = blocks(rng, n_calls, n_ch, M)
    x = ou.white_noise(n_ch, int(lens.sum(axis=0).max()) + 1, seed=seed)
    return lens, x


def run_ragged(b, x, lens, fs=None):
    """Ragged calls; fs[i] (per channel) set before call i.  Returns per channel the list of per-call outputs."""
    n_ch = x.shape[0]
    pos = np.zeros(n_ch, dtype=np.int64)
    got = [[] for _ in range(n_ch)]
    for i, l in enumerate(lens):
        if fs is not None:
            b.set_trim(np.arange(n_ch), fs[i])
        for c, y in enumerate(b.process_ragged([x[c, pos[c]:pos[c] + l[c]] for c in range(n_ch)])):
            got[c].append(y)
        pos += l
    return got


# ---- 1. constant factors against the reference -------------------------------------------------------------------------

# pairs and sides where the ordinary planner at (src, fl(dst * f)) builds the forced chain's stages and data
# (test_asrc_cpu.SAME_DATA_SIDES)
CONSTANT = [(48000.0, 48000.0, 1.0, 1.002), (44100.0, 88200.0, 0.998, 1.002), (32000.0, 48000.0, 0.998, 1.002)]


@pytest.mark.parametrize("atten", [A16, A24])
@pytest.mark.parametrize("src,dst,lo,hi", CONSTANT)
def test_constant_factors_match_the_reference(pkg, ref, src, dst, lo, hi, atten):
    M, n_ch, n_calls, tb = 4096, 6, 10, 2.0
    ap = pkg.Plan.asrc(src, dst, M, tb, atten, 0.002)
    rng = np.random.default_rng(int(src + dst + atten))
    fs = rng.uniform(lo, hi, n_ch)
    fs = np.where(fs == 1.0, hi, fs)
    for f in fs:
        op = pkg.Plan(src, dst * f, M, tb, atten)
        assert [s["name"] for s in op.stages()] == [s["name"] for s in ap.stages()]
        assert all(op.stage_data(i).tobytes() == ap.stage_data(i).tobytes() for i in range(len(op.stages())))
    b = pkg.Batch(ap, n_ch, 0)
    b.set_trim(np.arange(n_ch), fs)
    lens, x = feed(rng, n_calls, n_ch, M, 3)
    got = run_ragged(b, x, lens)
    pos = np.zeros(n_ch, dtype=np.int64)
    for c in range(n_ch):
        r = ref.Resampler(src, dst * fs[c], M, tb, atten)
        want = []
        for l in lens[:, c]:
            want.append(r.process(x[c, pos[c]:pos[c] + l]))
            pos[c] += l
        assert [len(v) for v in got[c]] == [len(v) for v in want]
        parity(np.concatenate(got[c]), np.concatenate(want))


# ---- 2. every forced chain against the stage-built oracle --------------------------------------------------------------

CHAINS = [(s, d, 2.0) for s, d in PAIRS] + [(44100.0, 352800.0, 40.0)]


@pytest.mark.parametrize("src,dst,tb", CHAINS)
def test_forced_chain_matches_the_stage_oracle(pkg, ref, src, dst, tb):
    """Channel 0 at f = 1 exactly, channel 1 at a constant factor, channels 2 and 3 under factors that change every
    call; ragged calls (every channel its own group, k_frac<true>)."""
    M, n_ch, n_calls = 2048, 4, 24
    ap = pkg.Plan.asrc(src, dst, M, tb, A24, 2e-4)
    rng = np.random.default_rng(int(src * 3 + dst + tb))
    fs = np.stack([np.ones(n_calls), np.full(n_calls, 1.0 - 1.3e-4)] +
                  [random_walk(rng, n_calls) for _ in range(n_ch - 2)], axis=1)
    lens, x = feed(rng, n_calls, n_ch, M, 9)
    b = pkg.Batch(ap, n_ch, 0)
    got = run_ragged(b, x, lens, fs)
    for c in range(n_ch):
        xs = np.split(x[c, :lens[:, c].sum()], np.cumsum(lens[:, c])[:-1])
        want = oracle(ref, ap, src, dst, tb, A24, xs, fs[:, c])
        assert [len(v) for v in got[c]] == [len(v) for v in want], c
        parity(np.concatenate(got[c]), np.concatenate(want))


# ---- 3. lock-step against ragged ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("fusion", ["default", "off"])
@pytest.mark.parametrize("src,dst,tb", CHAINS)
def test_lockstep_equals_ragged(pkg, ref, src, dst, tb, fusion, monkeypatch):
    """All channels share one factor (1, then a trimmed one, then another) and equal lengths.  The lock-step batch runs
    the lock-step kernels; the ragged batch carries one more channel fed other lengths, so it stays diverged and runs the
    ragged kernels.  Where both run the same unfused stages (the 1x chains, and every chain with R8BGPU_NO_FUSION) they
    agree bit for bit, fp64 and int16; the fused kernels' own FFT tiles round differently (DESIGN.md section 7), so
    there both meet the stage oracle at the parity bar."""
    if fusion == "off":
        monkeypatch.setenv("R8BGPU_NO_FUSION", "1")
    M, n_ch, n_calls = 2048, 3, 12
    ap = pkg.Plan.asrc(src, dst, M, tb, A24, 2e-4)
    exact = all(ap.fused_info(i)["kernel"] == "none" for i, s in enumerate(ap.stages()) if s["name"] == "blockconv")
    assert exact or fusion == "default"
    lk, rg = pkg.Batch(ap, n_ch, 0), pkg.Batch(ap, n_ch + 1, 0)
    lk16, rg16 = pkg.Batch(ap, n_ch, 0), pkg.Batch(ap, n_ch + 1, 0)
    rng = np.random.default_rng(int(src + dst))
    x = ou.white_noise(n_ch + 1, n_calls * M, seed=4)
    xi = (x * 30000).astype(np.int16)
    pos, extra = 0, 0
    fs, ls, got = [], [], [[] for _ in range(n_ch)]
    for i in range(n_calls):
        f = 1.0 if i < 4 else (1.0 + 1.7e-4 if i < 8 else 1.0 - 0.6e-4)
        for b in (lk, lk16):
            b.set_trim(np.arange(n_ch), np.full(n_ch, f))
        for b in (rg, rg16):
            b.set_trim(np.arange(n_ch + 1), np.full(n_ch + 1, f))
        l = int(rng.integers(1, M + 1))
        e = int(rng.integers(0, M + 1))
        e = e if e != l else l - 1
        ya = lk.process_host(x[:n_ch, pos:pos + l])
        yr = rg.process_ragged([x[c, pos:pos + l] for c in range(n_ch)] + [x[n_ch, extra:extra + e]])
        assert rg.channel_groups > 1 and lk.channel_groups == 1
        for c in range(n_ch):
            assert len(ya[c]) == len(yr[c])
            if exact:
                assert ya[c].tobytes() == yr[c].tobytes(), (i, c)
            got[c].append(ya[c])
        if exact:
            lens = np.array([l] * n_ch + [e], dtype=np.int32)
            xin = np.zeros((n_ch + 1, M), np.int16)
            xin[:n_ch, :l] = xi[:n_ch, pos:pos + l]
            xin[n_ch, :e] = xi[n_ch, extra:extra + e]
            qa = lk16.process_host_fmt(xi[:n_ch, pos:pos + l].copy(), out_dtype=np.int16, out_scale=30000.0)
            qr, cr = rg16.process_ragged_fmt(xin, lens, out_dtype=np.int16, out_scale=30000.0)
            for c in range(n_ch):
                assert cr[c] == qa.shape[1] == ya.shape[1]
                assert qa[c].tobytes() == qr[c, :cr[c]].tobytes(), (i, c)
        fs.append(f)
        ls.append(l)
        pos += l
        extra += e
    for c in range(n_ch):
        want = oracle(ref, ap, src, dst, tb, A24, np.split(x[c, :pos], np.cumsum(ls)[:-1]), fs)
        assert [len(v) for v in got[c]] == [len(v) for v in want]
        parity(np.concatenate(got[c]), np.concatenate(want))


# ---- 4. same plan, same bits ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("src,dst", [(44100.0, 48000.0), (48000.0, 44100.0)])
def test_asrc_batch_is_the_trim_batch(pkg, src, dst):
    M, n_ch, n_calls = 2048, 4, 10
    ap, tp = pkg.Plan.asrc(src, dst, M, 2.0, A24, 2e-4), pkg.Plan.trim(src, dst, M, 2.0, A24, 2e-4)
    assert ap.state_fingerprint == tp.state_fingerprint
    a, t = pkg.Batch(ap, n_ch, 0), pkg.Batch(tp, n_ch, 0)
    rng = np.random.default_rng(5)
    fs = np.stack([random_walk(rng, 2 * n_calls) for _ in range(n_ch)], axis=1)
    lens, x = feed(rng, 2 * n_calls, n_ch, M, 6)
    ga = run_ragged(a, x, lens[:n_calls], fs[:n_calls])
    gt = run_ragged(t, x, lens[:n_calls], fs[:n_calls])
    for c in range(n_ch):
        assert b"".join(v.tobytes() for v in ga[c]) == b"".join(v.tobytes() for v in gt[c])
    # blobs cross over: the trim batch continues the asrc batch's streams, and the other way round
    a2, t2 = pkg.Batch(ap, n_ch, 0), pkg.Batch(tp, n_ch, 0)
    a2.import_channels(list(range(n_ch)), t.export_channels(list(range(n_ch))))
    t2.import_channels(list(range(n_ch)), a.export_channels(list(range(n_ch))))
    pos = lens[:n_calls].sum(axis=0)
    xr = np.stack([np.concatenate([x[c, pos[c]:], np.zeros(pos[c])]) for c in range(n_ch)])
    for b1, b2 in ((a, t2), (t, a2)):
        g1 = run_ragged(b1, xr, lens[n_calls:], fs[n_calls:])
        g2 = run_ragged(b2, xr, lens[n_calls:], fs[n_calls:])
        for c in range(n_ch):
            assert b"".join(v.tobytes() for v in g1[c]) == b"".join(v.tobytes() for v in g2[c])


# ---- 5. moving a 48000 -> 48000 stream -----------------------------------------------------------------------------------

def test_same_rate_stream_moves(pkg):
    M = 2048
    ap = pkg.Plan.asrc(48000.0, 48000.0, M, 2.0, A24, 2e-4)
    A, B = pkg.Batch(ap, 3, 0), pkg.Batch(ap, 5, 0)
    rng = np.random.default_rng(12)
    x = ou.white_noise(5, 20 * M, seed=8)
    for i in range(4):
        A.set_trim([0, 1, 2], random_walk(rng, 3))
        A.process_ragged([x[c, i * M:i * M + 1500 + 100 * c] for c in range(3)])
    blob = A.export_channels([1])
    A.import_channels([2], blob)  # another slot of the same batch
    B.import_channels([4], blob)  # another batch
    assert A.trim()[2] == A.trim()[1] == B.trim()[4]
    xa = x[:3, 10 * M:]
    for i in range(6):
        f = 1.0 + 1e-5 * (i - 3)
        A.set_trim([1, 2], [f, f])
        B.set_trim([4], [f])
        l = int(rng.integers(0, M + 1))
        ya = A.process_ragged([xa[0, :l], xa[1, :l], xa[1, :l]])
        yb = B.process_ragged([np.zeros(7)] * 4 + [xa[1, :l]])
        assert ya[1].tobytes() == ya[2].tobytes() == yb[4].tobytes()
        xa = xa[:, l:]
    pp = pkg.Batch(pkg.Plan(48000.0, 48000.0, M, 2.0, A24), 2, 0)
    with pytest.raises(pkg.R8bGpuError, match="fingerprint"):
        pp.import_channels([0], blob)
    with pytest.raises(pkg.R8bGpuError, match="truncated blob"):  # (a passthrough stream's blob is shorter)
        A.import_channels([0], pp.export_channels([1]))


# ---- 6. mixed batch ------------------------------------------------------------------------------------------------------

def test_mixed_batch_with_a_passthrough_part_of_the_same_rates(pkg):
    M = 2048
    ap = pkg.Plan.asrc(48000.0, 48000.0, M, 2.0, A24, 2e-4)
    pp = pkg.Plan(48000.0, 48000.0, M, 2.0, A24)
    op = pkg.Plan(44100.0, 48000.0, M, 2.0, A24)
    po = np.array([0, 1, 2, 0, 1, 2, 1], dtype=np.int32)
    mb = pkg.Batch.mixed([ap, pp, op], po, 0)
    alone = [pkg.Batch(ap, 2, 0), pkg.Batch.mixed([pp], np.zeros(3, np.int32), 0), pkg.Batch.mixed([op], np.zeros(2, np.int32), 0)]
    chans = [np.nonzero(po == p)[0] for p in range(3)]
    rng = np.random.default_rng(21)
    x = ou.white_noise(7, 12 * M, seed=13)
    pos = np.zeros(7, dtype=np.int64)
    for i in range(8):
        f = random_walk(rng, 2)
        mb.set_trim(chans[0], f)
        alone[0].set_trim([0, 1], f)
        lens = blocks(rng, 1, 7, M)[0]
        xs = [x[c, pos[c]:pos[c] + lens[c]] for c in range(7)]
        ys = mb.process_ragged(xs)
        for p in range(3):
            ya = alone[p].process_ragged([xs[c] for c in chans[p]])
            for k, c in enumerate(chans[p]):
                assert ys[c].tobytes() == ya[k].tobytes(), (i, p, c)
        pos += lens
    for c in chans[1]:  # the passthrough part hands its input back
        assert mb.channel_totals()[1][c] == pos[c]


# ---- 7. R8BGPU_DEVICE_ALL ------------------------------------------------------------------------------------------------

def test_device_all_routes_factors_to_the_shards(pkg, monkeypatch):
    monkeypatch.setenv("R8BGPU_FORCE_SHARDS", "3")
    M, n_ch = 2048, 7
    ap = pkg.Plan.asrc(44100.0, 88200.0, M, 2.0, A24, 1e-3)
    front, one = pkg.Batch(ap, n_ch, pkg.DEVICE_ALL), pkg.Batch(ap, n_ch, 0)
    assert [s[1] for s in front.shards()] == [0, 3, 6]
    rng = np.random.default_rng(31)
    x = ou.white_noise(n_ch, 10 * M, seed=14)
    pos = np.zeros(n_ch, dtype=np.int64)
    order = np.array([6, 2, 4, 0, 5, 1, 3])
    for i in range(6):
        f = 1.0 + rng.uniform(-1e-3, 1e-3, n_ch)
        front.set_trim(order, f)
        one.set_trim(order, f)
        assert front.trim().tobytes() == one.trim().tobytes()
        lens = rng.integers(0, M + 1, n_ch)
        xs = [x[c, pos[c]:pos[c] + lens[c]] for c in range(n_ch)]
        for c, (a, b) in enumerate(zip(front.process_ragged(xs), one.process_ragged(xs))):
            assert a.tobytes() == b.tobytes(), (i, c)
        pos += lens
    for a, b in zip(front.channel_totals(), one.channel_totals()):
        assert a.tobytes() == b.tobytes()


# ---- 8. flush to an explicit target ---------------------------------------------------------------------------------------

def test_flush_to_explicit_targets(pkg, ref):
    M, n_ch = 2048, 3
    src = dst = 48000.0
    ap = pkg.Plan.asrc(src, dst, M, 2.0, A24, 2e-4)
    b = pkg.Batch(ap, n_ch, 0)
    rng = np.random.default_rng(41)
    n_calls = 6
    fs = np.stack([np.ones(n_calls), np.full(n_calls, 1.0 + 1.1e-4), random_walk(rng, n_calls)], axis=1)
    lens, x = feed(rng, n_calls, n_ch, M, 15)
    got = run_ragged(b, x, lens, fs)
    with pytest.raises(pkg.R8bGpuError, match="explicit"):
        b.flush([0])
    _, n_out = b.channel_totals()
    extra = np.array([3000, 1, 4500])
    y, cnt = b.flush([0, 1, 2], targets=n_out + extra)
    assert list(cnt) == list(extra)
    for c in range(n_ch):
        xs = np.split(x[c, :lens[:, c].sum()], np.cumsum(lens[:, c])[:-1])
        # the flush feeds silence at the last factor until the target is reached
        zeros = [np.zeros(M)] * 8
        want = oracle(ref, ap, src, dst, 2.0, A24, xs + zeros, np.concatenate([fs[:, c], np.full(8, fs[-1, c])]))
        want = np.concatenate(want)
        assert len(want) >= n_out[c] + extra[c]
        want = want[:n_out[c] + extra[c]]
        assert sum(len(v) for v in got[c]) == n_out[c]
        parity(np.concatenate(got[c] + [y[c, :cnt[c]]]), want)
    # the channels restart from clear(), each keeping its factor
    n_in, n_out = b.channel_totals()
    assert np.all(n_in == 0) and np.all(n_out == 0)
    assert b.trim().tobytes() == fs[-1].tobytes()
    y2 = run_ragged(b, x, lens[:3], np.tile(fs[-1], (3, 1)))
    for c in range(n_ch):
        xs = np.split(x[c, :lens[:3, c].sum()], np.cumsum(lens[:3, c])[:-1])
        want = oracle(ref, ap, src, dst, 2.0, A24, xs, np.full(3, fs[-1, c]))
        parity(np.concatenate(y2[c]), np.concatenate(want))
