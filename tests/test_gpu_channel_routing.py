"""GPU: per-channel calls on a multi-device batch route each channel to the shard that runs it.

R8BGPU_FORCE_SHARDS deals three shards to one device (7 channels: rows 0-2, 3-5 and 6), so the front's routing runs on a
one-GPU box.  Yardsticks:
  - per-channel trim factors named in scrambled order across shards, and a clear_channels that names a channel twice,
    give the trim factors, channel totals and ragged outputs of an ordinary batch fed the same calls, bit for bit;
  - a channel named twice is refused with the caller's channel number by set_trim, set_dither and flush, and the refused
    call changes nothing."""
import numpy as np
import pytest

import oracle_util as ou
from test_trim_cpu import A24

pytestmark = pytest.mark.gpu

M, N_CH = 2048, 7


def _pair(pkg, monkeypatch):
    monkeypatch.setenv("R8BGPU_FORCE_SHARDS", "3")
    tp = pkg.Plan.trim(44100.0, 48000.0, M, 2.0, A24, 1e-3)
    front, one = pkg.Batch(tp, N_CH, pkg.DEVICE_ALL), pkg.Batch(tp, N_CH, 0)
    assert [s[1] for s in front.shards()] == [0, 3, 6]
    return front, one


def _same(front, one):
    assert front.trim().tobytes() == one.trim().tobytes()
    for a, b in zip(front.channel_totals(), one.channel_totals()):
        assert a.tobytes() == b.tobytes()


def _run(front, one, x, pos, lens):
    xs = [x[c, pos[c]:pos[c] + lens[c]] for c in range(N_CH)]
    ya, yb = front.process_ragged(xs), one.process_ragged(xs)
    for c in range(N_CH):
        assert ya[c].tobytes() == yb[c].tobytes(), c
    pos += lens
    _same(front, one)


def test_trim_and_clear_route_like_an_ordinary_batch(pkg, monkeypatch):
    front, one = _pair(pkg, monkeypatch)
    rng = np.random.default_rng(11)
    x = ou.white_noise(N_CH, 12 * M, seed=5)
    pos = np.zeros(N_CH, dtype=np.int64)
    order = np.array([5, 0, 6, 3, 1, 4, 2])  # every shard, out of order
    for i in range(4):
        f = 1.0 + rng.uniform(-1e-3, 1e-3, N_CH)
        front.set_trim(order, f)
        one.set_trim(order, f)
        _same(front, one)
        _run(front, one, x, pos, rng.integers(0, M + 1, N_CH))
    for named in ([4, 1, 4], [6, 2, 6, 5]):  # one index named twice
        front.clear_channels(named)
        one.clear_channels(named)
        pos[named] = 0
        _same(front, one)
        for i in range(2):
            _run(front, one, x, pos, rng.integers(0, M + 1, N_CH))


def test_a_channel_named_twice_is_refused_with_the_callers_number(pkg, monkeypatch):
    front, _ = _pair(pkg, monkeypatch)
    x = ou.white_noise(N_CH, M, seed=6)
    front.set_trim(np.arange(N_CH), 1.0 + 1e-4 * np.arange(N_CH))
    front.process_ragged(list(x))
    trim, (n_in, n_out) = front.trim(), front.channel_totals()
    c = 4  # row 1 of the shard that starts at channel 3
    calls = [lambda: front.set_trim([c, c], [1.0, 1.0]),
             lambda: front.set_dither([c, c], 7),
             lambda: front.flush([c, c], targets=n_out[[c, c]] + 100)]
    for call in calls:
        with pytest.raises(pkg.R8bGpuError, match="channel %d named twice" % c):
            call()
        assert front.trim().tobytes() == trim.tobytes()
        got_in, got_out = front.channel_totals()
        assert got_in.tobytes() == n_in.tobytes() and got_out.tobytes() == n_out.tobytes()
