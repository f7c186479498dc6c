"""GPU: independent streams in one batch -- a block length per channel per call (process_ragged) and per-channel
clear() (clear_channels) -- against one compiled reference object per channel fed the same chunking.  Per-call counts
must be exactly equal; per channel max|d| <= 32 eps and rms(d) <= 4 eps (the parity bar of test_gpu_parity.py)."""
import numpy as np
import pytest

import oracle_util as ou
from test_gpu_parity import CHAINS

pytestmark = pytest.mark.gpu

LARGE = "k_bcl_gather+k_bcl_conv+k_bcl_scatter"


def _oracle(ext):
    flavor = "e1" if ext else "e0"
    if not ou.have_ref(flavor):
        pytest.skip("oracle/_ref not built (needs /root/reference at build time)")
    return ou.RefOracle(flavor)


class Streams:
    """A batch of independent streams next to one reference object per channel; feeds both and keeps the outputs."""

    def __init__(self, pkg, src, dst, max_in, n_ch, tb=2.0, atten=180.15, ext=0, device=0, seed=3, total=None):
        self.pkg, self.ref = pkg, _oracle(ext)
        self.args = (src, dst, max_in, tb, atten)
        self.plan = pkg.Plan(src, dst, max_in, tb, atten, extfft=ext)
        self.batch = pkg.Batch(self.plan, n_ch, device)
        self.n_ch = n_ch
        self.rs = [self.ref.Resampler(*self.args) for _ in range(n_ch)]
        self.x = ou.white_noise(n_ch, total or max_in * 40, seed)
        self.pos = [0] * n_ch
        self.got = [[] for _ in range(n_ch)]
        self.want = [[] for _ in range(n_ch)]

    def _blocks(self, lens):
        xs = []
        for c, l in enumerate(lens):
            xs.append(self.x[c, self.pos[c]:self.pos[c] + l])
            self.pos[c] += l
            assert len(xs[-1]) == l, "test signal too short"
        return xs

    def _keep(self, xs, ys):
        for c in range(self.n_ch):
            r = self.rs[c].process(xs[c])
            assert len(r) == len(ys[c]), "channel %d: ref %d gpu %d (l=%d)" % (c, len(r), len(ys[c]), len(xs[c]))
            self.got[c].append(np.asarray(ys[c]))
            self.want[c].append(r)

    def ragged(self, lens, device=False):
        xs = self._blocks(lens)
        if device:
            import torch
            ys = self.batch.process_ragged([torch.from_numpy(x.copy()).cuda() for x in xs])
            ys = [y.cpu().numpy() for y in ys]
        else:
            ys = self.batch.process_ragged([x.copy() for x in xs])
        self._keep(xs, ys)

    def lockstep(self, l):
        xs = self._blocks([l] * self.n_ch)
        y = self.batch.process_host(np.stack(xs))
        self._keep(xs, list(y))

    def clear(self, channels):
        self.batch.clear_channels(channels)
        for c in channels:
            self.rs[c] = self.ref.Resampler(*self.args)  # a fresh object, as after CDSPResampler::clear()
            self.got[c].append(None)
            self.want[c].append(None)

    def check(self):
        """Parity of every channel over each stretch between its clears."""
        n = 0
        for c in range(self.n_ch):
            for seg_g, seg_w in zip(self._segments(self.got[c]), self._segments(self.want[c])):
                a, b = np.concatenate(seg_g), np.concatenate(seg_w)
                assert len(a) == len(b)
                if len(b) == 0 or not np.any(b):
                    assert not np.any(a)
                    continue
                m, r = ou.parity_metrics(a, b)
                assert m <= 32 * ou.EPS and r <= 4 * ou.EPS, (self.args, c, m / ou.EPS, r / ou.EPS)
                n += 1
        assert n > 0

    @staticmethod
    def _segments(parts):
        seg = [np.zeros(0)]
        for p in parts:
            if p is None:
                yield seg
                seg = [np.zeros(0)]
            else:
                seg.append(p)
        yield seg


def ragged_lens(rng, n_calls, n_ch, max_in):
    lens = rng.integers(0, max_in + 1, size=(n_calls, n_ch))
    for c in range(n_ch):
        rows = rng.choice(n_calls, 3, replace=False)
        lens[rows, c] = (0, 1, max_in)
    return lens


@pytest.mark.parametrize("src,dst", CHAINS)
def test_chain_ragged_parity(pkg, src, dst):
    s = Streams(pkg, src, dst, 8192, 3)
    rng = np.random.default_rng(int(src + dst))
    for i, lens in enumerate(ragged_lens(rng, 8, 3, 8192)):
        s.ragged(list(lens), device=bool(i & 1))
    s.check()


def test_large_tile_chain(pkg):
    s = Streams(pkg, 48000.0, 16000.0, 65536, 3, tb=0.5)
    assert LARGE in [k for k, _ in s.batch.stage_kernels()]
    for lens in ([65536, 0, 30000], [1, 65536, 65536], [4000, 9000, 1], [65536, 65536, 65536], [0, 777, 65536]):
        s.ragged(lens)
    s.check()


def test_large_tile_several_scratch_groups(pkg, monkeypatch):
    # a 1 MB scratch holds one channel's tile pair of 65536 points: every run of channels is cut into groups of one
    monkeypatch.setenv("R8BGPU_BCL_SCRATCH_MB", "1")
    s = Streams(pkg, 48000.0, 16000.0, 65536, 4, tb=0.5)
    for lens in ([65536, 65536, 30000, 30000], [65536, 1, 65536, 65536], [5000, 5000, 5000, 0]):
        s.ragged(lens, device=True)
    s.check()


def test_hbdown_cascade(pkg):
    s = Streams(pkg, 2822400.0, 44100.0, 65536, 3, total=65536 * 8)
    assert s.batch.stage_kernels()[0] == ("k_hbdown_cascade", 5)
    for lens in ([65536, 1000, 65536], [7, 65536, 0], [65536, 65536, 33333], [65536, 0, 65536], [65536] * 3):
        s.ragged(lens)
    s.check()


def test_hbup_cascade_64x(pkg):
    s = Streams(pkg, 44100.0, 2822400.0, 2048, 3, ext=1)
    assert "k_hbup_cascade" in [k for k, _ in s.batch.stage_kernels()]
    for lens in ([2048, 100, 0], [1, 2048, 2048], [2048, 2048, 777], [2048, 5, 2048], [2048] * 3):
        s.ragged(lens, device=True)
    s.check()


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_ragged_sweep(pkg, seed):
    rng = np.random.default_rng(seed)
    src, dst = CHAINS[int(rng.integers(len(CHAINS)))]
    n_ch = int(rng.integers(2, 9))
    s = Streams(pkg, src, dst, 4096, n_ch, seed=seed)
    for i, lens in enumerate(ragged_lens(rng, 10, n_ch, 4096)):
        s.ragged(list(lens), device=bool(i % 3 == 0))
    s.check()


def test_idle_channels(pkg):
    """Channels that receive nothing for several calls while the others run, then resume."""
    s = Streams(pkg, 44100.0, 96000.0, 8192, 4)
    for _ in range(4):
        s.ragged([8192, 0, 8192, 0])
    for _ in range(3):
        s.ragged([0, 8192, 0, 8192])
    s.ragged([8192, 8192, 1, 0])
    s.check()


@pytest.mark.parametrize("src,dst", [(44100.0, 96000.0), (48000.0, 47999.0), (192000.0, 44100.0)])
def test_clear_channels_mid_stream(pkg, src, dst):
    s = Streams(pkg, src, dst, 8192, 4)
    for lens in ([8192] * 4, [8192, 100, 8192, 5000]):
        s.ragged(lens)
    s.clear([1, 3])
    for lens in ([8192] * 4, [0, 8192, 8192, 1], [8192] * 4):
        s.ragged(lens, device=True)
    s.clear([0])
    s.ragged([4000, 4000, 0, 8192])
    s.check()


def test_alternating_lockstep_and_ragged(pkg):
    s = Streams(pkg, 44100.0, 96000.0, 8192, 3)
    s.lockstep(8192)
    s.ragged([8192, 8192, 8192])
    assert s.batch.channel_groups == 1
    s.ragged([8192, 4000, 0])
    assert s.batch.channel_groups == 3
    # a lock-step call whose counts would differ per channel is refused and changes nothing
    hist = [[8192, 8192, 8192], [8192, 8192, 4000], [8192, 8192, 0]]
    l = next(l for l in range(1, 8193) if len({s.plan.simulate(h + [l])[-1] for h in hist}) > 1)
    before = s.batch.kernel_launches
    with pytest.raises(s.pkg.R8bGpuError, match="diverged"):
        s.batch.process_host(np.zeros((3, l)))
    assert s.batch.kernel_launches == before
    s.ragged([0, 4192, 8192])  # equal totals again: one schedule, lock-step calls run as before
    assert s.batch.channel_groups == 1
    s.lockstep(8192)
    s.ragged([100, 8192, 1])
    s.lockstep(0)
    s.check()


def test_restarted_channel_catches_up(pkg):
    """A channel cleared on its own diverges; once its total equals the others' again the batch is one schedule and
    lock-step calls run as before."""
    s = Streams(pkg, 44100.0, 96000.0, 8192, 3)
    s.lockstep(8192)
    s.clear([2])
    assert s.batch.channel_groups == 2
    s.lockstep(0)  # counts agree (nothing is produced): runs on the diverged batch
    s.ragged([0, 0, 8192])
    assert s.batch.channel_groups == 1
    s.lockstep(8192)
    s.check()


def test_forced_shards_host_ragged(pkg, monkeypatch):
    monkeypatch.setenv("R8BGPU_FORCE_SHARDS", "3")
    s = Streams(pkg, 48000.0, 44100.0, 8192, 7, device=pkg.DEVICE_ALL)
    assert len(s.batch.shards()) == 3
    rng = np.random.default_rng(9)
    for lens in ragged_lens(rng, 6, 7, 8192):
        s.ragged(list(lens))
    s.clear([0, 4, 6])
    s.ragged([8192] * 7)
    s.check()


def test_forced_shards_refused_call_changes_nothing(pkg, monkeypatch):
    """Shards in different states: a lock-step call whose counts differ between shards is refused before any shard runs."""
    monkeypatch.setenv("R8BGPU_FORCE_SHARDS", "2")
    s = Streams(pkg, 44100.0, 96000.0, 8192, 4, device=pkg.DEVICE_ALL)
    s.ragged([8192, 8192, 4000, 4000])
    assert s.batch.channel_groups == 2
    hist = [[8192], [4000]]
    l = next(l for l in range(1, 8193) if len({s.plan.simulate(h + [l])[-1] for h in hist}) > 1)
    before = s.batch.kernel_launches
    with pytest.raises(pkg.R8bGpuError, match="diverged"):
        s.batch.process_host(np.zeros((4, l)))
    assert s.batch.kernel_launches == before
    s.ragged([0, 0, 4192, 4192])
    assert s.batch.channel_groups == 1
    s.lockstep(8192)
    s.check()


def test_one_launch_per_stage(pkg):
    """A ragged call runs every stage once for all channels on its per-channel-record kernel (plus the history copy, and
    once per batch the refill of the links that lock-step calls keep in shared memory)."""
    s = Streams(pkg, 44100.0, 2822400.0, 2048, 16, ext=1)
    ns = len(s.plan.stages())
    s.lockstep(2048)
    rng = np.random.default_rng(4)
    l0 = s.batch.kernel_launches
    s.ragged(list(rng.integers(0, 2049, 16)))
    assert s.batch.kernel_launches - l0 <= 2 * ns + 1
    assert all("ragged" in k for k, _ in s.batch.stage_kernels()), s.batch.stage_kernels()
    l0 = s.batch.kernel_launches
    s.ragged(list(rng.integers(0, 2049, 16)))
    assert s.batch.kernel_launches - l0 <= ns + 1
    s.lockstep(0)
    s.check()


def test_fasttiming_refuses_ragged(pkg):
    plan = pkg.Plan(48000.0, 47999.0, 1024, 2.0, pkg.ATTEN_24, fasttiming=1)
    b = pkg.Batch(plan, 2, 0)
    with pytest.raises(pkg.R8bGpuError, match="FASTTIMING"):
        b.process_ragged([np.zeros(10), np.zeros(20)])
    with pytest.raises(pkg.R8bGpuError, match="FASTTIMING"):
        b.clear_channels([0])
    b.clear_channels([0, 1])  # every channel: an ordinary clear()
