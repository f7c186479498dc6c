"""GPU: plain fp64 ragged calls on a passthrough plan (equal rates) hand each channel's block back and write nothing past
lens[c] of its output row -- in the device form (r8bgpu_batch_process_ragged) and the host form (_host_ragged), on an
ordinary batch and on a multi-device batch (two shards on one GPU, whose device form runs on each shard)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_CH, MAX_IN = 7, 4096
SENTINEL = -12345.0


def _ok(pkg, rc):
    if rc < 0:
        raise pkg.R8bGpuError(pkg._err())


@pytest.mark.parametrize("shards", [1, 2])
def test_plain_passthrough_writes_nothing_past_lens(pkg, monkeypatch, shards):
    import torch
    if shards > 1:
        monkeypatch.setenv("R8BGPU_FORCE_SHARDS", str(shards))
    plan = pkg.Plan(48000.0, 48000.0, MAX_IN)
    assert plan.passthrough
    device = pkg.DEVICE_ALL if shards > 1 else 0
    host_b, dev_b = pkg.Batch(plan, N_CH, device), pkg.Batch(plan, N_CH, device)
    assert len(dev_b.shards()) == shards
    lib, cap = pkg.lib(), MAX_IN + 64
    rng = np.random.default_rng(41)
    # runs of channels with one block length (one copy each), 0, 1 and MaxInLen
    for lens in ([MAX_IN, MAX_IN, 0, 1, 1, 1, 777], [0, 5, 5, 5, MAX_IN, 0, 0], [MAX_IN] * N_CH):
        lens = np.array(lens, dtype=np.int32)
        x = rng.standard_normal((N_CH, MAX_IN))  # samples past lens[c] too: a copy reading on would carry them over
        yh = np.full((N_CH, cap), SENTINEL)
        ch = np.empty(N_CH, dtype=np.int32)
        _ok(pkg, lib.r8bgpu_batch_process_host_ragged(host_b._h, x.ctypes.data, MAX_IN, lens.ctypes.data, yh.ctypes.data,
                                                      cap, cap, ch.ctypes.data))
        xd = torch.from_numpy(x).cuda()
        yd = torch.full((N_CH, cap), SENTINEL, dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        cd = np.empty(N_CH, dtype=np.int32)
        for s, (_, c0, n, _) in enumerate(dev_b.shards()):
            h = lib.r8bgpu_batch_shard(dev_b._h, s)
            ln, cn = lens[c0:c0 + n].copy(), np.empty(n, dtype=np.int32)
            _ok(pkg, lib.r8bgpu_batch_process_ragged(h, xd[c0].data_ptr(), MAX_IN, ln.ctypes.data, yd[c0].data_ptr(), cap,
                                                     cap, cn.ctypes.data))
            _ok(pkg, lib.r8bgpu_batch_sync(h))
            cd[c0:c0 + n] = cn
        yd = yd.cpu().numpy()
        assert np.array_equal(ch, lens) and np.array_equal(cd, lens)
        assert np.array_equal(yh.view(np.uint64), yd.view(np.uint64))
        for c in range(N_CH):
            assert np.array_equal(yh[c, :lens[c]], x[c, :lens[c]]), c
            assert np.all(yh[c, lens[c]:] == SENTINEL), ("written past lens[c]", c, int(lens[c]))
