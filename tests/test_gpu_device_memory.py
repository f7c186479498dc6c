"""Batch.device_bytes (r8bgpu_batch_device_bytes) counts every device block a batch holds: it rises when a call first
needs a block, stays put while the same call repeats, and falls back when a feature lets its blocks go.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MAX_IN = 4096
N_CH = 5
DSD_SCALE = 0.5


# integer ratios: once the filter's latency is past, every call of the same block lengths has the same output counts
def _plan(pkg, src=44100.0, dst=88200.0):
    return pkg.Plan(src, dst, MAX_IN, 2.0, pkg.ATTEN_24)


def _x(n_ch, l=MAX_IN, seed=1):
    return np.random.default_rng(seed).uniform(-0.9, 0.9, (n_ch, l))


def _lens(n_ch):
    return np.arange(1, n_ch + 1, dtype=np.int32) * (MAX_IN // (n_ch + 1))


@pytest.fixture
def force_two_shards(monkeypatch):
    monkeypatch.setenv("R8BGPU_FORCE_SHARDS", "2")


def test_export_staging_is_counted(pkg):
    b = pkg.Batch(_plan(pkg), N_CH)
    b.process_ragged_fmt(_x(N_CH), _lens(N_CH))
    before = b.device_bytes
    b.export_channels([0, 2])
    assert b.device_bytes > before


def _lockstep_device(pkg):
    import torch
    b = pkg.Batch(_plan(pkg), N_CH)
    x = torch.from_numpy(_x(N_CH)).cuda()
    return b, lambda: b.process(x)


def _lockstep_host(pkg):
    b = pkg.Batch(_plan(pkg), N_CH)
    x = _x(N_CH)
    return b, lambda: b.process_host(x)


def _ragged_fmt(pkg):
    b = pkg.Batch(_plan(pkg), N_CH)
    x = (_x(N_CH) * 32767).astype(np.int16)
    return b, lambda: b.process_ragged_fmt(x, _lens(N_CH), out_dtype=np.int16)


def _flush(pkg):
    b = pkg.Batch(_plan(pkg), N_CH)
    x = _x(N_CH)

    def call():
        b.process_ragged_fmt(x, _lens(N_CH))
        b.flush([0, 1, 3], out_dtype="int32")
    return b, call


def _dsd_host(pkg):
    b = pkg.Batch(_plan(pkg, 44100.0, 2822400.0), N_CH)
    b.set_dsd_out(True)
    x = _x(N_CH)
    return b, lambda: b.process_host_fmt(x, out_fmt=pkg.DSD_LSB, out_scale=DSD_SCALE)


def _mixed_host(pkg):
    b = pkg.Batch.mixed([_plan(pkg), _plan(pkg, 48000.0, 24000.0)], [0, 1, 1, 0, 1])
    x = (_x(5) * 32767).astype(np.int16)
    return b, lambda: b.process_ragged_fmt(x, _lens(5), out_dtype=np.int16)


@pytest.mark.parametrize("make", [_lockstep_device, _lockstep_host, _ragged_fmt, _flush, _dsd_host, _mixed_host],
                         ids=lambda f: f.__name__.lstrip("_"))
def test_no_growth_in_steady_state(pkg, make):
    b, call = make(pkg)
    # the first call has fewer outputs (the latency), so blocks sized by a call's count grow once more on the second
    call()
    call()
    steady = b.device_bytes
    assert steady > 0
    for _ in range(3):
        call()
        assert b.device_bytes == steady


def _dsd_round_trip(pkg, b):
    before = b.device_bytes
    b.set_dsd_out(True)
    b.process_host_fmt(_x(b.n_channels), out_fmt=pkg.DSD_LSB, out_scale=DSD_SCALE)
    assert b.device_bytes > before
    b.set_dsd_out(False)
    assert b.device_bytes == before


def test_dsd_out_releases_its_memory(pkg):
    _dsd_round_trip(pkg, pkg.Batch(_plan(pkg, 44100.0, 2822400.0), N_CH))


def test_dsd_out_releases_its_memory_sharded(pkg, force_two_shards):
    b = pkg.Batch(_plan(pkg, 44100.0, 2822400.0), N_CH, pkg.DEVICE_ALL)
    assert len(b.shards()) == 2
    _dsd_round_trip(pkg, b)
