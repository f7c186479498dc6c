"""Moving streams on the host (no GPU): the size and fingerprint of a channel's state blob, and the refusals.

A blob carries, per stage input j, a window of H_j samples that depends on the plan only, so its size is known without a
device: 8 * (32 header words + 8 per stage + 16 dither history words + sum of H_j)."""
import ctypes as C
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _pkg():
    import __graft_entry__
    return __graft_entry__.load_package()


A24 = 180.15
# one chain of each planner branch
CHAINS = [
    (16000.0, 16000.0, 2.0),    # passthrough
    (44100.0, 96000.0, 2.0),    # 2x BlockConvolver + whole-stepping interpolator (the fused pair)
    (96000.0, 44100.0, 2.0),    # 1x pair
    (48000.0, 47999.0, 2.0),    # order-2 interpolator
    (44100.0, 176400.0, 2.0),   # half-band upsamplers
    (192000.0, 44100.0, 2.0),   # half-band downsamplers
    (2822400.0, 44100.0, 2.0),  # half-band decimator cascade
    (96000.0, 48000.0, 2.0),    # block-exact decimation
    (48000.0, 16000.0, 0.5),    # large-tile BlockConvolver
]


@pytest.mark.parametrize("src,dst,tb", CHAINS)
@pytest.mark.parametrize("max_in", [1024, 65536])
def test_state_bytes_is_the_window_formula(src, dst, tb, max_in):
    p = _pkg().Plan(src, dst, max_in, tb, A24)
    ns = len(p.stages())
    h = p.state_windows()
    assert len(h) == ns
    assert p.state_bytes == 8 * (32 + 8 * ns + 16 + int(h.sum()))
    for st, hj in zip(p.stages(), h):
        # every window reaches at least the stage's own history (src_history + 64 slack)
        if st["name"] in ("frac_whole", "frac_poly"):
            assert hj >= st["kernel_len"] + 8 + 64
        elif st["name"] == "hbup":
            assert hj >= 2 * st["kernel_len"] + 8 + 64
        elif st["name"] == "hbdown":
            assert hj >= 4 * st["kernel_len"] + 8 + 64
        else:
            assert hj >= st["kernel_len"] // max(1, st["up"])
    if src == dst:
        assert p.state_bytes == 8 * 48


def test_trim_plan_has_a_state_size():
    p = _pkg().Plan.trim(44100.0, 48000.0, 4096, 2.0, A24, 0.01)
    assert p.state_bytes == 8 * (32 + 8 * len(p.stages()) + 16 + int(p.state_windows().sum()))


BASE = dict(src=44100.0, dst=48000.0, max_in=4096, tb=2.0, atten=A24, extfft=0, fasttiming=0)


def _plan(**kw):
    a = dict(BASE, **kw)
    return _pkg().Plan(a["src"], a["dst"], a["max_in"], a["tb"], a["atten"], 0, a["extfft"], a["fasttiming"])


def test_equal_plans_have_equal_fingerprints():
    a, b = _plan(), _plan()
    assert len(a.state_fingerprint) == 64
    assert a.state_fingerprint == b.state_fingerprint
    assert a.state_bytes == b.state_bytes


@pytest.mark.parametrize("change", [dict(src=44100.5), dict(dst=48000.5), dict(max_in=4097), dict(tb=2.5),
                                    dict(atten=A24 - 1.0), dict(extfft=1), dict(fasttiming=1)])
def test_any_construction_parameter_changes_the_fingerprint(change):
    assert _plan(**change).state_fingerprint != _plan().state_fingerprint


def test_max_trim_changes_the_fingerprint():
    pkg = _pkg()
    a = pkg.Plan.trim(44100.0, 48000.0, 4096, 2.0, A24, 0.01)
    b = pkg.Plan.trim(44100.0, 48000.0, 4096, 2.0, A24, 0.005)
    assert a.state_fingerprint != b.state_fingerprint
    assert a.state_fingerprint != _plan().state_fingerprint


def test_without_a_device_nothing_moves():
    pkg = _pkg()
    L = pkg.lib()
    buf = (C.c_ubyte * 64)()
    ch = (C.c_int * 1)(0)
    for fn in (L.r8bgpu_batch_export, L.r8bgpu_batch_import, L.r8bgpu_batch_export_device, L.r8bgpu_batch_import_device):
        assert fn(None, ch, 1, buf, 64) == -1
        assert "bad arguments" in pkg._err()
    if pkg.device_count() > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(pkg.R8bGpuError):
        pkg.Batch(_plan(), 2, 0)
