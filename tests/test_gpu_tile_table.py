"""GPU: calls with more tiles than the fused kernel's tile table holds.

k_up2_frac2 keeps one bookkeeping entry per tile index of the call in the shared memory its plan leaves over and
computes the entries of tile indices past that per tile, as before the table.  For 44100->96000 (CDSPResampler24) the
plan keeps the filter spectrum on chip, which leaves room for 404 entries; a 2^21-sample block has about 620 tiles,
so a third of every such call takes the per-tile path.  Both must give the reference's results; a short call in
between moves every tile boundary.
"""
import pytest

from test_gpu_parity import check, run_both

pytestmark = pytest.mark.gpu


def test_long_blocks_past_the_tile_table(pkg, ref):
    big = 1 << 21
    ys, yr = run_both(pkg, ref, 44100.0, 96000.0, [big, 4097, big - 3], n_ch=2, seed=21)
    check(ys, yr)
