"""The fused read step (csrc/read_step.cuh) at the edges of its 128-row tiles: each consumer warpgroup owns 64 of a tile's
rows, so a last tile of 1 to 64 rows leaves warpgroup 1 with only TMA zero fill, and one of 65 to 127 rows splits it.  Each
shape is checked against the four-launch chain the kernel replaces, recomputed in fp64 from the same operands
(tests/test_gpu_read_step_tiles.py), with the bounds of tests/test_gpu_fullshape.py::test_fused_read_step_equals_unfused_chain."""
import pytest

from tests.test_gpu_read_step_tiles import _check_fused_against_chain, _sms

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,N,last", [
    (1, 129, 1),     # a second tile of one row
    (3, 43, 1),      # the same across sample boundaries
    (64, 49, 64),    # the GQA shape: 3136 rows, 24.5 tiles; warpgroup 1 of the last tile is all zero fill
    (1, 193, 65),    # warpgroup 1 of the last tile holds one row
    (1, 255, 127),   # the last tile one row short
    (5, 51, 127),
])
def test_fused_read_step_last_tile(B, N, last):
    assert B * N % 128 == last
    _check_fused_against_chain(B, N)


@pytest.mark.parametrize("B,N", [
    (8, 128),        # one tile per sample
    (8, 256),        # two tiles per sample
    (20, 49),        # a tile spans three or four samples
    (100, 17),       # a tile spans eight or nine samples
    (384, 196),      # the batched-request shape, ~4.5 tiles per SM
])
def test_fused_read_step_samples_per_tile(B, N):
    _check_fused_against_chain(B, N)


@pytest.mark.parametrize("waves", [1, 2])
def test_fused_read_step_128_row_tiles_one_above_a_multiple_of_the_sms(waves):
    tiles = waves * _sms() + 1                       # one 128-row sample per tile
    _check_fused_against_chain(tiles, 128)
