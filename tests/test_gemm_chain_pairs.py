"""`gemm_chain_kernel` at odd m-tile counts.  Its persistent CTAs take m-tiles round-robin.  Below one m-tile per SM the
grid is as large as the m-tile count; above it, some CTAs run one round more than others.  These encodes cover a
single m-tile, a partial last m-tile, one round per CTA, and CTAs with 1 to 3 rounds.  Each must match one launch per
layer (`LTR_CHAIN_MIN_TILES=0`) bit for bit.  Any scheme that pairs CTAs (for instance to share weight tiles) has to
get these shapes right, too."""
import pytest

from tests.test_gemm_chain import _assert_equal_paths, _batch


def _lines(tiles, P):
    """P pairs whose 2 P images hold 128 * tiles lines in all."""
    per_side = tiles * 64                       # lines on each side of the batch
    base = per_side // P
    return [base + (1 if i < per_side - base * P else 0) for i in range(P)]


@pytest.mark.gpu
@pytest.mark.parametrize("tiles, pairs", [
    (1, 1),      # one CTA
    (3, 3),      # three CTAs
    (129, 65),   # one round per CTA on a 132-SM H100
    (135, 68),   # more m-tiles than SMs: CTAs with 2 rounds and with 1
    (265, 133),  # up to three rounds
])
def test_chain_odd_tiles_equal_per_layer(tiles, pairs):
    sizes = _lines(tiles, pairs)
    batch, P = _batch(sizes, 400 + tiles, 21)
    assert (batch.n_lines + 127) // 128 == tiles
    _assert_equal_paths(batch, P, 1)


@pytest.mark.gpu
def test_chain_odd_tiles_ragged():
    """Three m-tiles, the last one partial (360 rows), ragged images."""
    batch, P = _batch([70, 60, 50], 500, 64)
    assert batch.n_lines == 360 and batch.uniform_lines is None
    _assert_equal_paths(batch, P, 1)
