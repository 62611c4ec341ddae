"""The packed kernel's FULL form against the oracle.

fill_uniforms sets X2Hot::full when the packed launch's grid is exactly the written part of the output (integer prologue, origin 0,
whole 32 x 8 blocks, no partly written last row) and both source-rect maps add +0.  Without a digital lens the kernel then drops the
bounds exit, the per-lane write tests and the final `+ 0` of the source-rect maps (warp_x2_body<..., FULL>).  These frames sit on
both sides of that choice: full frames (8-bit and 16-bit, with pixels that leave the source and take the cold path), and frames of
the same size that miss one condition (a source rect at a non-zero origin, one row short of whole blocks, one column short).
"""
import pytest

from tests.test_parity_gpu import assert_bit_exact

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", [
    dict(w=640, h=360),                                                    # full: 20 x 45 blocks of 32 x 8 pixels
    dict(w=640, h=360, pix="Luma8", ts=777.7),
    dict(w=640, h=360, pix="Luma16"),
    dict(w=512, h=256, fov=1.8),                                           # zoomed out: pixels outside the source, background fill
    dict(w=640, h=360, in_rect=(16, 8, 640, 360), in_size=(672, 376)),     # source rect at a non-zero origin: `+ add` stays
    dict(w=640, h=359),                                                    # the last block row half filled
    dict(w=639, h=360),                                                    # the last block column one pixel short
], ids=["full-rgba8", "full-luma8", "full-luma16", "full-zoomed-out", "src-origin", "rows-short", "cols-short"])
def test_full_grid_forms_match_oracle(case):
    assert_bit_exact(case)
