"""Scanline-block partition of one image (SURVEY 8e) on the GPU: two crtx contexts stand in for two ranks,
each decoding its own block of lines of every field (crtx_set_option line_lo/line_hi) into its own image;
rows are handed over / merged by the rules of ntsc_crt_b200.sharding.ImageSharder (support.decode_in_blocks).  The
merged image must equal the sequential decode (oracle).  The collective plumbing itself is covered on CPU by
tests/test_sharding_gloo.py."""
import pytest

import support as S

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("variant", ["ntsc", "ntsc_conv"])
@pytest.mark.parametrize("outw,outh,scanlines,blend,world", [
    (832, 624, 1, 1, 2),
    (640, 480, 0, 1, 2),   # spill row travels after odd fields
    (400, 1080, 0, 1, 3),  # two spill rows, uneven blocks
    (320, 360, 0, 1, 16),  # 1.5 rows per line: a block's last line can be ONE row tall, its computed (blended) row then
    (320, 360, 1, 1, 16),  # lands in the next block in odd fields -- needs that block's rows first (the halo)
])
def test_two_contexts_decode_one_image(variant, outw, outh, scanlines, blend, world):
    S.decode_in_blocks(variant, outw, outh, world, scanlines=scanlines, blend=blend)


@pytest.mark.parametrize("variant,outw,outh,scanlines,blend,world", [("pv1k", 640, 480, 0, 1, 2), ("template", 832, 624, 1, 1, 2),
                                                                    ("ntsc_bloom", 640, 480, 0, 1, 2), ("ntsc_bloom", 400, 1080, 0, 1, 3)])
def test_blocks_of_the_newer_variants(variant, outw, outh, scanlines, blend, world):
    """the line window (line_lo / line_hi) through the PV-1000 line kernel and through k_lines_bloom, whose energy
    chain still runs over every line of the field on every rank"""
    S.decode_in_blocks(variant, outw, outh, world, scanlines=scanlines, blend=blend)
