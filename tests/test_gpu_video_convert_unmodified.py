"""SURVEY 8b: extra/video_convert.c is a caller that must build AND RUN unchanged against the library.  The driver
leaves its NTSC_SETTINGS uninitialised (video_convert.c:153), so both builds of the unmodified source -- linked with the
reference's crt_core.c + crt_ntsc.c, and linked with libcrt_b200_ntsc.so -- get the same stack-clearing main() in front
(oracle/zero_stack_main.c, oracle/Makefile targets video_ref_ntsc_z / video_b200_ntsc_z).  Same frames/ in, the
output/ files must be byte-identical; the reference build is also pinned to the oracle's sequential loop, which proves
the cleared stack really gave xoffset = yoffset = 0."""
import os
import shutil

import pytest

import support as S

REF_VIDEO = os.path.join(S.REF_DIR, "video_ref_ntsc_z")
B200_VIDEO = os.path.join(S.REF_DIR, "video_b200_ntsc_z")

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(not (os.path.exists(REF_VIDEO) and os.path.exists(B200_VIDEO)), reason="oracle/_ref video drivers not built")
@pytest.mark.parametrize("flags,noise,w,bits", [("-o", 0, 320, 24), ("-o", 12, 333, 24), ("-om", 3, 320, 32), ("-osp", 0, 256, 24)])
def test_unmodified_video_convert_runs_against_the_library(tmp_path, flags, noise, w, bits):
    """the same unmodified driver source linked against libcrt_b200_ntsc.so writes byte-identical files (12 images,
    interlaced / progressive, colour / monochrome, scanline gaps filled or not, noise, odd widths, 24- and 32-bit input)"""
    frames = S.moving_bars(12, w, 240, seed=5)
    ref = S.run_video_convert(REF_VIDEO, str(tmp_path / "ref"), frames, flags, 640, 480, noise, bits)
    got = S.run_video_convert(B200_VIDEO, str(tmp_path / "b200"), frames, flags, 640, 480, noise, bits)
    for k, (a, b) in enumerate(zip(got, ref)):
        assert a == b, "output/%06d.bmp differs from the reference build's" % (k + 1)
    shutil.rmtree(str(tmp_path / "ref"))
    shutil.rmtree(str(tmp_path / "b200"))
