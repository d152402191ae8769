"""SURVEY 8f-1: tools/crtx_video.c, the C89 batch video driver over the crtx_* C-ABI, against the
sequential loop of extra/video_convert.c:226-277 run on the oracle: same BMP files in, same pixels (and the
same BMP container bmp_rw.c:96-146 writes) out."""
import os
import subprocess

import numpy as np
import pytest

import support as S
from ntsc_crt_b200 import layout

pytestmark = pytest.mark.gpu

DRIVER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ntsc-crt_b200", "bin", "crtx_video")


@pytest.mark.skipif(not os.path.exists(DRIVER), reason="tools/crtx_video not built")
@pytest.mark.parametrize("flags,noise,segments,w,bits", [([], 0, 5, 320, 24), ([], 12, 4, 321, 24), (["-m", "-a"], 5, 23, 320, 24),
                                                         (["-p"], 0, 3, 320, 24), ([], 3, 6, 323, 32)])
def test_batch_video_driver_writes_the_sequential_loops_images(tmp_path, flags, noise, segments, w, bits):
    n, h = 23, 240
    frames = S.moving_bars(n, w, h)
    os.mkdir(tmp_path / "frames")
    os.mkdir(tmp_path / "output")
    for k in range(n):
        S.write_bmp(str(tmp_path / "frames" / ("%06d.bmp" % (k + 1))), frames[k], bits)
    res = subprocess.run([DRIVER] + flags + ["-S", str(segments), str(n + 1), "640", "480", str(noise)],
                         cwd=str(tmp_path), stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=300)
    assert res.returncode == 0, res.stderr.decode()
    ora = S.OracleEngine("ntsc", 640, 480)
    ora.set(blend=0, scanlines=0 if "-a" in flags else 1, saturation=10)
    progressive = "-p" in flags
    for k in range(n):
        field, frame = (0, 0) if progressive else (k & 1, (k >> 1) & 1)
        ora.modulate(frames[k], format=layout.PIX_BGRA, as_color=0 if "-m" in flags else 1, field=field, frame=frame)
        ora.demodulate(noise)
        got = S.read_bmp32(str(tmp_path / "output" / ("%06d.bmp" % (k + 1))))
        assert np.array_equal(got, ora.out), "image %d: %s\n%s" % (k + 1, S.diff_report("image", got, ora.out),
                                                                   res.stdout.decode()[-300:])
    if noise == 0:
        assert b" 0 redone" in res.stdout
