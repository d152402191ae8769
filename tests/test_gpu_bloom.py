"""SURVEY 8f-4: the reference's CRT_DO_BLOOM 1 build (crt_core.h:70; crt_core.c:399-402, 512-531; crt_ntsc.c:148-161)
-- every line's width follows a filtered beam energy carried from line to line -- through
libcrt_b200_ntsc_bloom.so, bit for bit against the oracle and a reference compiled with the option on."""
import numpy as np
import pytest

import support as S
from ntsc_crt_b200 import layout
from support import check, run_all, trio

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("outw,outh,raw", [(832, 624, 0), (640, 480, 0), (333, 250, 1)])
def test_dropin_bloom(outw, outh, raw):
    img = S.bars_image(300, 260) if not raw else S.rand_image(200, 180, seed=5)
    gpu, ora, ref = trio("ntsc_bloom", outw, outh)
    run_all((gpu, ora, ref), lambda e: e.set(blend=1, scanlines=1, brightness=4, contrast=190))
    for it in range(5):
        run_all((gpu, ora, ref), lambda e: e.modulate(img, format=layout.PIX_BGRA, as_color=1, raw=raw,
                                                      field=it & 1 if not raw else 0, frame=(it >> 1) & 1))
        check(gpu, ora, ref, "bloom mod %d" % it)
        run_all((gpu, ora, ref), lambda e: e.demodulate(0 if it < 2 else 20))
        check(gpu, ora, ref, "bloom demod %d" % it)


@pytest.mark.parametrize("fmt,outw,outh,blend,scanlines", [(layout.PIX_RGB, 401, 300, 1, 0), (layout.PIX_ARGB, 256, 100, 1, 0),
                                                          (layout.PIX_ABGR, 1921, 241, 0, 1), (layout.PIX_BGR, 97, 31, 0, 0),
                                                          (layout.PIX_RGBA, 640, 720, 1, 1)])
def test_dropin_bloom_formats_and_geometries(fmt, outw, outh, blend, scanlines):
    """3-byte pixels, fewer output rows than decoded lines (lines share rows: ordered passes), more than two rows
    per line, knobs outside the packed equaliser's range, a bright picture (wide lines) after a dark one (narrow)"""
    dark = np.zeros((240, 320, 4), dtype=np.uint8)
    bright = np.full((240, 320, 4), 255, dtype=np.uint8)
    gpu, ora, ref = trio("ntsc_bloom", outw, outh, fmt)
    run_all((gpu, ora, ref), lambda e: e.set(blend=blend, scanlines=scanlines, saturation=25, brightness=-30, contrast=260, hue=77))
    for it, img in enumerate([dark, bright, S.rand_image(500, 300, seed=fmt), bright, dark]):
        run_all((gpu, ora, ref), lambda e: e.modulate(img, format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=0,
                                                      xoffset=4 * (it & 1), yoffset=it % 2))
        run_all((gpu, ora, ref), lambda e: e.demodulate(7 * it))
        check(gpu, ora, ref, "bloom fmt %d %dx%d call %d" % (fmt, outw, outh, it))
    run_all((gpu, ora, ref), lambda e: e.set(saturation=900, brightness=5000))
    run_all((gpu, ora, ref), lambda e: e.demodulate(3))
    check(gpu, ora, ref, "bloom extreme knobs")
