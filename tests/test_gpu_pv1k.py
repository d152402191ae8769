"""SURVEY 8f-3: CRT_SYSTEM_PV1K (crt_pv1k.c:120-331 and the CRT_CC_SAMPLES == 5 branches of crt_core.c:282, 459-467,
480-509, 545-549): 1920 samples per line, FIVE samples per chroma period, a 5-line chroma cycle, vertical sync at the
bottom of the field -- through libcrt_b200_pv1k.so, bit for bit against the oracle and the compiled reference."""
import pytest

import support as S
from ntsc_crt_b200 import layout
from support import check, run_all, trio

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("fmt,as_color,raw,outw,outh", [(layout.PIX_BGRA, 1, 0, 832, 624), (layout.PIX_BGR, 1, 0, 640, 480),
                                                        (layout.PIX_RGBA, 0, 0, 333, 250), (layout.PIX_ABGR, 1, 1, 100, 80)])
def test_dropin_pv1k(fmt, as_color, raw, outw, outh):
    rgb = S.rand_image(300 if not raw else 200, 260 if not raw else 180, bpp=3, seed=fmt)
    img = S.pack_rgb(rgb, fmt)
    gpu, ora, ref = trio("pv1k", outw, outh, fmt)
    run_all((gpu, ora, ref), lambda e: e.set(blend=1, scanlines=1, hue=25, saturation=11, black_point=2, white_point=95))
    for it in range(6):
        run_all((gpu, ora, ref), lambda e: e.modulate(img, format=fmt, as_color=as_color, raw=raw,
                                                      field=it & 1 if not raw else 0, frame=(it >> 1) & 1,
                                                      hue=(it * 50) % 360, dot_crawl_offset=it % 4,
                                                      xoffset=4 * (it & 1), yoffset=it % 3))
        check(gpu, ora, ref, "pv1k mod %d" % it)
        run_all((gpu, ora, ref), lambda e: e.demodulate(0 if it < 2 else 9))
        check(gpu, ora, ref, "pv1k demod %d" % it)


@pytest.mark.parametrize("w,h", [(1920, 1080), (97, 61), (1487, 240)])
def test_dropin_pv1k_source_geometries(w, h):
    """source sizes around the 1487-sample picture width; knobs that leave the fast equaliser path"""
    img = S.rand_image(w, h, seed=w)
    gpu, ora, ref = trio("pv1k", 640, 480)
    run_all((gpu, ora, ref), lambda e: e.set(blend=0, scanlines=0))
    for it in range(3):
        run_all((gpu, ora, ref), lambda e: e.modulate(img, format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=0,
                                                      hue=33 * it, dot_crawl_offset=it, yoffset=it & 1))
        run_all((gpu, ora, ref), lambda e: e.demodulate(5 * it))
        check(gpu, ora, ref, "pv1k %dx%d call %d" % (w, h, it))


def test_dropin_pv1k_generic_equaliser_and_geometries():
    """saturation / brightness far outside the packed path's exact range; fewer output rows than decoded lines;
    3-byte pixels at an odd width"""
    img = S.bars_image(400, 300)
    for (outw, outh, fmt, knobs) in [(320, 240, layout.PIX_BGRA, dict(saturation=400, brightness=5000, blend=0, scanlines=0)),
                                     (333, 100, layout.PIX_RGB, dict(blend=1, scanlines=0, brightness=3000)),
                                     (1921, 300, layout.PIX_ABGR, dict(blend=1, scanlines=1, contrast=300))]:
        gpu, ora, ref = trio("pv1k", outw, outh, fmt)
        run_all((gpu, ora, ref), lambda e: e.set(**knobs))
        for it in range(3):
            run_all((gpu, ora, ref), lambda e: e.modulate(img, format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=0,
                                                          hue=100 * it, dot_crawl_offset=it))
            run_all((gpu, ora, ref), lambda e: e.demodulate(4 * it))
            check(gpu, ora, ref, "pv1k %dx%d fmt %d call %d" % (outw, outh, fmt, it))
