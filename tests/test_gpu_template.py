"""SURVEY 8f-3: CRT_SYSTEM_TEMP (crt_template.c:125-336) -- the reference's worked example for new systems: NTSC
line timing, a 2-line chroma cycle walked by dot_crawl_offset, band-limited RGB encoder, field-dependent vertical
sync -- through libcrt_b200_template.so, bit for bit against the oracle and the compiled reference."""
import pytest

import support as S
from ntsc_crt_b200 import layout
from support import check, run_all, trio

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("fmt,as_color,raw,outw,outh", [(layout.PIX_BGRA, 1, 0, 832, 624), (layout.PIX_BGR, 1, 0, 640, 480),
                                                        (layout.PIX_RGBA, 0, 0, 333, 250), (layout.PIX_ABGR, 1, 1, 100, 80)])
def test_dropin_template(fmt, as_color, raw, outw, outh):
    rgb = S.rand_image(300 if not raw else 200, 260 if not raw else 180, bpp=3, seed=fmt)
    img = S.pack_rgb(rgb, fmt)
    gpu, ora, ref = trio("template", outw, outh, fmt)
    run_all((gpu, ora, ref), lambda e: e.set(blend=1, scanlines=1, hue=-15, saturation=12, black_point=2, white_point=95))
    for it in range(6):
        run_all((gpu, ora, ref), lambda e: e.modulate(img, format=fmt, as_color=as_color, raw=raw,
                                                      field=it & 1 if not raw else 0, frame=(it >> 1) & 1,
                                                      hue=(it * 50) % 360, dot_crawl_offset=it % 4,
                                                      xoffset=4 * (it & 1), yoffset=it % 3))
        check(gpu, ora, ref, "template mod %d" % it)
        run_all((gpu, ora, ref), lambda e: e.demodulate(0 if it < 2 else 9))
        check(gpu, ora, ref, "template demod %d" % it)


@pytest.mark.parametrize("w,h", [(1920, 1080), (97, 61), (753, 240)])
def test_dropin_template_source_geometries(w, h):
    """wide sources leave the staged encoder kernel for the gather variant; both carry the per-row carrier tables"""
    img = S.rand_image(w, h, seed=w)
    gpu, ora, ref = trio("template", 640, 480)
    run_all((gpu, ora, ref), lambda e: e.set(blend=0, scanlines=0))
    for it in range(3):
        run_all((gpu, ora, ref), lambda e: e.modulate(img, format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=0,
                                                      hue=33 * it, dot_crawl_offset=it, yoffset=it & 1))
        run_all((gpu, ora, ref), lambda e: e.demodulate(5 * it))
        check(gpu, ora, ref, "template %dx%d call %d" % (w, h, it))


def test_dropin_nes_chroma_pattern_1():
    """CRT_CHROMA_PATTERN 1 of the NES (crt_nes.h:33-34: 227.5 cycles per line, CRT_HRES 910), libcrt_b200_nes_p1.so --
    the third of the three patterns; same kernels, another line length."""
    for img in (S.nes_image(seed=5), S.nes_image(rainbow=True)):
        gpu, ora, ref = trio("nes_p1", 832, 624)
        run_all((gpu, ora, ref), lambda e: e.set(blend=0, scanlines=1))
        for it in range(5):
            run_all((gpu, ora, ref), lambda e: e.modulate(img, dot_crawl_offset=it % 3, hue=(it * 30) % 360))
            check(gpu, ora, ref, "nes_p1 mod %d" % it)
            run_all((gpu, ora, ref), lambda e: e.demodulate(it * 4))
            check(gpu, ora, ref, "nes_p1 demod %d" % it)


@pytest.mark.parametrize("variant", ["nesrgb_p0", "nesrgb_p1"])
def test_dropin_nesrgb_chroma_patterns(variant):
    """the NES-RGB system with the other two chroma patterns of crt_nesrgb.h:27-40 (912 / 910 samples per line)"""
    img = S.rand_image(256, 240, seed=8)
    gpu, ora, ref = trio(variant, 832, 624)
    run_all((gpu, ora, ref), lambda e: e.set(blend=1, scanlines=1, saturation=12))
    for it in range(4):
        run_all((gpu, ora, ref), lambda e: e.modulate(img, format=layout.PIX_BGRA, hue=(it * 70) % 360, dot_crawl_offset=it % 3,
                                                      xoffset=4 * (it & 1), yoffset=it % 2))
        check(gpu, ora, ref, "%s mod %d" % (variant, it))
        run_all((gpu, ora, ref), lambda e: e.demodulate(0 if it < 2 else 7))
        check(gpu, ora, ref, "%s demod %d" % (variant, it))
