"""Extreme geometries through the drop-in interface, every RGB variant: 1 x 1 in and out, one output row or column,
8192-pixel rows, eight output rows per decoded line, a source of one row or one column, raw sources smaller than the
picture.  Kernel library vs oracle vs the compiled reference after two fields with blend."""
import pytest

import support as S
from ntsc_crt_b200 import layout
from support import check, run_all, trio

pytestmark = pytest.mark.gpu

GEOMETRIES = [(1, 1, 5, 1, 1, 0), (1, 240, 0, 1, 1, 1), (8192, 1, 5, 3, 2, 0), (5, 2000, 1, 2, 1, 1), (2, 3, 3, 1000, 1, 0),
              (7, 239, 4, 1, 700, 1)]


@pytest.mark.parametrize("variant", ["ntsc", "ntsc_conv", "snes", "template", "pv1k", "ntsc_bloom"])
def test_extreme_geometries(variant):
    for (outw, outh, fmt, w, h, raw) in GEOMETRIES:
        img = S.rand_image(w, h, seed=w + h)
        gpu, ora, ref = trio(variant, outw, outh, fmt)
        run_all((gpu, ora, ref), lambda e: e.set(blend=1, scanlines=1))
        for f in (0, 1):
            kw = dict(format=layout.PIX_BGRA, as_color=1, field=f if h > 1 else 0, frame=0, raw=raw)
            if variant in ("pv1k", "template", "snes"):
                kw["dot_crawl_offset"] = f
            run_all((gpu, ora, ref), lambda e: e.modulate(img, **kw))
            run_all((gpu, ora, ref), lambda e: e.demodulate(3))
        check(gpu, ora, ref, "%s out %dx%d fmt %d src %dx%d raw %d" % (variant, outw, outh, fmt, w, h, raw))
