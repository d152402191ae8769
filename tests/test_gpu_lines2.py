"""k_lines2 (csrc/crt_lines2.cuh): the line pass the common geometries take -- two monitors per CTA, tabulated
resampler, ring of decoded samples.  Every case runs the batch interface twice, with the kernel on (and proven to
have been taken: crtx_lines2_count) and with `lines2` off (k_lines), and compares both with the oracle after every
field: the whole state.  Geometries at and beyond the kernel's limits, every 4-byte pixel format, odd
monitor counts (a CTA with one monitor), scanline-block windows, knobs that move the luma bias, and a batch in which
one monitor of a CTA's pair needs the wrap-exact equaliser (it must be left to k_lines<generic>)."""
import numpy as np
import pytest

import support as S
from ntsc_crt_b200 import layout

pytestmark = pytest.mark.gpu

FMT4 = (layout.PIX_ARGB, layout.PIX_RGBA, layout.PIX_ABGR, layout.PIX_BGRA)


def _run(variant, outw, outh, n, fields, fmt=layout.PIX_BGRA, noise=0, expect_lines2=True, options=(), knobs=None,
         per_monitor_knobs=None, src=(256, 240), line_window=None):
    options = tuple(options) + ((("line_lo", line_window[0]), ("line_hi", line_window[1])) if line_window else ())
    mons = [dict(outw=outw, outh=outh, fmt=fmt, noise=noise + i, knobs=dict(knobs or {}, **(per_monitor_knobs or {}).get(i, {})))
            for i in range(n)]
    imgs = [S.rand_image(src[0], src[1], seed=70 + i) for i in range(n)]
    results = {}
    for lines2 in (1, 0):
        rig = S.BatchRig(variant, mons, options=(("lines2", lines2),) + options)
        for f in range(fields):
            for i in range(n):
                rig.source(i, imgs[i], format=layout.PIX_BGRA, as_color=1, field=f & 1, frame=(f >> 1) & 1)
            rig.modulate()
            rig.demodulate()
            if line_window is None:
                rig.check("lines2=%d field %d" % (lines2, f))
        took = rig.b.lines2_launches
        if lines2 == 1:
            assert (took > 0) == expect_lines2, "k_lines2 launches: %d (expected %s)" % (took, expect_lines2)
        else:
            assert took == 0
        results[lines2] = [o.cpu().numpy().copy() for o in rig.outs]
        rig.close()
    for i in range(n):  # the two kernels agree bit for bit (this is the whole check for the scanline-window case)
        assert np.array_equal(results[1][i], results[0][i]), "monitor %d: %s" % (i, S.diff_report("k_lines2 vs k_lines", results[1][i], results[0][i]))
    return results


@pytest.mark.parametrize("outw,outh,blend,scanlines", [(832, 624, 1, 1), (640, 480, 0, 1), (832, 624, 0, 0), (1280, 960, 1, 0), (1920, 1080, 1, 0)])
def test_driver_geometries(outw, outh, blend, scanlines):
    """what crt_main.c (blend 1, scanlines 1) and video_convert.c (blend 0) ask for, interlaced, 4 fields, 3 monitors;
    1920 is wider than the kernel's descriptor table has room for and stays with k_lines"""
    _run("ntsc", outw, outh, n=3, fields=4, knobs=dict(blend=blend, scanlines=scanlines), noise=0 if blend else 6, expect_lines2=outw <= 1312)


@pytest.mark.parametrize("fmt", FMT4)
def test_every_four_byte_format(fmt):
    _run("ntsc", 704, 480, n=2, fields=2, fmt=fmt, knobs=dict(blend=1, scanlines=0), noise=4)


@pytest.mark.parametrize("outw,expect", [(528, True), (524, False), (1000, True), (1312, True), (1316, False), (830, False), (256, False)])
def test_limits_of_the_geometry(outw, expect):
    """narrowest / widest output the ring and the descriptor table cover, widths that are not a multiple of 4 or 16,
    and the widths just outside, which must fall back to k_lines -- same bits either way"""
    _run("ntsc", outw, 240, n=2, fields=2, expect_lines2=expect, knobs=dict(blend=1, scanlines=0), noise=3)


def test_one_monitor_and_odd_counts():
    for n in (1, 5):
        _run("ntsc", 832, 624, n=n, fields=2, knobs=dict(blend=1, scanlines=1))


def test_brightness_contrast_black_point():
    """the luma bias that k_lines2 moves out of the filter (crt_core.c:304, 538) and the other monitor knobs"""
    _run("ntsc", 832, 480, n=3, fields=2, noise=5,
         knobs=dict(blend=1, scanlines=0, brightness=37, contrast=201, black_point=9, white_point=93, hue=25, saturation=14),
         per_monitor_knobs={1: dict(brightness=-300, black_point=-40), 2: dict(brightness=4000, contrast=60)})


def test_generic_monitor_inside_a_pair():
    """monitor 1 leaves the fast equaliser's exact range (saturation 400): k_lines2 must skip exactly its lanes and
    k_lines<generic> must take them, while monitors 0 and 2 -- its CTA neighbours -- stay on the fast path"""
    _run("ntsc", 832, 624, n=3, fields=3, noise=8, knobs=dict(blend=1, scanlines=1),
         per_monitor_knobs={1: dict(saturation=400, brightness=5000)})


def test_generic_everywhere():
    _run("ntsc", 640, 480, n=2, fields=2, options=(("generic_eq", 1),), knobs=dict(blend=0, scanlines=1))


def test_signal_windows_at_odd_byte_phases():
    """the signal windows reach shared memory by three 16-byte cp.async per lane and stage from the 16-byte aligned address
    below them; odd byte phases of the windows come from the noise-driven hsync"""
    _run("ntsc", 832, 624, n=3, fields=4, knobs=dict(blend=1, scanlines=1), noise=9)
    _run("ntsc", 640, 480, n=2, fields=2, knobs=dict(blend=0, scanlines=1), noise=0)


def test_scanline_window():
    """the scanline-block partition of one image (line_lo / line_hi): only those lines' rows are touched"""
    r = _run("ntsc", 832, 624, n=2, fields=2, knobs=dict(blend=1, scanlines=1), line_window=(60, 157))
    img = r[1][0]
    assert img[: 60 * 624 // 240].any() == 0 and img[157 * 624 // 240 + 3:].any() == 0 and img.any()


@pytest.mark.parametrize("variant", ["vhs", "template", "nes", "snes", "nesrgb"])
def test_other_systems_take_it_too(variant):
    """every build with four samples per chroma period and the IIR equaliser has the kernel"""
    n, outw, outh = 3, 832, 624
    nes = variant == "nes"
    imgs = [S.nes_image(seed=5 + i) if nes else S.rand_image(256, 240, seed=5 + i) for i in range(n)]
    res = {}
    for lines2 in (1, 0):
        rig = S.BatchRig(variant, [dict(outw=outw, outh=outh, fmt=layout.PIX_BGRA, noise=2 + i, knobs=dict(blend=1, scanlines=1))
                                   for i in range(n)], options=(("lines2", lines2),))
        for f in range(3):
            for i in range(n):
                if nes:
                    kw = dict(dot_crawl_offset=f % 3, hue=0)
                elif variant == "nesrgb":
                    kw = dict(format=layout.PIX_BGRA, dot_crawl_offset=f % 3, hue=0)
                else:
                    kw = dict(format=layout.PIX_BGRA, as_color=1, field=f & 1, frame=0, dot_crawl_offset=f % 3)
                rig.source(i, imgs[i], reinit=int(f == 0), **kw)
            rig.modulate()
            rig.demodulate()
            rig.check("%s lines2=%d field %d" % (variant, lines2, f))
        assert (rig.b.lines2_launches > 0) == (lines2 == 1)
        res[lines2] = [o.cpu().numpy().copy() for o in rig.outs]
        rig.close()
    for i in range(n):
        assert np.array_equal(res[1][i], res[0][i])


def test_pv1k_conv_and_bloom_builds_do_not_have_it():
    import torch
    from ntsc_crt_b200 import capi
    for variant in ("pv1k", "ntsc_conv", "ntsc_bloom"):
        b = capi.Batch(variant, 1)
        out = torch.zeros(480, 832, 4, dtype=torch.uint8, device="cuda")
        b.set_monitor(0, out, fmt=layout.PIX_BGRA, blend=1)
        b.commit_monitors()
        b.set_source(0, torch.from_numpy(S.rand_image(64, 48, seed=1)).cuda(), format=layout.PIX_BGRA, as_color=1)
        b.modulate()
        b.demodulate()
        torch.cuda.synchronize()
        assert b.lines2_launches == 0 and out.any()
        b.close()
