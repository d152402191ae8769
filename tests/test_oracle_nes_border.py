"""Pin the CPU model of the NES border colour (tests/nes_border_oracle.py; crt_nes.c:64-69, 138-161) against the
reference compiled with NES_BORDER 1 (oracle/_ref/libref_nes_border.so, libref_nes_p0_border.so, built by
oracle/Makefile): every border colour, the dot crawl, black and white points, every picture offset that keeps the
picture inside its line, and re-initialisations followed by plain calls with the colour changed between them.

Where oracle/_ref holds the reference builds they are run; elsewhere their digests, recorded in
tests/golden/ref_states.json (support.from_reference), stand in for them."""
import hashlib
import json

import pytest

import support as S
from nes_border_oracle import COLOURS, XMAX
from ntsc_crt_b200 import capi


def check(variant, run):
    """run(make) with make(w, h) making the CPU model, against the same on the reference build of `variant`"""
    want = S.from_reference(S.ref_path(variant), lambda path: run(lambda w, h: S.CEngine(path, variant, w, h)))
    got = run(lambda w, h: S.oracle_engine(variant, w, h))
    assert len(got) == len(want), (len(got), len(want))
    bad = [i for i, (a, b) in enumerate(zip(got, want)) if a != b]
    assert not bad, "%d of %d digests differ from the reference's, first at call %d: %r != %r" % (
        len(bad), len(want), bad[0], got[bad[0]], want[bad[0]])


def encodes(calls, knobs):
    """run: the analog[] digest after each modulate of `calls` (NTSC_SETTINGS keyword dicts), on a 64x48 monitor"""
    def run(make):
        e = make(64, 48)
        e.set(**knobs)
        out = []
        for kw in calls:
            kw = dict(kw)
            e.modulate(kw.pop("img"), **kw)
            out.append(S.digest(e.analog))
        return [hashlib.sha256("".join(out).encode()).hexdigest()[:16]] + out[-1:]
    return run


@pytest.mark.parametrize("variant", capi.BORDER_VARIANTS)
def test_every_border_colour(variant):
    """every 9-bit colour and three with higher bits, the dot crawl cycling, non-default black and white points"""
    img = S.nes_image(seed=12)
    calls = [dict(img=img, border_color=c, dot_crawl_offset=k % 3, hue=(7 * k) % 360, xoffset=k % (XMAX[variant] + 1),
                  yoffset=k % 8, field_initialized=int(k != 0)) for k, c in enumerate(COLOURS)]
    check(variant, encodes(calls, dict(black_point=5, white_point=85)))


@pytest.mark.parametrize("variant", capi.BORDER_VARIANTS)
@pytest.mark.parametrize("knobs", [dict(), dict(black_point=-6, white_point=120)], ids=["default", "points"])
def test_every_picture_offset(variant, knobs):
    """xoffset 0 .. the largest that keeps the picture inside its line, with every yoffset 0 .. 7"""
    img = S.nes_image(rainbow=True)
    calls = [dict(img=img, border_color=(0x22 + 13 * x + 57 * y) & 0x1ff, dot_crawl_offset=(x + y) % 3, xoffset=x, yoffset=y,
                  field_initialized=int(x + y != 0)) for x in range(XMAX[variant] + 1) for y in range(8)]
    check(variant, encodes(calls, knobs))


@pytest.mark.parametrize("variant", capi.BORDER_VARIANTS)
@pytest.mark.parametrize("knobs", [dict(blend=1, scanlines=1, black_point=3, white_point=93),
                                   dict(blend=0, scanlines=1, black_point=-2, white_point=108, hue=40)], ids=["a", "b"])
def test_fields_after_reinit(variant, knobs):
    """a re-initialising call, then plain ones with the border colour, dot crawl and offsets changed between them, and a
    second re-initialisation; the whole state (analog, inp, out, ccf, hsync, vsync, rn) after every call"""
    img = S.nes_image(seed=31)

    def run(make):
        e = make(832, 624)
        e.set(**knobs)
        out = []
        for it in range(7):
            kw = dict(border_color=[0x22, 0x1ff, 0x0d, 0x130, 0x2a5, 0x0f, 0x3c][it], dot_crawl_offset=it % 3,
                      hue=(25 * it) % 360, xoffset=[0, XMAX[variant], 13, 4, 22, 9, 30][it], yoffset=[0, 7, 3, 5, 1, 6, 2][it])
            if it in (0, 4):
                kw["field_initialized"] = 0
            e.modulate(img, **kw)
            out.append(S.state_digest(e.state()))
            e.demodulate(5 * it)
            out.append(S.state_digest(e.state()))
        return [json.dumps(d, sort_keys=True) for d in out]
    check(variant, run)
