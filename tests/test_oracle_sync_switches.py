"""Pin the CPU model of the decoder with its sync searches off (tests/sync_oracle.py; CRT_DO_VSYNC 0 / CRT_DO_HSYNC 0,
crt_core.h:71-72) against the reference compiled with the switches off (oracle/_ref/libref_<system>_<switches>.so, built
by oracle/Makefile): every system, each of the three switch sets, the whole state (analog, inp, out, ccf, hsync, vsync,
rn) after every call.  The fields span noise 0, 12, 60 and 255, interlaced and progressive sequences, vsync and hsync
poked to far values through the struct, the knobs with v_fac, raw sources, and VHS with do_aberration.

Where oracle/_ref holds the reference builds they are run; elsewhere their digests, recorded in
tests/golden/ref_states.json (support.from_reference), stand in for them."""
import hashlib
import json

import pytest

import support as S
from ntsc_crt_b200 import layout
from sync_oracle import SWITCHES, SYSTEMS

VARIANTS = ["%s_%s" % (s, w) for s in SYSTEMS for w in SWITCHES]


def check(variant, run):
    """run(make) with make(w, h, fmt) making the CPU model, against the same on the reference build of `variant` (VHS:
    libc rand() seeded as the oracle's)"""
    want = S.from_reference(S.ref_path(variant), lambda path: run(lambda w, h, fmt: S.RefEngine(variant, w, h, fmt, seed=1)))
    got = run(lambda w, h, fmt: S.oracle_engine(variant, w, h, fmt))
    assert len(got) == len(want), (len(got), len(want))
    bad = [i for i, (a, b) in enumerate(zip(got, want)) if a != b]
    assert not bad, "%d of %d states differ from the reference's, first after call %d" % (len(bad), len(want), bad[0])


def state_hash(e):
    return hashlib.sha256(json.dumps(S.state_digest(e.state()), sort_keys=True).encode()).hexdigest()[:16]


def source(variant, it, raw=False):
    """(image, NTSC_SETTINGS keywords) of call `it` for the system of `variant`"""
    system = layout.system_spec(variant).system
    if system == layout.SYS_NES:
        return S.nes_image(seed=3 + it % 2), dict(dot_crawl_offset=it % 3, hue=(41 * it) % 360, xoffset=4 * (it % 3),
                                                   yoffset=it % 3)
    img = S.bars_image(300, 200) if raw else S.lcg_image(96, 72, seed=7 + it % 2)
    if system == layout.SYS_NESRGB:
        return img, dict(format=layout.PIX_BGRA, dot_crawl_offset=it % 3, hue=(41 * it) % 360, xoffset=4 * (it % 3),
                         yoffset=it % 3)
    kw = dict(format=layout.PIX_BGRA, as_color=int(it % 3 != 2), raw=int(raw), hue=(41 * it) % 360,
              xoffset=4 * (it % 3), yoffset=it % 3)
    if system in (layout.SYS_SNES, layout.SYS_TEMP, layout.SYS_PV1K):
        kw["dot_crawl_offset"] = it % 4
    if system == layout.SYS_VHS:
        kw["do_aberration"] = 0
    return img, kw


@pytest.mark.parametrize("variant", VARIANTS)
def test_interlaced_with_noise_and_poked_sync(variant):
    """interlaced fields at noise 0, 12, 60, 255, with vsync / hsync poked to 130 / 700, -50 / -50 and 700 / 130 between
    them"""
    pokes = {3: dict(vsync=130, hsync=700), 5: dict(vsync=-50, hsync=-50), 7: dict(vsync=700, hsync=130)}

    def run(make):
        e = make(640, 480, layout.PIX_BGRA)
        e.set(blend=1, scanlines=1)
        out = []
        for it in range(8):
            if it in pokes:
                e.set(**pokes[it])
            img, kw = source(variant, it)
            if layout.system_spec(variant).system not in (layout.SYS_NES, layout.SYS_NESRGB):
                kw.update(field=it & 1, frame=(it >> 1) & 1)
            e.modulate(img, **kw)
            out.append(state_hash(e))
            e.demodulate([0, 12, 60, 255][it % 4])
            out.append(state_hash(e))
        return out
    check(variant, run)


@pytest.mark.parametrize("variant", VARIANTS)
def test_progressive_knobs_vfac_raw(variant):
    """progressive fields on an odd-sized 3-byte monitor with every knob off its default, v_fac 7, raw sources every
    other call, and VHS with do_aberration"""
    def run(make):
        e = make(333, 250, layout.PIX_BGR)
        e.set(hue=37, brightness=9, contrast=200, saturation=14, black_point=3, white_point=90, blend=0, scanlines=1,
              v_fac=7)
        out = []
        for it in range(6):
            img, kw = source(variant, it, raw=(it % 2 == 1))
            if "raw" in kw:
                kw.update(field=0, frame=0)
            if "do_aberration" in kw:
                kw["do_aberration"] = int(it % 2 == 0)
            e.modulate(img, **kw)
            out.append(state_hash(e))
            e.demodulate([255, 60, 12, 0][it % 4])
            out.append(state_hash(e))
        return out
    check(variant, run)
