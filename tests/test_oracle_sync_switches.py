"""Pin the CPU model of the decoder with its sync searches off (tests/sync_oracle.py; CRT_DO_VSYNC 0 / CRT_DO_HSYNC 0,
crt_core.h:71-72) against the reference compiled with the switches off (oracle/_ref/libref_<system>_<switches>.so, built
by oracle/sync.mk): every system, each of the three switch sets, the whole state (analog, inp, out, ccf, hsync, vsync,
rn) after every call.  The fields span noise 0, 12, 60 and 255, interlaced and progressive sequences, vsync and hsync
poked to far values through the struct, the knobs with v_fac, raw sources, and VHS with do_aberration.

The reference builds' digests are recorded in tests/golden/sync_switches_ref.json.  Where oracle/_ref holds the builds
they are run and must still give the recorded digests; elsewhere the records stand in for them.  SYNC_SWITCHES_RECORD=1
rewrites the records of the tests it runs."""
import hashlib
import json
import os

import pytest

import support as S
from ntsc_crt_b200 import layout
from sync_oracle import SWITCHES, SYSTEMS, oracle_engine

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sync_switches_ref.json")
RECORD = os.environ.get("SYNC_SWITCHES_RECORD") == "1"
VARIANTS = ["%s_%s" % (s, w) for s in SYSTEMS for w in SWITCHES]


def reference_digests(key, variant, run):
    """run(make) on the reference build of `variant` where it exists, which must give the digests recorded under `key`
    (SYNC_SWITCHES_RECORD=1 records them instead); else the recorded digests"""
    path = S.ref_path(variant)
    recs = json.load(open(GOLDEN)) if os.path.exists(GOLDEN) else {}
    if not os.path.exists(path):
        assert key in recs, "%s: no recorded reference digests in %s (oracle/_ref is not built here)" % (key, GOLDEN)
        return recs[key]
    got = run(lambda w, h, fmt: S.RefEngine(variant, w, h, fmt, seed=1))  # (VHS: libc rand() seeded as the oracle's)
    if RECORD:
        recs[key] = got
        with open(GOLDEN, "w") as f:
            f.write("{\n" + ",\n".join("%s: %s" % (json.dumps(k), json.dumps(recs[k])) for k in sorted(recs)) + "\n}\n")
    else:
        assert key in recs, "%s: no recorded reference digests in %s (record them with SYNC_SWITCHES_RECORD=1)" % (key, GOLDEN)
        assert got == recs[key], "%s: the reference build no longer gives the digests recorded in %s" % (key, GOLDEN)
    return got


def check(key, variant, run):
    want = reference_digests(key, variant, run)
    got = run(lambda w, h, fmt: oracle_engine(variant, w, h, fmt))
    assert len(got) == len(want), (key, len(got), len(want))
    bad = [i for i, (a, b) in enumerate(zip(got, want)) if a != b]
    assert not bad, "%s: %d of %d states differ from the reference's, first after call %d" % (key, len(bad), len(want), bad[0])


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
    check("interlaced[%s]" % variant, variant, run)


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
    check("progressive[%s]" % variant, variant, run)
