"""v_fac, the vertical stretch of struct CRT (crt_core.h:86), in the oracle against the compiled reference.

Every decoded line k writes the output rows
    beg = k * (outh + v_fac) / CRT_LINES + field  ..  end = (k + 1) * (outh + v_fac) / CRT_LINES + field
(crt_core.c:428-432), and v_fac is unsigned: the sum and the products are 32-bit unsigned arithmetic.  So a "negative"
v_fac shrinks the span outh + v_fac (lines then share rows, applied in line order), a span can wrap to any value, and
above (2^32 - 1) / CRT_LINES the products wrap too: beg and end no longer grow with the line, and lines far apart
write the same rows.  All of it is inside the parity domain.  The cases below walk those edges for H = outh below
and above the line count, with blend and scanlines on and off in both fields, with and without noise.

Where oracle/_ref is not built the reference's side is replayed from tests/golden/ref_states.json
(support.RefEngine); `CRT_RECORD_REF=1 python -m pytest tests/test_oracle_vfac.py` records it afresh.
"""
import pytest

import support as S
from ntsc_crt_b200 import layout

M32 = 1 << 32


def vfac_cases(lines, outh):
    """(name, v_fac) pairs: the knob's edges for CRT_LINES = lines and this output height"""
    cases = [("0", 0), ("1", 1), ("3H", 3 * outh)]
    if outh < lines:  # the last span at which lines share rows, the first at which each owns one, and one more
        cases += [("L-H-1", lines - outh - 1), ("L-H", lines - outh), ("L-H+1", lines - outh + 1)]
    # spans reached by wrapping the sum: v_fac = 2^32 - H + span
    edge = (M32 - 1) // lines  # the largest span at which no product wraps
    for name, span in (("span 0", 0), ("span 1", 1), ("span L-1", lines - 1), ("span L", lines), ("span L+1", lines + 1),
                       ("span (2^32-1)/L", edge), ("span (2^32-1)/L+1", edge + 1), ("span 2^31+H", (1 << 31) + outh)):
        cases.append((name, (span - outh) % M32))
    return cases


# one call per row: the knobs the reference reads from struct CRT, the field the picture is encoded in, the noise
CALLS = [dict(blend=0, scanlines=0, field=0, noise=0),
         dict(blend=1, scanlines=1, field=1, noise=0),
         dict(blend=1, scanlines=0, field=0, noise=9),
         dict(blend=0, scanlines=1, field=1, noise=17),
         dict(blend=1, scanlines=1, field=0, noise=0)]


def source(variant, it):
    if variant.startswith("nes"):
        return S.nes_image(seed=30 + it), dict(dot_crawl_offset=it % 3, hue=20 * it)
    img = S.rand_image(256, 220, seed=30 + it)
    return img, dict(format=layout.PIX_BGRA, as_color=1, frame=(it >> 1) & 1)


def modulate_kw(variant, call, kw):
    kw = dict(kw)
    if not variant.startswith("nes"):
        kw["field"] = call["field"]
    return kw


@pytest.mark.parametrize("outw,outh,fmt", [(320, 200, layout.PIX_BGRA), (300, 480, layout.PIX_RGB)])
@pytest.mark.parametrize("variant", ["ntsc", "nes", "pv1k", "ntsc_bloom"])
def test_vfac_edges_match_the_reference(variant, outw, outh, fmt):
    lines = layout.system_spec(variant).lines
    for name, v_fac in vfac_cases(lines, outh):
        ref = S.RefEngine(variant, outw, outh, fmt, seed=1)
        ora = S.OracleEngine(variant, outw, outh, fmt, seed=1)
        for e in (ref, ora):
            e.set(v_fac=v_fac)
        for it, call in enumerate(CALLS):
            img, kw = source(variant, it)
            for e in (ref, ora):
                e.set(blend=call["blend"], scanlines=call["scanlines"])
                e.modulate(img, **modulate_kw(variant, call, kw))
            S.assert_same_state(ref.state(), ora.state(), "%s %dx%d v_fac %s (%d) mod %d" % (variant, outw, outh, name, v_fac, it))
            for e in (ref, ora):
                e.demodulate(call["noise"])
            S.assert_same_state(ref.state(), ora.state(), "%s %dx%d v_fac %s (%d) demod %d" % (variant, outw, outh, name, v_fac, it))


def test_vfac_cases_reach_every_row_mapping_class():
    """the case list covers what it claims: shared rows, disjoint rows, every line on one row, and wrapping products"""
    for outh in (200, 480):
        spans = {name: (outh + v) % M32 for name, v in vfac_cases(240, outh)}
        assert spans["span 0"] == 0 and spans["span L-1"] == 239 and spans["span L"] == 240
        assert spans["span (2^32-1)/L"] * 240 < M32 <= spans["span (2^32-1)/L+1"] * 240
        assert spans["span 2^31+H"] == (1 << 31) + outh
        if outh < 240:
            assert (spans["L-H-1"], spans["L-H"], spans["L-H+1"]) == (239, 240, 241)
