"""The picture knobs, the noise and the source settings over their whole domain (tests/knob_domain.py), in the oracle
against the compiled reference, on every variant.

Each case sets one value on an edge of its arithmetic -- where a product wraps, a sum clamps or a path changes -- or
draws all of them at random, log-uniform in magnitude, and runs three fields (modulate, demodulate) with blend and
scanlines on, so that the state carries from field to field.  With oracle/_ref built the reference runs beside the
oracle and the two are compared bit for bit on analog, inp, out, ccf, hsync, vsync and rn after every call; its
settings must hold field & 1 and frame & 1 afterwards, as crt_modulate writes them back (crt_ntsc.c:195-196).  Where
oracle/_ref is not built, one digest of all the reference's states of a case is replayed from
tests/golden/ref_states.json (`CRT_RECORD_REF=1` records them afresh).
"""
import hashlib
import json

import pytest

import knob_domain as K
import support as S
from ntsc_crt_b200 import capi


def drive(engine, variant, mon, src, noise, after):
    """the case's calls on one engine; after(what, settings) after each of them"""
    engine.set(blend=1, scanlines=1, **mon)
    for it, img in enumerate(K.images(variant)):
        kw = K.modulate_settings(src, it)
        engine.modulate(img, **kw)
        after("field %d modulate" % it, kw)
        engine.demodulate(noise)
        after("field %d demodulate" % it, kw)


def chain(digests):
    return hashlib.sha256(json.dumps(digests).encode()).hexdigest()[:16]


def settings_fields(engine):
    s = getattr(engine, "settings", None) or engine.rgb
    return s.field, s.frame


def run_case(variant, name, mon, src, noise):
    what = "%s %s (monitor %r, source %r, noise %d)" % (variant, name, mon, src, noise)
    ora = S.oracle_engine(variant, K.OUTW, K.OUTH, K.FMT)
    states = []

    def keep(call, kw):
        states.append(ora.state())
        if "field" in kw and call.endswith("modulate") and not call.endswith("demodulate"):
            assert settings_fields(ora) == (kw["field"] & 1, kw["frame"] & 1), "%s %s: oracle settings" % (what, call)

    drive(ora, variant, mon, src, noise, keep)

    def live(path):
        ref = S.RefEngine(variant, K.OUTW, K.OUTH, K.FMT, seed=1)
        got = []

        def compare(call, kw):
            st = dict(ref.state())
            S.assert_same_state(st, states[len(got)], "%s %s" % (what, call))
            got.append(S.state_digest(st))
            if "field" in kw and not call.endswith("demodulate"):
                assert settings_fields(ref) == (kw["field"] & 1, kw["frame"] & 1), (
                    "%s %s: the reference wrote back field %d, frame %d" % ((what, call) + settings_fields(ref)))

        drive(ref, variant, mon, src, noise, compare)
        return chain(got)

    want = S.from_reference(S.ref_path(variant), live)
    assert chain([S.state_digest(st) for st in states]) == want, "%s: the oracle's states are not the reference's" % what


@pytest.mark.parametrize("variant", capi.ALL_VARIANTS)
def test_knob_domain_matches_the_reference(variant):
    for name, mon, src, noise in K.cases(variant):
        run_case(variant, name, mon, src, noise)


def test_cases_are_inside_the_domain():
    """every case the knob-domain tests run is inside the predicate and its decode reads at most the struct tail past
    inp[], and the predicate rejects the values just past each offset bound"""
    for variant in capi.ALL_VARIANTS:
        for name, mon, src, noise in K.cases(variant):
            assert K.inside_all_fields(variant, mon, src, noise), (variant, name)
            assert K.case_reach(variant, mon, src, noise) <= K.STRUCT_TAIL, (variant, name)
        base = K.stock_source(variant, K.SRC_W, K.SRC_H)
        for which in ("xoffset", "yoffset"):
            lo, hi = K.offset_range(variant, which, base)
            assert lo < 0 < hi, (variant, which, lo, hi)
            assert not K.inside_reference_domain(variant, {}, dict(base, **{which: lo - 1}))
            assert not K.inside_reference_domain(variant, {}, dict(base, **{which: hi + 1}))


def test_edge_table_reaches_the_wraps():
    """the edges the table claims: 100 * white_point wraps between its two values, the NES's largest ire times
    white_point between its two, and the source hue's (deg + 33) * 8192 between 262 110 and 262 111"""
    wp = K.MONITOR_EDGES["white_point"]
    assert 100 * 21474836 <= K.INT_MAX < 100 * 21474837 and {21474836, 21474837} <= set(wp)
    assert K.NES_IRE_MAX * 4752 <= K.INT_MAX < K.NES_IRE_MAX * 4753 and {4752, 4753} <= set(wp)
    assert (262110 + 33) * 8192 <= K.INT_MAX < (262111 + 33) * 8192
    assert {262110, 262111, 262110 - 270, 262111 - 270} <= set(K.SOURCE_HUE_EDGES)
    for values in list(K.MONITOR_EDGES.values()) + [K.NOISE_EDGES, K.SOURCE_HUE_EDGES]:
        assert K.INT_MIN in values or K.INT_MAX in values
