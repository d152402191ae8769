"""The values a caller may give the picture knobs of struct CRT, the noise of crt_demodulate and the settings of
crt_modulate, as far as the reference defines what it computes from them (DESIGN.md section 2), and the cases the
knob-domain tests draw from it.

Every int is in the domain, INT_MIN and INT_MAX included, except where a bound below says otherwise: the reference's
arithmetic on these values wraps in 32 bits like the oracle's (-fwrapv) and the kernels', and where gcc -O3 makes use of
signed overflow being undefined, the oracle and the kernels restate what it made of the expression (the white scale of
the RGB encoders, crt_ntsc.c:318).  The bounds are those under which the reference reads or writes outside its arrays
or divides by zero.  One more rule is a property of the decoded signal, not of these values: a sync search or decode
window may run at most 16 bytes past inp[] (struct CRT's outw, outh, out_format and padding, k_struct_tail); the cases
below stay inside it, which their comparison with the live reference shows.
"""
import functools
import hashlib

import numpy as np

import support as S
from ntsc_crt_b200 import layout

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1

# crt_reset's values (crt_core.c:252-260), and a noise as the drivers use it
STOCK_MONITOR = dict(hue=0, brightness=0, contrast=180, saturation=10, black_point=0, white_point=100)
STOCK_NOISE = 6
# the largest noise of the CRT_DO_BLOOM build: the beam energy scale max_e = (128 + noise / 2) * AV_LEN is positive,
# ((max_e >> 1) - e) << 10 does not overflow for any line energy e, and the line width it gives keeps the decode window
# inside the line (crt_core.c:399-402, 512-526); a negative noise can make max_e 0 (a division by zero)
BLOOM_NOISE = (0, 1 << 13)
# the noise of the VHS build: past 2^24 in magnitude the compiled reference's decode of the lost-sync signal is not
# reproducible from run to run of the same calls (noise -2^30 and -2^31 give different images with other memory layouts)
VHS_NOISE = (-(1 << 24), 1 << 24)


def is_int32(v):
    return INT_MIN <= v <= INT_MAX


def wrap32(v):
    return (v + (1 << 31)) % (1 << 32) - (1 << 31)


def _cdiv(a, b):
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def _cmod(a, b):
    return a - b * _cdiv(a, b)


def _picture(spec, source):
    """(xo, yo, destw, desth) of the picture the encoder of `spec` writes, computed without wrapping, or None where
    computing them overflows an int"""
    s, xoff, yoff = spec.system, source.get("xoffset", 0), source.get("yoffset", 0)
    if s in (layout.SYS_NES, layout.SYS_NESRGB):  # crt_nes.c:131-135, crt_nesrgb.c:86-88
        xo, yo, destw, desth = spec.av_beg + xoff, spec.top + yoff, spec.av_len, spec.lines
        if not (is_int32(xo) and is_int32(yo)):
            return None
        return xo & ~3, yo, destw, desth
    bloom = spec.name.endswith("_bloom")  # picture_size, crt_ntsc.c:148-172
    maxw = (spec.av_len * 55500) >> 16 if bloom else spec.av_len
    maxh = (spec.lines * 63500) >> 16 if bloom else (spec.lines * 64500) >> 16
    destw, desth = (min(source["w"], maxw), min(source["h"], maxh)) if source.get("raw", 0) else (maxw, maxh)
    xo = spec.av_beg + xoff + _cdiv(spec.av_len - destw, 2)
    yo = spec.top + yoff + _cdiv(spec.lines - desth, 2)
    if not (is_int32(xo) and is_int32(yo)):
        return None
    if s in (layout.SYS_NTSC, layout.SYS_VHS):
        xo &= ~3  # crt_ntsc.c:199
    else:
        xo -= _cmod(xo, spec.cc_samples)  # crt_snes.c:196
    return xo, yo, destw, desth


def inside_reference_domain(variant, monitor, source, noise=STOCK_NOISE):
    """whether the reference defines what it computes for these knobs (monitor: struct CRT's, any subset), settings
    (source: NTSC_SETTINGS, with the image's w and h) and crt_demodulate noise"""
    spec = layout.system_spec(variant)
    values = list(monitor.values()) + [noise] + [v for k, v in source.items()]
    if not all(is_int32(v) for v in values):
        return False
    if variant.endswith("_bloom") and not BLOOM_NOISE[0] <= noise <= BLOOM_NOISE[1]:
        return False
    if layout.system_spec(variant).system == layout.SYS_VHS and not VHS_NOISE[0] <= noise <= VHS_NOISE[1]:
        return False
    pic = _picture(spec, source)
    if pic is None:
        return False
    xo, yo, destw, desth = pic
    H = spec.hres
    # the carrier tables are indexed by (x + xo) % CRT_CC_SAMPLES and (y + yo) % CRT_CC_VPER, the NES burst and phase
    # tables by (y + yo) % 3 and phasetab[(y + yo + dot_crawl_offset) % 3] (crt_ntsc.c:300, crt_snes.c:266,
    # crt_nes.c:166, 180, crt_nesrgb.c:96, 128): C's % keeps the sign, so these sums must not be negative (the NES's
    # xo, below)
    if yo < 0 or xo < 0:
        return False
    # the picture, and on the NES systems each line's burst, are written inside analog[] (crt_ntsc.c:321,
    # crt_nes.c:160-190, crt_nesrgb.c:96-160): a write past it lands in inp[] of the reference's struct CRT
    lo, hi = xo, xo + destw - 1
    if spec.system in (layout.SYS_NES, layout.SYS_NESRGB):
        lo, hi = min(lo, spec.cb_beg), max(hi, spec.cb_beg + burst_len(spec) - 1)
    if lo + yo * H < 0 or hi + (yo + desth - 1) * H >= spec.input_size:
        return False
    if "field" in source and spec.system != layout.SYS_SNES:
        # the source row of picture line y is y * h / desth + (field * h + desth) / desth / 2, clamped to h, not h - 1
        # (crt_ntsc.c:264-270, crt_template.c:255-262): a raw picture as tall as its image reads the row past it in
        # the odd field
        field, h = source["field"] & 1, source["h"]
        if (desth - 1) * h // desth + (field * h + desth) // desth // 2 >= h:
            return False
    # A bound of the library, not of the reference: its NES, NES-RGB and SNES encoders write each line's template and
    # picture from the CTA that owns the line (k_mod_nes, k_mod_nesrgb, k_mod_snes), so the picture must stay inside its
    # own line, xo >= 0 and xo + destw <= CRT_HRES (tests/nes_border_oracle.py draws the same range)
    if spec.system in (layout.SYS_NES, layout.SYS_NESRGB, layout.SYS_SNES) and xo + destw > H:
        return False
    if spec.system == layout.SYS_NES:
        dco = source.get("dot_crawl_offset", 0)
        if yo + dco < 0 or not is_int32(yo + desth - 1 + dco):  # phasetab[(y + yo + dot_crawl_offset) % 3], crt_nes.c:180
            return False
        if spec.border and (spec.top + dco < 0 or not is_int32(spec.bot + 2 + dco)):  # crt_nes.c:145 (NES_BORDER)
            return False
    return True


STRUCT_TAIL = 16  # bytes behind inp[] a decode may read (DESIGN.md section 2)


def decode_reach(ora, noise):
    """how far past inp[] the decode of the field the CPU model `ora` holds reads, in bytes (0: not past it), as the
    reference reads: the hsync search from the previous line's hsync up to where it breaks (crt_core.c:437-445), the
    burst (crt_core.c:456-463) and the decode window (crt_core.c:511-540).  Decodes the field on `ora`, in stages."""
    spec, o = ora.spec, ora.sys.contents
    ora.noise_pass(noise)
    h0 = ora.mon.hsync
    _, table = ora.sync_pass()
    far = 0
    for k in range(spec.lines):
        r = table[k]
        if r.skip:
            continue
        ln = ((spec.top + k + ora.mon.vsync) % spec.vres) * spec.hres
        i = (r.hsync - h0) % spec.hres  # where the search broke, or its window's end
        if i >= o.hsync_window:
            i -= spec.hres
        i = max(min(i, o.hsync_window - 1), -o.hsync_window) if spec.do_hsync else o.hsync_window - 1
        far = max(far, ln + h0 + o.sync_beg + i + 1, r.pos + spec.av_len,
                  ln + r.hsync - r.hsync % spec.cc_samples + o.cb_beg + o.burst_len)
        h0 = r.hsync
    ora.line_pass(table)
    return max(0, far - spec.input_size)


def burst_len(spec):
    """CB_CYCLES * CRT_CB_FREQ samples of colour burst: 10 cycles of the carrier (crt_ntsc.h:79-85, crt_pv1k.h)"""
    return 10 * spec.cc_samples


def offset_range(variant, which, source):
    """the smallest and largest xoffset (or yoffset) inside the domain with the other settings of `source`"""
    def ok(v):
        return inside_reference_domain(variant, {}, dict(source, **{which: v}))
    # the domain in one offset is an interval around the stock picture: bisect both ends
    lo, hi = 0, 0
    assert ok(0), (variant, source)
    for sign in (-1, 1):
        a, b = 0, sign * (1 << 20)  # ok(a), not ok(b)
        assert not ok(b)
        while abs(b - a) > 1:
            m = (a + b) // 2
            a, b = (m, b) if ok(m) else (a, m)
        if sign < 0:
            lo = a
        else:
            hi = a
    return lo, hi


# ----------------------------------------------------------------------------------
# the edge table
# ----------------------------------------------------------------------------------

# white_point: 100 * white_point wraps past 21 474 836 (the RGB encoders' WHITE_LEVEL * white_point, crt_ntsc.c:318);
# the NES's (ire * white_point / 100) with the largest ire of a pixel, 4 * 112965 + BLACK_LEVEL 0, wraps past 4752
NES_IRE_MAX = 4 * 112965
MONITOR_EDGES = dict(
    hue=[INT_MIN, INT_MIN + 1, -361, -360, -45, 359, 360, 719, INT_MAX - 1, INT_MAX],
    # bright = brightness - (BLACK_LEVEL + black_point) (crt_core.c:305) wraps near INT_MIN; sig + bright wraps near
    # INT_MAX; the equaliser's products wrap far before either (the wrap-exact equaliser)
    brightness=[INT_MIN, INT_MIN + 6, INT_MIN + 7, INT_MIN + 8, -(1 << 24), -4301, 4301, 1 << 16, 1 << 24,
                INT_MAX - 127, INT_MAX],
    # ((y + 3879 i + 2556 q) >> 12) * contrast (crt_core.c:573-575): the sum's shifted value stays under 2^11 on a
    # decoded line, so the product first wraps between 2^20 and 2^21 for the brightest pixels, and for every pixel near
    # INT_MAX; 0 and negative contrasts clamp every channel to 0
    contrast=[INT_MIN, -1, 0, 1, 255, 256, 1 << 19, 1 << 20, (1 << 20) + (1 << 19), 1 << 21, 1 << 24, INT_MAX],
    # ((dci * huecs - dcq * huesn) >> 4) * saturation (crt_core.c:472-473): powers of two drive a wave value to INT_MIN
    # exactly (the llabs of k_sync's guard), the others past it
    saturation=[INT_MIN, INT_MIN + 1, -(1 << 30), -1, 0, 1 << 16, 1 << 20, 1 << 24, 1 << 28, 1 << 30, INT_MAX],
    # the encoders clamp BLACK_LEVEL + black_point + picture to 0 .. 110 (crt_ntsc.c:319-320); the sum wraps near both ends
    black_point=[INT_MIN, INT_MIN + 1, -111, -110, -7, 110, 111, INT_MAX - 8, INT_MAX - 7, INT_MAX],
    white_point=[INT_MIN, -21474837, -21474836, -1, 0, 4752, 4753, 21474836, 21474837, 30000000, INT_MAX],
)
# (b - 127) * noise >> 8 per sample (crt_core.c:366): past 255 the noise saturates the signal, past 2^24 the product wraps
NOISE_EDGES = [INT_MIN, -(1 << 16), -40, -1, 256, 1 << 16, 1 << 23, 1 << 24, (1 << 24) + 1, INT_MAX]
# (deg + 33) * 8192 / 180 with deg = hue + k * 90 (crt_ntsc.c:180): the product wraps from deg = 262 111 on
SOURCE_HUE_EDGES = [INT_MIN, INT_MIN + 1, -262144 - 33, -360, -1, 262110 - 270, 262111 - 270, 262110, 262111,
                    INT_MAX - 270, INT_MAX]
FIELD_EDGES = [-1, 2, 3, INT_MIN, INT_MAX]


def stock_source(variant, w, h):
    """the settings every case starts from (with the image's size)"""
    s = layout.system_spec(variant).system
    if s in (layout.SYS_NES, layout.SYS_NESRGB):
        return dict(w=w, h=h, dot_crawl_offset=0, hue=0, xoffset=0, yoffset=0)
    src = dict(w=w, h=h, raw=0, as_color=1, field=0, frame=0, hue=0, xoffset=0, yoffset=0)
    if s in (layout.SYS_SNES, layout.SYS_TEMP, layout.SYS_PV1K):
        src["dot_crawl_offset"] = 0
    return src


def edge_cases(variant, w, h):
    """[(name, monitor knobs, source settings, noise)]: one value off its stock at a time, on every edge above, with the
    offsets' edges of this variant (the domain's ends, negative offsets, the picture pushed into the next line's sync)"""
    spec = layout.system_spec(variant)
    base = stock_source(variant, w, h)
    cases = []
    for knob, values in MONITOR_EDGES.items():
        for v in values:
            cases.append(("%s %d" % (knob, v), {knob: v}, {}, STOCK_NOISE))
    for v in NOISE_EDGES:
        if variant.endswith("_bloom"):
            v = min(max(v, BLOOM_NOISE[0]), BLOOM_NOISE[1])
        if spec.system == layout.SYS_VHS:
            v = min(max(v, VHS_NOISE[0]), VHS_NOISE[1])
        cases.append(("noise %d" % v, {}, {}, v))
    for v in SOURCE_HUE_EDGES:
        cases.append(("source hue %d" % v, {}, {"hue": v}, STOCK_NOISE))
    if spec.system not in (layout.SYS_NES, layout.SYS_NESRGB):
        for knob in ("field", "frame"):
            for v in FIELD_EDGES:
                cases.append(("%s %d" % (knob, v), {}, {knob: v}, STOCK_NOISE))
        for knob, v in (("as_color", -1), ("as_color", INT_MIN)):
            cases.append(("%s %d" % (knob, v), {}, {knob: v}, STOCK_NOISE))
        for v, field in ((-1, 2), (2, -2)):  # (an even field: a raw picture as tall as the image reads past it in odd ones)
            cases.append(("raw %d field %d" % (v, field), {}, {"raw": v, "field": field}, STOCK_NOISE))
    if "dot_crawl_offset" in base:
        for v in (-4, -1, 3, 4, 5, INT_MAX // 2):
            cases.append(("dot_crawl_offset %d" % v, {}, {"dot_crawl_offset": v}, STOCK_NOISE))
    for which in ("xoffset", "yoffset"):
        lo, hi = offset_range(variant, which, base)
        values = {lo, lo + 1, -1, -4, -5, hi - 1, hi}
        if which == "xoffset":  # the end of the picture past the line's end, into the next line's sync
            values |= {v for v in (spec.hres - spec.av_len - spec.av_beg + spec.sync_beg + 40,) if lo <= v <= hi}
        for v in sorted(values):
            if lo <= v <= hi:
                cases.append(("%s %d" % (which, v), {}, {which: v}, STOCK_NOISE))
    if spec.system == layout.SYS_NES:
        ylo = offset_range(variant, "yoffset", base)[0]
        dco_lo = -(spec.top + ylo)
        for yoff, dco in ((ylo, dco_lo), (ylo, dco_lo + 1), (0, -spec.top), (0, INT_MAX - spec.bot - 2)):
            cases.append(("yoffset %d dot_crawl_offset %d" % (yoff, dco), {}, {"yoffset": yoff, "dot_crawl_offset": dco},
                          STOCK_NOISE))
    cases = [(n, m, dict(base, **s), z) for n, m, s, z in cases]
    for name, mon, src, noise in cases:
        assert inside_all_fields(variant, mon, src, noise), (variant, name)
    return cases


# ----------------------------------------------------------------------------------
# the random draw
# ----------------------------------------------------------------------------------

def inside_all_fields(variant, mon, src, noise):
    """the case is inside the domain with the settings of every field it runs (modulate_settings)"""
    return all(inside_reference_domain(variant, mon, dict(src, **{k: v for k, v in modulate_settings(src, it).items()
                                                                  if k in src}), noise)
               for it in range(FIELDS))


def log_uniform(rng):
    """an int of log-uniform magnitude 0 .. 2^31 and either sign, clipped to the int range"""
    v = int(2.0 ** rng.uniform(0, 31.0)) * (1 if rng.integers(0, 2) else -1)
    if rng.integers(0, 8) == 0:
        v -= 1
    return min(max(v, INT_MIN), INT_MAX)


def draw_case(rng, variant, w, h):
    """(monitor knobs, source settings, noise) drawn over the domain: each value log-uniform with half the chance of its
    stock value; a draw outside the domain keeps the stock value"""
    base = stock_source(variant, w, h)
    mon = {k: (log_uniform(rng) if rng.integers(0, 2) else v) for k, v in STOCK_MONITOR.items()}
    src = dict(base)
    for k in base:
        if k in ("w", "h") or rng.integers(0, 2):
            continue
        v = log_uniform(rng)
        if k in ("xoffset", "yoffset", "dot_crawl_offset"):
            v = int(v) >> int(rng.integers(0, 31))  # mostly small offsets
        if inside_all_fields(variant, mon, dict(src, **{k: v}), STOCK_NOISE):
            src[k] = v
    noise = log_uniform(rng) if rng.integers(0, 2) else STOCK_NOISE
    if not inside_all_fields(variant, mon, src, noise):
        noise = STOCK_NOISE
    assert inside_all_fields(variant, mon, src, noise)
    return mon, src, noise


# ----------------------------------------------------------------------------------
# the cases the knob-domain tests run: three fields on a 256 x 200 BGRA monitor with blend and scanlines on
# ----------------------------------------------------------------------------------

OUTW, OUTH, FMT = 256, 200, layout.PIX_BGRA
SRC_W, SRC_H = 192, 160
FIELDS = 3
RANDOM_CASES = 16


def images(variant):
    if layout.system_spec(variant).system == layout.SYS_NES:
        return [S.nes_image(seed=40 + it) for it in range(FIELDS)]
    return [S.rand_image(SRC_W, SRC_H, seed=40 + it) for it in range(FIELDS)]


def modulate_settings(src, it):
    """crt_modulate's settings of field `it` of a case: its source values, with the field and frame walking their cycle
    where the case leaves them at the stock 0"""
    kw = {k: v for k, v in src.items() if k not in ("w", "h")}
    if "field" in kw:
        kw["format"] = layout.PIX_BGRA
        kw["field"] = kw["field"] or it & 1
        kw["frame"] = kw["frame"] or (it >> 1) & 1
    return kw


def case_reach(variant, mon, src, noise):
    """the furthest any field of the case reads past inp[] (decode_reach)"""
    ora = S.oracle_engine(variant, OUTW, OUTH, FMT)
    ora.set(blend=1, scanlines=1, **mon)
    far = 0
    for it, img in enumerate(images(variant)):
        ora.modulate(img, **modulate_settings(src, it))
        far = max(far, decode_reach(ora, noise))
    return far


def _seed(variant):
    return int(hashlib.sha256(variant.encode()).hexdigest()[:8], 16)


@functools.lru_cache(maxsize=None)
def cases(variant):
    """the edge table and RANDOM_CASES random draws for this variant, each inside the domain: an offset edge whose
    decode reads further than the struct tail moves toward the stock picture until it does not, another edge that does
    is left out, a random draw that does is drawn again"""
    out = []
    for name, mon, src, noise in edge_cases(variant, SRC_W, SRC_H):
        which = name.split()[0]
        if which not in ("xoffset", "yoffset", "noise"):  # (the other values leave the sync pulses as they are)
            out.append((name, mon, src, noise))
            continue
        reach = case_reach(variant, mon, src, noise)
        while which != "noise" and reach > STRUCT_TAIL:
            assert src[which] != 0, (variant, name)
            src = dict(src, **{which: src[which] - (1 if src[which] > 0 else -1)})
            name = "%s %d" % (which, src[which])
            reach = case_reach(variant, mon, src, noise)
        if reach <= STRUCT_TAIL:  # (a noise that loses sync can read further)
            out.append((name, mon, src, noise))
    rng = np.random.default_rng(_seed(variant))
    k = 0
    while k < RANDOM_CASES:
        mon, src, noise = draw_case(rng, variant, SRC_W, SRC_H)
        if case_reach(variant, mon, src, noise) <= STRUCT_TAIL:
            out.append(("random %d" % k, mon, src, noise))
            k += 1
    return out
