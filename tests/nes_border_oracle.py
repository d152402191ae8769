"""TEST INFRASTRUCTURE: the CPU model of the NES border colour (NES_BORDER 1, crt_nes.c:64-69, 138-161), on top of the
stock NES oracle.

The reference draws, on every crt_modulate, lines CRT_TOP .. CRT_BOT + 2 from LAV_BEG to the end of the line in
settings.border_color (pixel 0xf0 at LAV_BEG), with the picture's square-wave encoding, after the sync template and
before burst and picture.  So the border build's analog[] is the stock encoder's, except that every border byte the
field's burst and picture do not write holds the border sample.  BorderOracleEngine runs support.OracleEngine's stock
encode and then stores exactly those bytes.  It is pinned against the reference built with the switch on by
tests/test_oracle_nes_border.py.
"""
import numpy as np

import support as S
from ntsc_crt_b200 import capi, layout

BORDER_VARIANTS = list(capi.BORDER_VARIANTS)
# the largest xoffset that keeps the picture inside its line: xo = (AV_BEG + xoffset) & ~3, xo + AV_LEN <= CRT_HRES
XMAX = {"nes_border": 30, "nes_p0_border": 34}
# every 9-bit border colour, and colours with bits above bit 8 (square_sample reads bits 0-8 only)
COLOURS = list(range(512)) + [0x222, 0x10f0, 0xffffffff]

_LEVEL = (-12042, 0, 34406, 81427, -17203, -8028, 19497, 57342,  # crt_nes.c:26-35
          43581, 75693, 112965, 112965, 26951, 52181, 83721, 83721)
_EMPH = (0o300, 0o100, 0o500, 0o400, 0o600, 0o200)  # crt_nes.c:36-40


def square_sample(p, phase):
    """crt_nes.c:21-61 (p: a C int; only bits 0-8 take part)"""
    hue = p & 0x0F
    if hue >= 0x0E:
        return 0
    v = ((hue + phase) % 12) < 6
    e = ((p & 0o700) & _EMPH[(phase >> 1) % 6]) > 0
    l = 1 if hue == 0 else 0 if hue == 0x0D else int(v)
    return _LEVEL[(l << 3) + (int(e) << 2) + ((p >> 4) & 3)]


def _c_int(v):
    return ((v + (1 << 31)) % (1 << 32)) - (1 << 31)


def sample_byte(p, phase, black_point, white_point, black_level=0):
    """the signal byte of pixel p at a chroma phase (crt_nes.c:151-157): (ire * white_point / 100) >> 12, as C computes it"""
    ire = black_level + black_point + sum(square_sample(p, phase + k) for k in range(4))
    prod = _c_int(ire * white_point)
    q = abs(prod) // 100
    q = -q if prod < 0 else q  # C division truncates toward zero
    v = q >> 12  # arithmetic shift
    return ((v + 128) % 256) - 128


def lav_beg(spec):
    """LAV_BEG of crt_nes.h: PPU pixel 9 + 25 + 4 + 15 + 5 of a 341-pixel line"""
    return (9 + 25 + 4 + 15 + 5) * spec.hres // 341


def border_rows(spec, color, dot_crawl, black_point, white_point):
    """{line n: its border bytes from LAV_BEG on} for n = CRT_TOP .. CRT_BOT + 2 (crt_nes.c:138-161)"""
    lb = lav_beg(spec)
    c = _c_int(color & 0xFFFFFFFF)
    tab = {p: np.array([sample_byte(p, ph, black_point, white_point) for ph in range(12)], dtype=np.int8) for p in (c, 0xF0)}
    t = np.arange(lb, spec.hres)
    rows = {}
    for n in range(spec.top, spec.bot + 3):
        phase = (((n + dot_crawl) % 3) * 4 + 6 + 3 * (t - lb)) % 12  # phasetab, crt_nes.c:116, 145
        row = tab[c][phase]
        row[0] = tab[0xF0][phase[0]]
        rows[n] = row
    return rows


class BorderOracleEngine(S.OracleEngine):
    """support.OracleEngine for the NES_BORDER 1 variants: the stock NES encode, then the border bytes it leaves alone.
    border_color persists between calls like a field of the caller's NTSC_SETTINGS."""

    def __init__(self, variant, *a, **kw):
        super().__init__(variant, *a, **kw)
        assert self.spec.system == layout.SYS_NES and self.spec.border, variant
        self.border_color = 0

    def modulate(self, img, **kw):
        if "border_color" in kw:
            self.border_color = kw["border_color"]
        super().modulate(img, **kw)
        spec, src = self.spec, self.nes
        H = spec.hres
        analog = np.ctypeslib.as_array(self.mon.analog, shape=(spec.input_size,))  # (the oracle's own buffer, in place)
        # the bytes burst and picture wrote in this call (crt_nes.c:162-194)
        drawn = np.zeros(spec.input_size, dtype=bool)
        xo = (spec.av_beg + src.xoffset) & ~3
        yo = spec.top + src.yoffset
        burst_len = 10 * 4
        for y in range(spec.lines):
            n = y + yo
            drawn[n * H + spec.cb_beg:n * H + spec.cb_beg + burst_len] = True
            lo = max(n * H + xo, 0)
            drawn[lo:max(n * H + xo + spec.av_len, lo)] = True
        lb = lav_beg(spec)
        for n, row in border_rows(spec, self.border_color, src.dot_crawl_offset, self.mon.black_point,
                                  self.mon.white_point).items():
            keep = ~drawn[n * H + lb:(n + 1) * H]
            analog[n * H + lb:(n + 1) * H][keep] = row[keep]


def oracle_engine(variant, *a, **kw):
    """the CPU model of any NES variant: BorderOracleEngine for the border builds, support.OracleEngine otherwise"""
    return (BorderOracleEngine if layout.system_spec(variant).border else S.OracleEngine)(variant, *a, **kw)
