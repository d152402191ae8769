"""ctypes mirror of the reference's C interface for the hot path.

The reference's plugin surface is compile-time polymorphic: `struct CRT`
(crt_core.h:74-92) embeds `analog[CRT_INPUT_SIZE]`, `inp[CRT_INPUT_SIZE]` and
`ccf[CRT_CC_VPER][4]`, and `struct NTSC_SETTINGS` differs per system
(crt_ntsc.h:111-124, crt_ntscvhs.h:133-147, crt_nes.h:132-143).  One shared library is
built per variant; this module lays the matching ctypes views over them.  The same
views are used for the product libraries (ntsc-crt_b200/lib) and, in the tests, for the
compiled reference (oracle/_ref), which is how layout identity is checked.
"""
import ctypes as C
from dataclasses import dataclass, replace

PIX_RGB, PIX_BGR, PIX_ARGB, PIX_RGBA, PIX_ABGR, PIX_BGRA = range(6)  # crt_core.h:62-67

SYS_NTSC, SYS_NES, SYS_PV1K, SYS_SNES, SYS_TEMP, SYS_VHS, SYS_NESRGB = 0, 1, 2, 3, 4, 5, 6  # crt_core.h:30-36


def bpp4fmt(fmt):
    """crt_bpp4fmt (crt_core.c:63-78)."""
    if fmt in (PIX_RGB, PIX_BGR):
        return 3
    if fmt in (PIX_ARGB, PIX_RGBA, PIX_ABGR, PIX_BGRA):
        return 4
    return 0


@dataclass(frozen=True)
class SystemSpec:
    name: str          # library suffix: ntsc | ntsc_conv[6|5|4] | vhs | nes | nes_p0 | nes_border | snes | ntsc_nosync | ...
    system: int        # CRT_SYSTEM
    pattern: int       # CRT_CHROMA_PATTERN
    hres: int
    vres: int
    top: int
    bot: int
    vper: int          # CRT_CC_VPER
    sync_beg: int
    bw_beg: int
    cb_beg: int
    av_beg: int
    av_len: int
    hsync_window: int
    vsync_window: int
    white: int
    burst: int
    black: int
    sync: int
    border: bool = False  # NES_BORDER 1 (crt_nes.c:64-69): the NES encoder draws settings.border_color
    do_vsync: bool = True  # CRT_DO_VSYNC (crt_core.h:71); off: field from analog[] before the noise, vsync -3
    do_hsync: bool = True  # CRT_DO_HSYNC (crt_core.h:72); off: hsync 0 after every decoded line

    @property
    def input_size(self):
        return self.hres * self.vres

    @property
    def lines(self):
        return self.bot - self.top

    @property
    def cc_samples(self):
        """CRT_CC_SAMPLES: 4 everywhere but the PV-1000 (crt_pv1k.h)."""
        return 5 if self.system == SYS_PV1K else 4


def _rgb_spec(name, system):
    # crt_ntsc.h:25-109 (CRT_CHROMA_PATTERN 1 -> 227.5 cycles/line)
    hres = 2275 * 4 // 10
    line_ns = 1500 + 4700 + 600 + 2500 + 1600 + 52600
    p = lambda ns: ns * hres // line_ns
    return SystemSpec(name, system, 1, hres, 262, 21, 261, 1,
                      p(1500), p(6200), p(6800), p(10900), p(52600),
                      8, 8, 100, 20, 7, -40)


def _nes_spec(name, pattern, border=False):
    # crt_nes.h:30-130
    hres = {0: 2280, 1: 2275, 2: 2273}[pattern] * 4 // 10
    p = lambda px: px * hres // 341
    return SystemSpec(name, SYS_NES, pattern, hres, 262, 15, 255, 3,
                      p(9), p(34), p(38), p(74), p(256),
                      6, 6, 110, 30, 0, -37, border)


def _snes_spec(name):
    # crt_snes.h:20-109: the NES line layout (227.3 cycles per line), composite NTSC levels
    n = _nes_spec(name, 2)
    return SystemSpec(name, SYS_SNES, 2, n.hres, n.vres, n.top, n.bot, n.vper, n.sync_beg, n.bw_beg, n.cb_beg,
                      n.av_beg, n.av_len, n.hsync_window, n.vsync_window, 100, 20, 7, -40)


def _nesrgb_spec(name, pattern=2):
    # crt_nesrgb.h: NES layout (any of its three chroma patterns), sync and burst levels; white at 100
    n = _nes_spec(name, pattern)
    return SystemSpec(name, SYS_NESRGB, pattern, n.hres, n.vres, n.top, n.bot, n.vper, n.sync_beg, n.bw_beg, n.cb_beg,
                      n.av_beg, n.av_len, n.hsync_window, n.vsync_window, 100, 30, 0, -37)


SPECS = {
    "ntsc": _rgb_spec("ntsc", SYS_NTSC),
    # the USE_CONVOLUTION 1 build of crt_core.c (line 85): same layouts and timing, FIR decoder filters
    "ntsc_conv": _rgb_spec("ntsc_conv", SYS_NTSC),
    # ... and its 6-, 5- and 4-tap kernels (crt_core.c:86-88)
    "ntsc_conv6": _rgb_spec("ntsc_conv6", SYS_NTSC),
    "ntsc_conv5": _rgb_spec("ntsc_conv5", SYS_NTSC),
    "ntsc_conv4": _rgb_spec("ntsc_conv4", SYS_NTSC),
    "vhs": _rgb_spec("vhs", SYS_VHS),
    "nes": _nes_spec("nes", 2),
    "nes_p0": _nes_spec("nes_p0", 0),
    "nes_p1": _nes_spec("nes_p1", 1),  # crt_nes.h:33-34: 227.5 cycles per line (the NTSC line length, HRES 910)
    # NES_BORDER 1 (crt_nes.c:64-69): the stock NES timing, and pattern 0 (HRES 912)
    "nes_border": _nes_spec("nes_border", 2, border=True),
    "nes_p0_border": _nes_spec("nes_p0_border", 0, border=True),
    "snes": _snes_spec("snes"),
    "nesrgb": _nesrgb_spec("nesrgb"),
    "nesrgb_p0": _nesrgb_spec("nesrgb_p0", 0),
    "nesrgb_p1": _nesrgb_spec("nesrgb_p1", 1),
    # the NTSC system built with CRT_DO_BLOOM 1 (crt_core.h:70; reference-side only so far)
    "ntsc_bloom": _rgb_spec("ntsc_bloom", SYS_NTSC),
    # crt_pv1k.h (reference-side only so far): 1920 samples per line, 5 samples per chroma period, 5-line cycle
    "pv1k": (lambda h, u: SystemSpec("pv1k", SYS_PV1K, 0, h, 262, 21, 261, 5, 3 * u * h // (71 * u), 6 * u * h // (71 * u),
                                     8 * u * h // (71 * u), 16 * u * h // (71 * u), 55 * u * h // (71 * u), 8, 8,
                                     100, 20, 7, -40))(2304 * 5 // 6, 892),
    # crt_template.h (reference-side only so far: used to pin the oracle ahead of a product library)
    "template": SystemSpec("template", SYS_TEMP, 1, *(lambda n: (n.hres, n.vres, n.top, n.bot, 2, n.sync_beg, n.bw_beg,
                                                                  n.cb_beg, n.av_beg, n.av_len, n.hsync_window,
                                                                  n.vsync_window, n.white, n.burst, n.black, n.sync))(
        _rgb_spec("template", SYS_NTSC))),
}


# The sync switches of crt_core.h:71-72 go with every system: `<stock variant><suffix>` names its build with them off
# (capi.SYNC_VARIANTS are built as libraries, the other combinations through `make custom`).  Not combined with the
# convolution decoder or bloom.
SYNC_SUFFIXES = {"_novsync": (False, True), "_nohsync": (True, False), "_nosync": (False, False)}
_sync_specs = {}


def system_spec(name):
    if name in SPECS:
        return SPECS[name]
    if name not in _sync_specs:
        for suffix, (do_vsync, do_hsync) in SYNC_SUFFIXES.items():
            base = name[:-len(suffix)]
            if name.endswith(suffix) and base in SPECS and not uses_convolution(base) and not base.endswith("_bloom"):
                _sync_specs[name] = replace(SPECS[base], name=name, do_vsync=do_vsync, do_hsync=do_hsync)
                break
        else:
            raise KeyError(name)
    return _sync_specs[name]


def conv_taps(name):
    """Taps of the FIR kernel for variants built from the reference's USE_CONVOLUTION 1 decoder
    (crt_core.c:85-147), 0 for the stock three-band equaliser."""
    if "_conv" not in name:
        return 0
    tail = name.split("_conv")[1]
    return int(tail) if tail else 7


def uses_convolution(name):
    return conv_taps(name) != 0


_crt_cache = {}


def crt_struct(spec):
    """ctypes view of `struct CRT` for one variant (crt_core.h:74-92)."""
    key = (spec.input_size, spec.vper, spec.cc_samples)
    if key not in _crt_cache:
        class CRT(C.Structure):
            _fields_ = [
                ("analog", C.c_byte * spec.input_size),
                ("inp", C.c_byte * spec.input_size),
                ("outw", C.c_int), ("outh", C.c_int), ("out_format", C.c_int),
                ("out", C.c_void_p),
                ("hue", C.c_int), ("brightness", C.c_int), ("contrast", C.c_int),
                ("saturation", C.c_int),
                ("black_point", C.c_int), ("white_point", C.c_int),
                ("scanlines", C.c_int), ("blend", C.c_int),
                ("v_fac", C.c_uint),
                ("ccf", (C.c_int * spec.cc_samples) * spec.vper),
                ("hsync", C.c_int), ("vsync", C.c_int),
                ("rn", C.c_int),
            ]
        CRT.__name__ = "CRT_%s" % spec.name
        _crt_cache[key] = CRT
    return _crt_cache[key]


class RgbSettings(C.Structure):
    """struct NTSC_SETTINGS, CRT_SYSTEM_NTSC (crt_ntsc.h:111-124)."""
    _fields_ = [
        ("data", C.c_void_p), ("format", C.c_int), ("w", C.c_int), ("h", C.c_int),
        ("raw", C.c_int), ("as_color", C.c_int), ("field", C.c_int), ("frame", C.c_int),
        ("hue", C.c_int), ("xoffset", C.c_int), ("yoffset", C.c_int),
        ("iirs_initialized", C.c_int),
    ]


class VhsSettings(C.Structure):
    """struct NTSC_SETTINGS, CRT_SYSTEM_NTSCVHS (crt_ntscvhs.h:133-147)."""
    _fields_ = [
        ("data", C.c_void_p), ("format", C.c_int), ("w", C.c_int), ("h", C.c_int),
        ("raw", C.c_int), ("as_color", C.c_int), ("field", C.c_int), ("frame", C.c_int),
        ("hue", C.c_int), ("xoffset", C.c_int), ("yoffset", C.c_int),
        ("do_aberration", C.c_int),
        ("iirs_initialized", C.c_int),
    ]


class SnesSettings(C.Structure):
    """struct NTSC_SETTINGS, CRT_SYSTEM_SNES (crt_snes.h:108-124)."""
    _fields_ = [
        ("data", C.c_void_p), ("format", C.c_int), ("w", C.c_int), ("h", C.c_int),
        ("raw", C.c_int), ("as_color", C.c_int), ("field", C.c_int), ("frame", C.c_int),
        ("hue", C.c_int), ("xoffset", C.c_int), ("yoffset", C.c_int),
        ("dot_crawl_offset", C.c_int),
        ("iirs_initialized", C.c_int),
    ]


class NesRgbSettings(C.Structure):
    """struct NTSC_SETTINGS, CRT_SYSTEM_NESRGB (crt_nesrgb.h)."""
    _fields_ = [
        ("data", C.c_void_p), ("format", C.c_int), ("w", C.c_int), ("h", C.c_int),
        ("dot_crawl_offset", C.c_int), ("hue", C.c_int), ("xoffset", C.c_int), ("yoffset", C.c_int),
        ("field_initialized", C.c_int),
    ]


class NesSettings(C.Structure):
    """struct NTSC_SETTINGS, CRT_SYSTEM_NES (crt_nes.h:132-143)."""
    _fields_ = [
        ("data", C.c_void_p), ("w", C.c_int), ("h", C.c_int),
        ("border_color", C.c_uint), ("dot_crawl_offset", C.c_int),
        ("hue", C.c_int), ("xoffset", C.c_int), ("yoffset", C.c_int),
        ("field_initialized", C.c_int),
    ]


def settings_struct(spec):
    return {SYS_NTSC: RgbSettings, SYS_VHS: VhsSettings, SYS_NES: NesSettings, SYS_SNES: SnesSettings, SYS_TEMP: SnesSettings, SYS_PV1K: SnesSettings,
            SYS_NESRGB: NesRgbSettings}[spec.system]


def bind_crt_api(lib, spec):
    """Declare the seven reference entry points (crt_core.h:100-139) on a loaded library."""
    crt_p = C.POINTER(crt_struct(spec))
    set_p = C.POINTER(settings_struct(spec))
    lib.crt_init.argtypes = [crt_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.crt_init.restype = None
    lib.crt_resize.argtypes = [crt_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.crt_resize.restype = None
    lib.crt_reset.argtypes = [crt_p]
    lib.crt_reset.restype = None
    lib.crt_modulate.argtypes = [crt_p, set_p]
    lib.crt_modulate.restype = None
    lib.crt_demodulate.argtypes = [crt_p, C.c_int]
    lib.crt_demodulate.restype = None
    lib.crt_bpp4fmt.argtypes = [C.c_int]
    lib.crt_bpp4fmt.restype = C.c_int
    lib.crt_sincos14.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int]
    lib.crt_sincos14.restype = None
    return lib
