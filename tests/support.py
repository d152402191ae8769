"""Test support: three interchangeable engines over the same call sequence.

  RefEngine      the UNMODIFIED reference compiled into oracle/_ref/libref_<variant>.so
  OracleEngine   our CPU restatement, oracle/libcrt_oracle.so
  ProductEngine  the CUDA product library, ntsc-crt_b200/lib/libcrt_b200_<variant>.so,
                 through the same C-ABI as the reference (defined in test files that
                 need it; shares CEngine below)

All of them expose: set(**knobs), modulate(img, **settings), demodulate(noise) and the
state arrays analog / inp / out / ccf / hsync / vsync / rn.
"""
import atexit
import ctypes as C
import hashlib
import json
import os

import numpy as np

import pkgload

pkg = pkgload.load()
from ntsc_crt_b200 import layout  # noqa: E402

ROOT = pkg.REPO_ROOT
ORACLE_DIR = os.path.join(ROOT, "oracle")
REF_DIR = os.path.join(ORACLE_DIR, "_ref")

KNOBS = ("hue", "brightness", "contrast", "saturation", "black_point", "white_point",
         "scanlines", "blend", "v_fac")


def ref_path(variant):
    return os.path.join(REF_DIR, "libref_%s.so" % variant)


def have_ref(variant="ntsc"):
    return os.path.exists(ref_path(variant))


# ----------------------------------------------------------------------------------
# synthetic inputs (SURVEY.md 8d): seeded LCG noise, colour bars, 1-px checker, flats
# ----------------------------------------------------------------------------------

def lcg_image(w, h, bpp=4, seed=12345):
    """x = x*1664525 + 1013904223; px = (x >> 8) & 0xffffff (SURVEY.md 8d config 1)."""
    n = w * h
    a, c, m = 1664525, 1013904223, 0xFFFFFFFF
    v = seed & m
    out = np.empty(n, dtype=np.uint32)
    for i in range(n):
        v = (v * a + c) & m
        out[i] = (v >> 8) & 0xFFFFFF
    img = np.zeros((h, w, bpp), dtype=np.uint8)
    img[..., 0] = (out & 0xFF).reshape(h, w)
    img[..., 1] = ((out >> 8) & 0xFF).reshape(h, w)
    img[..., 2] = ((out >> 16) & 0xFF).reshape(h, w)
    if bpp == 4:
        img[..., 3] = 0xFF
    return img


def rand_image(w, h, bpp=4, seed=1):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, size=(h, w, bpp), dtype=np.uint8)


def bars_image(w, h, bpp=4, fmt=layout.PIX_BGRA):
    """75% colour bars over a luma ramp and a 1-px checker (artifact colours)."""
    cols = [(191, 191, 191), (191, 191, 0), (0, 191, 191), (0, 191, 0),
            (191, 0, 191), (191, 0, 0), (0, 0, 191), (0, 0, 0)]
    rgb = np.zeros((h, w, 3), dtype=np.uint8)
    for x in range(w):
        rgb[: (2 * h) // 3, x] = cols[min(7, x * 8 // w)]
    ramp = (np.arange(w) * 255 // max(1, w - 1)).astype(np.uint8)
    rgb[(2 * h) // 3: (5 * h) // 6] = ramp[None, :, None]
    yy, xx = np.mgrid[(5 * h) // 6: h, 0:w]
    rgb[(5 * h) // 6:] = (((xx + yy) & 1) * 255).astype(np.uint8)[..., None]
    return pack_rgb(rgb, fmt)


def pack_rgb(rgb, fmt):
    """(h, w, 3) RGB -> (h, w, bpp) in one of the CRT_PIX_FORMATs."""
    h, w, _ = rgb.shape
    bpp = layout.bpp4fmt(fmt)
    out = np.full((h, w, bpp), 0xFF, dtype=np.uint8)
    order = {layout.PIX_RGB: (0, 1, 2), layout.PIX_BGR: (2, 1, 0),
             layout.PIX_ARGB: (1, 2, 3), layout.PIX_RGBA: (0, 1, 2),
             layout.PIX_ABGR: (3, 2, 1), layout.PIX_BGRA: (2, 1, 0)}[fmt]
    for ch, pos in enumerate(order):
        out[..., pos] = rgb[..., ch]
    return out


def nes_image(w=256, h=240, seed=3, rainbow=False):
    """9-bit PPU pixels (crt_nes.c:44-60): hue[3:0] level[5:4] emphasis[8:6]."""
    if rainbow:
        xx = np.arange(w)[None, :] + np.zeros((h, 1), dtype=np.int64)
        yy = np.arange(h)[:, None] + np.zeros((1, w), dtype=np.int64)
        hue = 1 + ((xx + yy // 8) % 12)
        lvl = 1 + ((xx // 16) % 3)
        return (hue | (lvl << 4) | (((yy // 60) % 8) << 6)).astype(np.uint16)
    rng = np.random.default_rng(seed)
    return rng.integers(0, 512, size=(h, w), dtype=np.uint16)


# ----------------------------------------------------------------------------------
# engines
# ----------------------------------------------------------------------------------

class CEngine:
    """Drives any library exporting the reference's C interface (crt_core.h:100-139)."""

    def __init__(self, lib_path, variant, outw, outh, fmt=layout.PIX_BGRA, out=None):
        self.spec = layout.system_spec(variant)
        self.lib = layout.bind_crt_api(C.CDLL(lib_path), self.spec)
        self.CRT = layout.crt_struct(self.spec)
        self.Settings = layout.settings_struct(self.spec)
        self.crt = self.CRT()
        bpp = max(1, layout.bpp4fmt(fmt))
        self.out = out if out is not None else np.zeros((outh, outw, bpp), dtype=np.uint8)
        self.lib.crt_init(C.byref(self.crt), outw, outh, fmt, self.out.ctypes.data)
        self.settings = self.Settings()  # zeroed, as crt_ntsc.h:122 demands
        self._img = None

    def set(self, **kw):
        for k, v in kw.items():
            assert k in KNOBS or k in ("hsync", "vsync", "rn"), k
            setattr(self.crt, k, v)
        return self

    def resize(self, outw, outh, fmt, out):
        self.out = out
        self.lib.crt_resize(C.byref(self.crt), outw, outh, fmt, out.ctypes.data)

    def reset(self):
        self.lib.crt_reset(C.byref(self.crt))

    def modulate(self, img, **kw):
        self._img = np.ascontiguousarray(img)
        s = self.settings
        s.data = self._img.ctypes.data
        s.h, s.w = self._img.shape[0], self._img.shape[1]
        for k, v in kw.items():
            setattr(s, k, v)
        self.lib.crt_modulate(C.byref(self.crt), C.byref(s))

    def demodulate(self, noise=0):
        self.lib.crt_demodulate(C.byref(self.crt), noise)

    @property
    def analog(self):
        return np.frombuffer(self.crt, dtype=np.int8, count=self.spec.input_size, offset=0).copy()

    @property
    def inp(self):
        return np.frombuffer(self.crt, dtype=np.int8, count=self.spec.input_size,
                             offset=self.spec.input_size).copy()

    @property
    def ccf(self):
        return np.array([[self.crt.ccf[n][x] for x in range(self.spec.cc_samples)] for n in range(self.spec.vper)])

    @property
    def hsync(self):
        return self.crt.hsync

    @property
    def vsync(self):
        return self.crt.vsync

    @property
    def rn(self):
        return self.crt.rn

    def state(self):
        return dict(analog=self.analog, inp=self.inp, out=self.out.copy(), ccf=self.ccf,
                    hsync=self.hsync, vsync=self.vsync, rn=self.rn)


# ----------------------------------------------------------------------------------
# the reference, recorded
# ----------------------------------------------------------------------------------
# A checkout without the reference sources has no oracle/_ref.  The comparisons with the reference still run there:
# tests/golden/ref_states.json holds, per test and in call order, digests of every reference state the test compares
# and every value it probes from a reference build.  Where oracle/_ref exists the reference itself is used, and
#     CRT_RECORD_REF=1 python -m pytest tests/<file>.py
# rewrites the records of the tests it runs.

REF_STATES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_states.json")
RECORD = os.environ.get("CRT_RECORD_REF") == "1"
_records = None
_cursor = {}
_recorded_now = {}


def digest(a):
    """64-bit sha256 prefix of an array's bytes (what the records keep of large arrays)"""
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def _test_id():
    """the running test as `<file>::<name>[params]`, independent of the directory pytest was started from"""
    t = os.environ.get("PYTEST_CURRENT_TEST", "").rsplit(" (", 1)[0]
    f, _, rest = t.partition("::")
    return os.path.basename(f) + "::" + rest


def _load_records():
    global _records
    if _records is None:
        _records = json.load(open(REF_STATES)) if os.path.exists(REF_STATES) else {}
    return _records


def _save_records():
    recs = dict(_load_records())
    recs.update(_recorded_now)
    with open(REF_STATES, "w") as f:
        f.write("{\n" + ",\n".join("%s: %s" % (json.dumps(k), json.dumps(recs[k], separators=(",", ":")))
                                   for k in sorted(recs)) + "\n}\n")


def _record(value):
    if RECORD:
        if not _recorded_now:
            atexit.register(_save_records)
        tid = _test_id()
        _recorded_now.setdefault(tid, []).append(value)  # (replaces what the file held for this test)
    return value


def _replay():
    tid = _test_id()
    recs = _load_records().get(tid)
    k = _cursor.get(tid, 0)
    assert recs is not None and k < len(recs), (
        "%s: no recorded reference value #%d in %s (oracle/_ref is not built here)" % (tid, k, REF_STATES))
    _cursor[tid] = k + 1
    return recs[k]


def begin_reference_scope():
    """start of a test: its recorded reference values are consumed from the first one again (and re-recorded afresh)"""
    tid = _test_id()
    _cursor.pop(tid, None)
    _recorded_now.pop(tid, None)


def end_reference_scope():
    """end of a test: one that replayed reference values must have compared every one of them"""
    tid = _test_id()
    k = _cursor.get(tid)
    if k is not None:
        n = len(_load_records().get(tid, []))
        assert k == n, "%s: compared %d of the %d recorded reference values" % (tid, k, n)


def from_reference(path, compute):
    """compute(path) where the reference build `path` (under oracle/_ref) exists, else the value it gave when recorded.
    The value must be JSON data: probe large outputs through digest()."""
    if os.path.exists(path):
        return _record(compute(path))
    return _replay()


STATE_KEYS = ("sync", "ccf", "analog", "inp", "out")  # a recorded state: these, in this order


def state_digest(st):
    return dict(sync=[int(st["hsync"]), int(st["vsync"]), int(st["rn"])], ccf=digest(np.asarray(st["ccf"], dtype=np.int64)),
                analog=digest(st["analog"]), inp=digest(st["inp"]), out=digest(st["out"]))


class RefState(dict):
    """state() of the live reference: recorded when a comparison consumes it (after any masking the test applies)"""


class RecordedState(dict):
    """state() of the replayed reference: state_digest() of what the reference held at this point of the test"""


class _LiveRef(CEngine):
    def __init__(self, variant, outw, outh, fmt=layout.PIX_BGRA, out=None, seed=None):
        super().__init__(ref_path(variant), variant, outw, outh, fmt, out)
        self.lib.ref_srand.argtypes = [C.c_uint]
        if seed is not None:
            self.lib.ref_srand(seed)

    def state(self):
        return RefState(super().state())


class _ReplayRef:
    """The reference where oracle/_ref is absent: the calls change nothing, state() hands out the recorded states in order."""

    def __init__(self, variant, outw, outh, fmt=layout.PIX_BGRA, out=None, seed=None):
        self.spec = layout.system_spec(variant)

    def set(self, **kw):
        return self

    def modulate(self, img, **kw):
        pass

    def demodulate(self, noise=0):
        pass

    def state(self):
        return RecordedState(zip(STATE_KEYS, _replay()))


def RefEngine(variant, outw, outh, fmt=layout.PIX_BGRA, out=None, seed=None):
    """the compiled reference (oracle/_ref/libref_<variant>.so), or its recorded states where that is not built"""
    cls = _LiveRef if have_ref(variant) else _ReplayRef
    return cls(variant, outw, outh, fmt, out, seed)


class _OSys(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        "system", "chroma_pattern", "hres", "vres", "input_size", "top", "bot", "lines",
        "cc_vper", "hsync_window", "vsync_window", "hsync_thresh", "vsync_thresh",
        "sync_beg", "bw_beg", "cb_beg", "av_beg", "av_len", "burst_len",
        "white_level", "burst_level", "black_level", "blank_level", "sync_level",
        "vhs_noise", "nes_vsync_end")] + [("eq", (C.c_int * 5) * 3), ("iir_c", C.c_int * 3), ("conv", C.c_int), ("cc_samples", C.c_int), ("bloom", C.c_int)]


class _OMonitor(C.Structure):
    _fields_ = [
        ("analog", C.POINTER(C.c_byte)), ("inp", C.POINTER(C.c_byte)),
        ("outw", C.c_int), ("outh", C.c_int), ("out_format", C.c_int),
        ("out", C.c_void_p),
        ("hue", C.c_int), ("brightness", C.c_int), ("contrast", C.c_int),
        ("saturation", C.c_int), ("black_point", C.c_int), ("white_point", C.c_int),
        ("scanlines", C.c_int), ("blend", C.c_int), ("v_fac", C.c_uint),
        ("ccf", (C.c_int * 5) * 5), ("hsync", C.c_int), ("vsync", C.c_int), ("rn", C.c_int),
        ("last_noise", C.c_int),
    ]


class _ORgb(C.Structure):
    _fields_ = [("data", C.c_void_p)] + [(n, C.c_int) for n in (
        "format", "w", "h", "raw", "as_color", "field", "frame", "hue", "xoffset",
        "yoffset", "do_aberration", "dot_crawl_offset")]


class _ONes(C.Structure):
    _fields_ = [("data", C.c_void_p)] + [(n, C.c_int) for n in (
        "w", "h", "dot_crawl_offset", "hue", "xoffset", "yoffset", "field_initialized")]


class _ONesRgb(C.Structure):
    _fields_ = [("data", C.c_void_p)] + [(n, C.c_int) for n in (
        "format", "w", "h", "dot_crawl_offset", "hue", "xoffset", "yoffset", "field_initialized")]


class _ORand(C.Structure):
    _fields_ = [("r", C.c_uint * 31), ("f", C.c_int), ("b", C.c_int)]


class OLine(C.Structure):
    _fields_ = [("skip", C.c_int), ("beg", C.c_int), ("end", C.c_int), ("hsync", C.c_int),
                ("pos", C.c_int), ("wave", C.c_int * 4), ("wave_i", C.c_int * 5), ("wave_q", C.c_int * 5)]


_oracle = None


def oracle_lib():
    global _oracle
    if _oracle is None:
        lib = C.CDLL(os.path.join(ORACLE_DIR, "libcrt_oracle.so"))
        lib.ocrt_system.restype = C.POINTER(_OSys)
        lib.ocrt_system.argtypes = [C.c_int, C.c_int]
        lib.ocrt_system_conv.restype = C.POINTER(_OSys)
        lib.ocrt_system_conv.argtypes = [C.c_int, C.c_int]
        lib.ocrt_system_conv_taps.restype = C.POINTER(_OSys)
        lib.ocrt_system_conv_taps.argtypes = [C.c_int, C.c_int, C.c_int]
        lib.ocrt_system_bloom.restype = C.POINTER(_OSys)
        lib.ocrt_system_bloom.argtypes = [C.c_int, C.c_int]
        lib.ocrt_monitor_create.argtypes = [C.POINTER(_OSys), C.POINTER(_OMonitor), C.c_int,
                                            C.c_int, C.c_int, C.c_void_p]
        lib.ocrt_monitor_create.restype = C.c_int
        lib.ocrt_monitor_destroy.argtypes = [C.POINTER(_OMonitor)]
        lib.ocrt_monitor_reset.argtypes = [C.POINTER(_OMonitor)]
        lib.ocrt_encode_rgb.argtypes = [C.POINTER(_OSys), C.POINTER(_OMonitor),
                                        C.POINTER(_ORgb), C.POINTER(_ORand)]
        lib.ocrt_encode_nes.argtypes = [C.POINTER(_OSys), C.POINTER(_OMonitor), C.POINTER(_ONes)]
        lib.ocrt_encode_snes.argtypes = [C.POINTER(_OSys), C.POINTER(_OMonitor), C.POINTER(_ORgb)]
        lib.ocrt_encode_nesrgb.argtypes = [C.POINTER(_OSys), C.POINTER(_OMonitor), C.POINTER(_ONesRgb)]
        lib.ocrt_encode_template.argtypes = [C.POINTER(_OSys), C.POINTER(_OMonitor), C.POINTER(_ORgb)]
        lib.ocrt_encode_pv1k.argtypes = [C.POINTER(_OSys), C.POINTER(_OMonitor), C.POINTER(_ORgb)]
        lib.ocrt_decode.argtypes = [C.POINTER(_OSys), C.POINTER(_OMonitor), C.c_int,
                                    C.POINTER(_ORand)]
        lib.ocrt_noise_pass.argtypes = lib.ocrt_decode.argtypes
        lib.ocrt_sync_pass.argtypes = [C.POINTER(_OSys), C.POINTER(_OMonitor), C.POINTER(OLine)]
        lib.ocrt_sync_pass.restype = C.c_int
        lib.ocrt_line_pass.argtypes = [C.POINTER(_OSys), C.POINTER(_OMonitor), C.POINTER(OLine),
                                       C.c_int, C.c_int]
        lib.ocrt_rand_seed.argtypes = [C.POINTER(_ORand), C.c_uint]
        lib.ocrt_rand_next.argtypes = [C.POINTER(_ORand)]
        lib.ocrt_rand_next.restype = C.c_int
        lib.ocrt_sincos14.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int]
        lib.ocrt_bpp.argtypes = [C.c_int]
        lib.ocrt_bpp.restype = C.c_int
        lib.ocrt_lcg_jump.argtypes = [C.c_uint, C.POINTER(C.c_uint), C.POINTER(C.c_uint)]
        _oracle = lib
    return _oracle


class OracleEngine:
    """Same call sequence, on the CPU restatement."""

    def __init__(self, variant, outw, outh, fmt=layout.PIX_BGRA, out=None, seed=1):
        self.spec = layout.system_spec(variant)
        self.lib = oracle_lib()
        taps = layout.conv_taps(variant)
        if variant.endswith("_bloom"):
            self.sys = self.lib.ocrt_system_bloom(self.spec.system, self.spec.pattern)
        else:
            self.sys = (self.lib.ocrt_system_conv_taps(self.spec.system, self.spec.pattern, taps) if taps
                        else self.lib.ocrt_system(self.spec.system, self.spec.pattern))
        assert self.sys, "unknown system"
        self.mon = _OMonitor()
        bpp = max(1, layout.bpp4fmt(fmt))
        self.out = out if out is not None else np.zeros((outh, outw, bpp), dtype=np.uint8)
        assert self.lib.ocrt_monitor_create(self.sys, C.byref(self.mon), outw, outh, fmt,
                                            self.out.ctypes.data)
        self.rand = _ORand()
        self.lib.ocrt_rand_seed(C.byref(self.rand), seed)
        self.rgb = _ORgb()
        self.nes = _ONes()
        self.nesrgb = _ONesRgb()
        self._img = None

    def __del__(self):
        try:
            self.lib.ocrt_monitor_destroy(C.byref(self.mon))
        except Exception:
            pass

    def set(self, **kw):
        for k, v in kw.items():
            setattr(self.mon, k, v)
        return self

    def resize(self, outw, outh, fmt, out):
        self.out = out
        self.mon.outw, self.mon.outh, self.mon.out_format = outw, outh, fmt
        self.mon.out = out.ctypes.data

    def reset(self):
        self.lib.ocrt_monitor_reset(C.byref(self.mon))

    def modulate(self, img, **kw):
        self._img = np.ascontiguousarray(img)
        if self.spec.system == layout.SYS_NES:
            s = self.nes
            kw.pop("border_color", None)
        elif self.spec.system == layout.SYS_NESRGB:
            s = self.nesrgb
        else:
            s = self.rgb
            kw.pop("iirs_initialized", None)
        s.data = self._img.ctypes.data
        s.h, s.w = self._img.shape[0], self._img.shape[1]
        for k, v in kw.items():
            setattr(s, k, v)
        if self.spec.system == layout.SYS_NES:
            self.lib.ocrt_encode_nes(self.sys, C.byref(self.mon), C.byref(s))
        elif self.spec.system == layout.SYS_SNES:
            self.lib.ocrt_encode_snes(self.sys, C.byref(self.mon), C.byref(s))
        elif self.spec.system == layout.SYS_NESRGB:
            self.lib.ocrt_encode_nesrgb(self.sys, C.byref(self.mon), C.byref(s))
        elif self.spec.system == layout.SYS_TEMP:
            self.lib.ocrt_encode_template(self.sys, C.byref(self.mon), C.byref(s))
        elif self.spec.system == layout.SYS_PV1K:
            self.lib.ocrt_encode_pv1k(self.sys, C.byref(self.mon), C.byref(s))
        else:
            self.lib.ocrt_encode_rgb(self.sys, C.byref(self.mon), C.byref(s), C.byref(self.rand))

    def demodulate(self, noise=0):
        self.lib.ocrt_decode(self.sys, C.byref(self.mon), noise, C.byref(self.rand))

    # staged decode, for comparing the kernels' intermediate tables
    def noise_pass(self, noise=0):
        self.lib.ocrt_noise_pass(self.sys, C.byref(self.mon), noise, C.byref(self.rand))

    def sync_pass(self):
        table = (OLine * self.spec.lines)()
        field = self.lib.ocrt_sync_pass(self.sys, C.byref(self.mon), table)
        return field, table

    def line_pass(self, table, first=0, count=None):
        self.lib.ocrt_line_pass(self.sys, C.byref(self.mon), table, first,
                                self.spec.lines if count is None else count)

    @property
    def analog(self):
        return np.ctypeslib.as_array(self.mon.analog, shape=(self.spec.input_size,)).astype(np.int8).copy()

    @property
    def inp(self):
        return np.ctypeslib.as_array(self.mon.inp, shape=(self.spec.input_size,)).astype(np.int8).copy()

    @property
    def ccf(self):
        return np.array([[self.mon.ccf[n][x] for x in range(self.spec.cc_samples)] for n in range(self.spec.vper)])

    @property
    def hsync(self):
        return self.mon.hsync

    @property
    def vsync(self):
        return self.mon.vsync

    @property
    def rn(self):
        return self.mon.rn

    def state(self):
        return dict(analog=self.analog, inp=self.inp, out=self.out.copy(), ccf=self.ccf,
                    hsync=self.hsync, vsync=self.vsync, rn=self.rn)


def assert_same_state(a, b, what=""):
    """Bit-exact comparison of two engine states with a useful first-mismatch report.  `a` may be a reference state,
    live or recorded (see RefEngine)."""
    if isinstance(a, RecordedState):
        got = state_digest(b)
        for key in STATE_KEYS:
            assert got[key] == a[key], "%s %s: %r != %r (the reference's, recorded)" % (what, key, got[key], a[key])
        return
    if isinstance(a, RefState):
        d = state_digest(a)
        _record([d[k] for k in STATE_KEYS])
    for key in ("hsync", "vsync", "rn"):
        assert a[key] == b[key], "%s %s: %r != %r" % (what, key, a[key], b[key])
    assert np.array_equal(a["ccf"], b["ccf"]), "%s ccf: %r != %r" % (what, a["ccf"], b["ccf"])
    for key in ("analog", "inp", "out"):
        x, y = a[key], b[key]
        assert x.shape == y.shape, "%s %s shape %r != %r" % (what, key, x.shape, y.shape)
        if not np.array_equal(x, y):
            bad = np.argwhere(x != y)
            first = tuple(int(v) for v in bad[0])
            raise AssertionError("%s %s: %d mismatches, first at %r: %r != %r" % (
                what, key, len(bad), first, x[first], y[first]))


def cli_sequence(engine, img, noise=0, progressive=False, field=0, **settings):
    """The accumulate loop of the CLI driver (crt_main.c:221-255)."""
    engine.set(blend=1, scanlines=1)
    s = dict(settings)
    s.setdefault("as_color", 1)
    f, fr = field & 1, 0
    for it in range(4):
        engine.modulate(img, field=f, frame=fr, **s)
        engine.demodulate(noise)
        if not progressive:
            f ^= 1
            engine.modulate(img, field=f, frame=fr, **s)
            engine.demodulate(noise)
            if (it & 1) == 0:
                fr ^= 1


class ProductEngine(CEngine):
    """The CUDA product library through the reference's own C interface (host buffers)."""

    def __init__(self, variant, outw, outh, fmt=layout.PIX_BGRA, out=None):
        from ntsc_crt_b200 import capi
        capi.load(variant)  # raises if the library is not built: there is no fallback
        super().__init__(capi.lib_path(variant), variant, outw, outh, fmt, out)


def diff_report(name, x, y, shape_hint=None):
    """One-line description of how two arrays differ (for the GPU diagnostics)."""
    x = np.asarray(x)
    y = np.asarray(y)
    if x.shape != y.shape:
        return "%s: SHAPE %r vs %r" % (name, x.shape, y.shape)
    bad = np.argwhere(x != y)
    if len(bad) == 0:
        return "%s: identical (%d values)" % (name, x.size)
    first = tuple(int(v) for v in bad[0])
    last = tuple(int(v) for v in bad[-1])
    return "%s: %d/%d differ, first %r got %r want %r, last %r" % (
        name, len(bad), x.size, first, x[first], y[first], last)
