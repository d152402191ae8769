"""Loader and thin ctypes bindings for the product libraries (lib/libcrt_b200_<variant>.so).

Two faces of the same library:
  * the reference's own C interface (crt_init / crt_modulate / crt_demodulate ..., host
    buffers, synchronous) -- bound with layout.bind_crt_api, used like the reference;
  * the device-resident batch interface crtx_* (include/crtx_batch.h).

There is deliberately no fallback: a missing library raises, and the library itself aborts
or reports an error if CUDA is unusable -- nothing here ever computes on the CPU.
"""
import ctypes as C
import os

from . import LIB_DIR
from . import layout

VARIANTS = ("ntsc", "ntsc_conv", "ntsc_conv6", "ntsc_conv5", "ntsc_conv4", "vhs", "nes", "nes_p0", "nes_p1", "snes", "nesrgb", "nesrgb_p0", "nesrgb_p1", "template", "pv1k", "ntsc_bloom")


def lib_path(variant):
    return os.path.join(LIB_DIR, "libcrt_b200_%s.so" % variant)


class Monitor(C.Structure):  # crtx_monitor
    _fields_ = [("out", C.c_void_p), ("outw", C.c_int), ("outh", C.c_int), ("out_format", C.c_int),
                ("hue", C.c_int), ("brightness", C.c_int), ("contrast", C.c_int),
                ("saturation", C.c_int), ("black_point", C.c_int), ("white_point", C.c_int),
                ("scanlines", C.c_int), ("blend", C.c_int), ("v_fac", C.c_uint), ("noise", C.c_int),
                ("out_pitch", C.c_int)]


class Source(C.Structure):  # crtx_source
    _fields_ = [("data", C.c_void_p), ("format", C.c_int), ("w", C.c_int), ("h", C.c_int),
                ("raw", C.c_int), ("as_color", C.c_int), ("field", C.c_int), ("frame", C.c_int),
                ("hue", C.c_int), ("xoffset", C.c_int), ("yoffset", C.c_int),
                ("do_aberration", C.c_int), ("dot_crawl_offset", C.c_int), ("reinit", C.c_int), ("pitch", C.c_int)]


def source_table(sources):
    """numpy structured view (shared memory) of a ctypes array of Source: whole columns of settings can be filled with
    array assignments instead of one Python attribute store per field and monitor (video.VideoConverter)."""
    import numpy as np
    dt = np.dtype([(n, "u8" if t is C.c_void_p else "i4") for n, t in Source._fields_], align=True)
    assert dt.itemsize == C.sizeof(Source), (dt.itemsize, C.sizeof(Source))
    return np.frombuffer(sources, dtype=dt)


def row_pitch(t):
    """Bytes between the starts of two rows of an image tensor: (h, w, bpp) bytes, or (h, w) 2-byte NES pixels.  The
    rows may sit anywhere in a larger buffer (a column view of a mosaic, a crop), but each row's pixels must be packed:
    anything else raises ValueError rather than letting a kernel write at the wrong offsets."""
    if t.dim() == 3:
        packed = t.stride(1) == t.shape[2] and t.stride(2) == 1
    elif t.dim() == 2:
        packed = t.stride(1) == 1
    else:
        raise ValueError("an image tensor is (h, w, bpp) or (h, w), not %s" % (tuple(t.shape),))
    if not packed:
        raise ValueError("image rows must hold packed pixels, got strides %s for shape %s" % (t.stride(), tuple(t.shape)))
    return t.stride(0) * t.element_size()


class State(C.Structure):  # crtx_state
    _fields_ = [("ccf", (C.c_int * 5) * 5), ("hsync", C.c_int), ("vsync", C.c_int), ("rn", C.c_int)]


class Line(C.Structure):  # crtx_line
    _fields_ = [("pos", C.c_int), ("wave0", C.c_int), ("wave1", C.c_int), ("beg", C.c_int),
                ("end", C.c_int), ("hsync", C.c_int), ("pad0", C.c_int), ("pad1", C.c_int)]


CRT_EXPORTS = ("crt_init", "crt_resize", "crt_reset", "crt_modulate", "crt_demodulate",
               "crt_bpp4fmt", "crt_sincos14")
CRTX_EXPORTS = ("crtx_system", "crtx_chroma_pattern", "crtx_hres", "crtx_input_size", "crtx_lines",
                "crtx_cc_vper", "crtx_create", "crtx_destroy", "crtx_set_monitors", "crtx_set_state",
                "crtx_get_state", "crtx_seed", "crtx_analog", "crtx_inp", "crtx_read_signal",
                "crtx_write_signal", "crtx_modulate",
                "crtx_demodulate", "crtx_frames_host", "crtx_get_lines", "crtx_get_paths", "crtx_launch_count",
                "crtx_lines2_count", "crtx_set_option", "crtx_get_timing", "crtx_last_error")

_libs = {}


def load(variant):
    """dlopen the product library of one variant and declare both interfaces on it."""
    if variant in _libs:
        return _libs[variant]
    path = lib_path(variant)
    if not os.path.exists(path):
        raise RuntimeError("ntsc-crt_b200: %s is not built (run __graft_entry__.build()); "
                           "there is no CPU fallback" % path)
    lib = C.CDLL(path)
    spec = layout.system_spec(variant)
    layout.bind_crt_api(lib, spec)
    vp, ip = C.c_void_p, C.c_int
    lib.crtx_create.argtypes = [C.POINTER(vp), ip]
    lib.crtx_destroy.argtypes = [vp]
    lib.crtx_destroy.restype = None
    lib.crtx_set_monitors.argtypes = [vp, ip, ip, C.POINTER(Monitor)]
    lib.crtx_set_state.argtypes = [vp, ip, ip, C.POINTER(State), vp]
    lib.crtx_get_state.argtypes = [vp, ip, ip, C.POINTER(State), vp]
    lib.crtx_seed.argtypes = [vp, ip, ip, C.c_uint]
    lib.crtx_analog.argtypes = [vp, ip]
    lib.crtx_analog.restype = vp
    lib.crtx_inp.argtypes = [vp, ip]
    lib.crtx_inp.restype = vp
    lib.crtx_read_signal.argtypes = [vp, ip, ip, vp, vp]
    lib.crtx_write_signal.argtypes = [vp, ip, ip, vp, vp]
    lib.crtx_modulate.argtypes = [vp, ip, ip, C.POINTER(Source), vp]
    lib.crtx_demodulate.argtypes = [vp, ip, ip, vp]
    lib.crtx_frames_host.argtypes = [vp, ip, ip, C.POINTER(Source), C.POINTER(vp), vp]
    lib.crtx_get_lines.argtypes = [vp, ip, C.POINTER(Line), vp]
    lib.crtx_get_paths.argtypes = [vp, ip, ip, C.POINTER(C.c_int), vp]
    lib.crtx_launch_count.argtypes = [vp]
    lib.crtx_launch_count.restype = C.c_long
    lib.crtx_lines2_count.argtypes = [vp]
    lib.crtx_lines2_count.restype = C.c_long
    lib.crtx_set_option.argtypes = [vp, C.c_char_p, ip]
    lib.crtx_get_timing.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_long)]
    lib.crtx_last_error.restype = C.c_char_p
    assert lib.crtx_system() == spec.system and lib.crtx_hres() == spec.hres, "variant mismatch"
    _libs[variant] = lib
    return lib


class CrtxError(RuntimeError):
    pass


class Batch:
    """N monitors advanced one field per step (crtx_* interface), images as torch CUDA tensors."""

    def __init__(self, variant, n):
        self.variant = variant
        self.spec = layout.system_spec(variant)
        self.lib = load(variant)
        self.n = n
        self._ctx = C.c_void_p()
        self._check(self.lib.crtx_create(C.byref(self._ctx), n))
        self.monitors = (Monitor * n)()
        self.sources = (Source * n)()
        self._keep = {}

    def _check(self, rc):
        if rc:
            raise CrtxError(self.lib.crtx_last_error().decode())

    def close(self):
        if self._ctx:
            self.lib.crtx_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_option(self, name, value):
        self._check(self.lib.crtx_set_option(self._ctx, name.encode(), int(value)))

    def set_monitor(self, i, out, fmt=layout.PIX_BGRA, noise=0, **knobs):
        """out: torch uint8 CUDA tensor (outh, outw, bpp) whose rows may be strided (row_pitch); knobs default to
        crt_reset's."""
        pitch = row_pitch(out)
        m = self.monitors[i]
        m.out = out.data_ptr()
        m.outh, m.outw = out.shape[0], out.shape[1]
        m.out_pitch = pitch
        m.out_format = fmt
        m.hue, m.brightness, m.contrast, m.saturation = 0, 0, 180, 10
        m.black_point, m.white_point, m.scanlines, m.blend, m.v_fac = 0, 100, 0, 0, 0
        m.noise = noise
        for k, v in knobs.items():
            setattr(m, k, v)
        self._keep[("out", i)] = out

    def commit_monitors(self, first=0, count=None):
        count = self.n - first if count is None else count
        self._check(self.lib.crtx_set_monitors(self._ctx, first, count,
                                               C.cast(C.byref(self.monitors, first * C.sizeof(Monitor)),
                                                      C.POINTER(Monitor))))

    def set_source(self, i, img, **settings):
        """img: torch CUDA tensor (h, w, bpp) uint8, or (h, w) int16/uint16 for the NES, whose rows may be strided
        (row_pitch)."""
        pitch = row_pitch(img)
        s = self.sources[i]
        s.data = img.data_ptr()
        s.h, s.w = img.shape[0], img.shape[1]
        s.pitch = pitch
        for k, v in settings.items():
            setattr(s, k, v)
        self._keep[("src", i)] = img

    def modulate(self, stream=0, first=0, count=None):
        count = self.n - first if count is None else count
        self._check(self.lib.crtx_modulate(self._ctx, first, count,
                                           C.cast(C.byref(self.sources, first * C.sizeof(Source)),
                                                  C.POINTER(Source)), stream))

    def demodulate(self, stream=0, first=0, count=None):
        count = self.n - first if count is None else count
        self._check(self.lib.crtx_demodulate(self._ctx, first, count, stream))

    def frames_host(self, host_ptrs, stream=0, first=0, count=None):
        count = self.n - first if count is None else count
        arr = (C.c_void_p * count)(*host_ptrs)
        self._check(self.lib.crtx_frames_host(self._ctx, first, count,
                                              C.cast(C.byref(self.sources, first * C.sizeof(Source)),
                                                     C.POINTER(Source)), arr, stream))

    def get_state(self, first=0, count=None, stream=0):
        count = self.n - first if count is None else count
        st = (State * count)()
        self._check(self.lib.crtx_get_state(self._ctx, first, count, st, stream))
        return st

    def set_state(self, states, first=0, stream=0):
        self._check(self.lib.crtx_set_state(self._ctx, first, len(states), states, stream))

    def seed(self, seed, first=0, count=None):
        """VHS: put the monitors' rand() replica in the state srand(seed) leaves glibc in."""
        count = self.n - first if count is None else count
        self._check(self.lib.crtx_seed(self._ctx, first, count, seed))

    def get_lines(self, i, stream=0):
        t = (Line * self.spec.lines)()
        self._check(self.lib.crtx_get_lines(self._ctx, i, t, stream))
        return t

    PATH_GENERIC_EQ = 1  # CRTX_PATH_GENERIC_EQ: the last demodulate decoded the monitor with the wrap-exact equaliser
    PATH_STAGED_MOD = 2  # CRTX_PATH_STAGED_MOD: the last modulate encoded its picture with the staged encoder
    PATH_ROW16 = 4  # CRTX_PATH_ROW16: the line pass writes the monitor's rows with 16-byte stores (16-byte aligned rows)

    def paths(self, first=0, count=None, stream=0):
        """crtx_get_paths: per monitor, the PATH_* bits of the code paths its last modulate and demodulate took"""
        count = self.n - first if count is None else count
        out = (C.c_int * count)()
        self._check(self.lib.crtx_get_paths(self._ctx, first, count, out, stream))
        return list(out)

    def analog_ptr(self, i):
        return self.lib.crtx_analog(self._ctx, i)

    def inp_ptr(self, i):
        return self.lib.crtx_inp(self._ctx, i)

    def signal(self, i, which="analog", stream=0):
        """Copy monitor i's analog[] or inp[] to a numpy int8 array (synchronises the stream)."""
        import numpy as np
        host = np.empty(self.spec.input_size, dtype=np.int8)
        self._check(self.lib.crtx_read_signal(self._ctx, i, 0 if which == "analog" else 1,
                                              host.ctypes.data, stream))
        return host

    def write_signal(self, i, data, which="analog", stream=0):
        import numpy as np
        host = np.ascontiguousarray(data, dtype=np.int8)
        assert host.size == self.spec.input_size
        self._check(self.lib.crtx_write_signal(self._ctx, i, 0 if which == "analog" else 1,
                                               host.ctypes.data, stream))

    KERNELS = ("mod_skeleton", "mod_picture", "noise", "sync", "lines")

    def timing(self):
        """{kernel: (total_ms, launches)} since the last call (needs set_option("timing", 1))."""
        ms = (C.c_float * 5)()
        cnt = (C.c_long * 5)()
        self._check(self.lib.crtx_get_timing(self._ctx, ms, cnt))
        return {k: (ms[i], cnt[i]) for i, k in enumerate(self.KERNELS)}

    @property
    def launches(self):
        return self.lib.crtx_launch_count(self._ctx)

    @property
    def lines2_launches(self):
        """line passes so far that took k_lines2 (csrc/crt_lines2.cuh) instead of k_lines"""
        return self.lib.crtx_lines2_count(self._ctx)
