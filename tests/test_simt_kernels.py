"""The GPU parity tests, run on the CPU through the SIMT interpreter (tests/simt/): the product's CUDA sources,
unchanged, compiled by g++ and executed one CUDA thread per fiber.  This is how kernel logic is checked in a
container without a GPU -- block / warp synchronisation, shuffles, ballots, mbarriers and deferred bulk copies
included -- against the same oracle and reference the `-m gpu` tests use.  It says nothing about timing, and the
`-m gpu` tests on the H100 remain the parity proof of the real binary.

The test bodies are the ones of tests/test_gpu_*.py, re-collected here without the gpu mark; a fixture points the
loaders at tests/simt/_build/libcrt_simt_<variant>.so and lets "device" tensors be host tensors.
"""
import os
import sys

import pytest

import support as S
from ntsc_crt_b200 import capi

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "simt"))
import build as simt_build  # noqa: E402

import test_gpu_batch_api as _api  # noqa: E402
import test_gpu_batch_fuzz as _bfuzz  # noqa: E402
import test_gpu_bloom as _bloom  # noqa: E402
import test_gpu_conv as _conv  # noqa: E402
import test_gpu_dropin_cli as _cli  # noqa: E402
import test_gpu_edges as _edges  # noqa: E402
import test_gpu_fullsize as _fullsize  # noqa: E402
import test_gpu_fuzz as _fuzz  # noqa: E402
import test_gpu_guard_edges as _guard  # noqa: E402
import test_gpu_inp_elision as _elision  # noqa: E402
import test_gpu_lines2 as _lines2  # noqa: E402
import test_gpu_lineshard as _lineshard  # noqa: E402
import test_gpu_parity as _parity  # noqa: E402
import test_gpu_pv1k as _pv1k  # noqa: E402
import test_gpu_template as _template  # noqa: E402
import test_gpu_still_cli as _still  # noqa: E402
import test_gpu_video as _video  # noqa: E402
import test_gpu_video_driver as _vdriver  # noqa: E402
import test_gpu_video_convert_unmodified as _vconv  # noqa: E402
import test_gpu_vfac as _vfac  # noqa: E402
import test_gpu_vhs as _vhs  # noqa: E402
import test_gpu_wire as _wire  # noqa: E402


ASAN = os.environ.get("SIMT_ASAN") == "1"  # see tests/simt/build.py: run with LD_PRELOAD=libasan.so SIMT_TIGHT_ALLOC=1


def _lib_path(variant):
    p = simt_build.lib_path(variant)
    return os.path.join(simt_build.OUT, "asan", os.path.basename(p)) if ASAN else p


@pytest.fixture(scope="session")
def simt_libs():
    simt_build.build(asan=ASAN)
    # The C drivers (the reference's unmodified crt_main.c, tools/crtx_video.c) are linked against
    # libcrt_b200_ntsc.so with a RUNPATH; a directory earlier on LD_LIBRARY_PATH that holds the interpreter build
    # under that name makes the very same binaries run their kernels on the CPU.
    stand_in = os.path.join(simt_build.OUT, "stand_in")
    os.makedirs(stand_in, exist_ok=True)
    for v in simt_build.variant_defines():
        link = os.path.join(stand_in, "libcrt_b200_%s.so" % v)
        if os.path.lexists(link):
            os.remove(link)
        os.symlink(_lib_path(v), link)
    return _lib_path


@pytest.fixture(autouse=True)
def simt_backend(simt_libs, monkeypatch):
    import torch
    monkeypatch.setenv("LD_LIBRARY_PATH", os.path.join(simt_build.OUT, "stand_in") + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))
    monkeypatch.setattr(capi, "lib_path", simt_libs)
    monkeypatch.setattr(capi, "_libs", {})
    real_zeros, real_empty, real_full = torch.zeros, torch.empty, torch.full

    def host_only(fn):
        def wrapped(*a, **kw):
            kw.pop("device", None)
            return fn(*a, **kw)
        return wrapped
    monkeypatch.setattr(torch, "zeros", host_only(real_zeros))
    monkeypatch.setattr(torch, "empty", host_only(real_empty))
    monkeypatch.setattr(torch, "full", host_only(real_full))
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **kw: self)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self, *a, **kw: self)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **kw: None)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **kw: type("S", (), {"cuda_stream": 0})())
    yield


def _adopt(module, prefix):
    for name in dir(module):
        if name.startswith("test_"):
            globals()["test_%s_%s" % (prefix, name[5:])] = getattr(module, name)


_adopt(_parity, "parity")
_adopt(_conv, "conv")
_adopt(_fuzz, "fuzz")
_adopt(_lineshard, "lineshard")
_adopt(_lines2, "lines2")
_adopt(_video, "video")
_adopt(_template, "template")
_adopt(_pv1k, "pv1k")
_adopt(_wire, "wire")
_adopt(_bloom, "bloom")
_adopt(_api, "api")
_adopt(_guard, "guard")
_adopt(_vfac, "vfac")
_adopt(_vhs, "vhs")
test_cli_unmodified_cli_driver_is_byte_identical = _cli.test_unmodified_cli_driver_is_byte_identical
_adopt(_still, "still")
test_vconv_unmodified_video_convert_runs_against_the_library = _vconv.test_unmodified_video_convert_runs_against_the_library
# k_sync leaving inp[] unwritten and the line pass that then decodes from analog[] must agree (not the 264-monitor batch)
test_elision_mixed_batch = _elision.test_mixed_batch
test_elision_poked_minus_128 = _elision.test_poked_minus_128
test_elision_inp_after_a_later_modulate = _elision.test_inp_after_a_later_modulate


def _bare(fn):
    """the test function without its marks (to give it a shorter parameter list here)"""
    import types
    g = types.FunctionType(fn.__code__, fn.__globals__, fn.__name__, fn.__defaults__, fn.__closure__)
    g.__doc__ = fn.__doc__
    return g


@pytest.fixture(autouse=True)
def small_vhs_runs(monkeypatch):
    """tests/test_gpu_vhs.py with 4 monitors, 3 fields and one case of two calls per seed: every monitor and field costs
    a whole interpreted noise pass here"""
    monkeypatch.setattr(_vhs, "BATCH", 4)
    monkeypatch.setattr(_vhs, "FIELDS", 3)
    monkeypatch.setattr(_vhs, "SWEEP_CASES", 1)
    monkeypatch.setattr(_vhs, "SWEEP_CALLS", 2)


_BFUZZ_FULL = dict(MAX_MONITORS=_bfuzz.MAX_MONITORS, FIELDS=_bfuzz.FIELDS, MAX_OUTW=_bfuzz.MAX_OUTW)


@pytest.fixture(autouse=True)
def small_batch_sweeps(monkeypatch):
    """tests/test_gpu_batch_fuzz.py with at most 4 monitors, 3 fields and outputs of 832 pixels or less; its streams are
    stand-ins here (the interpreter runs every call in order, whatever the stream)"""
    import contextlib
    monkeypatch.setattr(_bfuzz, "MAX_MONITORS", 4)
    monkeypatch.setattr(_bfuzz, "FIELDS", 3)
    monkeypatch.setattr(_bfuzz, "MAX_OUTW", 832)
    monkeypatch.setattr(_bfuzz, "make_streams", lambda k: [type("S", (), {"cuda_stream": 0})() for _ in range(k)])
    monkeypatch.setattr(_bfuzz, "on_stream", lambda s: contextlib.nullcontext())


# one draw each of a few systems (a whole draw of every variant costs minutes here); the coverage of the draws is the
# GPU test's
BFUZZ_CASES = [("ntsc", 1), ("ntsc", 2), ("pv1k", 1), ("nes", 1), ("nesrgb", 1), ("vhs", 1), ("ntsc_conv", 1), ("ntsc_bloom", 1),
                ("nes_border", 1), ("ntsc_nosync", 1)]


@pytest.mark.parametrize("variant,seed", BFUZZ_CASES, ids=["%s_seed%d" % c for c in BFUZZ_CASES])
def test_bfuzz_random_batches(variant, seed):
    _bfuzz.sweep(variant, seed)


def test_bfuzz_full_size_draw(monkeypatch):
    """one draw at the GPU test's sizes: ntsc seed 5 puts two monitors that differ in scanlines into one k_lines2 pair on
    an image with more rows than lines, where scanlines changes the rows a line writes"""
    for name, value in _BFUZZ_FULL.items():
        monkeypatch.setattr(_bfuzz, name, value)
    assert "lines2 pair differing in scanlines" in _bfuzz.sweep("ntsc", 5)


@pytest.mark.parametrize("host", [0, 1])
def test_bfuzz_streams(host, monkeypatch):
    monkeypatch.setenv("SIMT_HOST_MAPPED", "1")  # (only the interpreter build of the library reads this)
    _bfuzz.check_streams("ntsc", host, n_streams=2, fields=3)


def test_bfuzz_dropin_resize():
    _bfuzz.test_dropin_resize_between_fields("pv1k")


def test_fullsize_property_on_a_small_batch(monkeypatch):
    """tests/test_gpu_fullsize.py with 6 monitors instead of 264 (a field costs ~60 ms per monitor here)"""
    monkeypatch.setattr(_fullsize, "BATCH", 6)
    monkeypatch.setattr(_fullsize, "GROUPS", 3)
    monkeypatch.setattr(_fullsize, "FIELDS", 3)
    _fullsize.test_full_size_batch_is_consistent_and_matches_the_oracle()


# the unmodified CLI driver built for the other systems: one flag set per system here (the GPU test runs three)
test_cli_other_systems = pytest.mark.parametrize("system", ["pv1k", "template", "snes", "vhs"])(
    pytest.mark.parametrize("flags,noise,hue", [("-o", 12, 0)])(_bare(_cli.test_unmodified_cli_driver_other_systems)))

# extreme geometries: half of the GPU test's variants (~12 s each here)
test_edges_extreme_geometries = pytest.mark.parametrize("variant", ["ntsc", "pv1k", "ntsc_bloom"])(_bare(_edges.test_extreme_geometries))

# the C89 video driver: two of the five GPU cases (noise that forces repairs; 32-bit files, odd width) -- each costs ~15 s here
test_vdriver_batch_video_driver = pytest.mark.skipif(not os.path.exists(_vdriver.DRIVER), reason="tools/crtx_video not built")(
    pytest.mark.parametrize("flags,noise,segments,w,bits", [([], 12, 4, 321, 24), ([], 3, 6, 323, 32)])(
        _bare(_vdriver.test_batch_video_driver_writes_the_sequential_loops_images)))


import test_golden as _golden  # noqa: E402


@pytest.mark.parametrize("name", [c["name"] for c in _golden.G.CASES])
def test_golden_vectors_through_the_interpreter(name):
    """the committed digests of the compiled reference (tests/golden/), reproduced by the interpreted kernels"""
    import ctypes as C
    C.CDLL(None).srand(1)  # the VHS drop-in draws from libc rand() like the reference
    _golden.check(name, lambda v, w, h, f: S.ProductEngine(v, w, h, f))


def test_the_interpreter_ran_kernels(simt_libs):
    """Guard against a silent fall-through: the library under test is the interpreter build and it launches."""
    import ctypes as C
    lib = C.CDLL(simt_libs("ntsc"))
    lib.simt_launches.restype = C.c_long
    before = lib.simt_launches()
    e = S.ProductEngine("ntsc", 64, 48)
    e.modulate(S.rand_image(32, 24), format=5, as_color=1)
    e.demodulate(0)
    assert lib.simt_launches() >= before + 4


@pytest.mark.parametrize("variant", sorted(simt_build.variant_defines()))
def test_launch_count_is_the_kernels_launched(simt_libs, variant, monkeypatch):
    """crtx_launch_count counts every kernel a context launches: over modulates of mixed source formats, demodulates of
    every kind of line-pass plan (a row per line and more, rows shared by consecutive lines with and without blend,
    products that wrap) and crtx_frames_host, its delta equals the kernels the interpreter ran.  The drop-in calls
    launch what a one-monitor context counts for the same field, except that on VHS the context also draws its noise
    and aberration on the device (k_vhs_aberration, and k_noise_vhs + k_vhs_commit for the drop-in's k_noise_terms)."""
    import ctypes as C
    import torch
    from ntsc_crt_b200 import layout
    monkeypatch.setenv("SIMT_HOST_MAPPED", "1")  # crtx_frames_host takes its row copies
    lib = C.CDLL(simt_libs(variant))
    lib.simt_launches.restype = C.c_long
    spec = layout.system_spec(variant)
    nes = spec.system == layout.SYS_NES  # (NES sources are palette indices; NES-RGB ones are RGB images)
    lines = spec.lines
    edge = ((1 << 32) - 1) // lines

    def counted(b, call):
        ran, counts = lib.simt_launches(), b.launches
        call()
        return lib.simt_launches() - ran, b.launches - counts

    outw, outh = 640, 200
    # (format, span outh + v_fac, blend): one run of line passes each
    monitors = [(layout.PIX_BGRA, lines, 1), (layout.PIX_RGB, 100, 1), (layout.PIX_ARGB, 100, 0), (layout.PIX_BGRA, edge + 1, 0)]
    fmts = [layout.PIX_BGRA, layout.PIX_RGB, layout.PIX_RGBA, 9]  # (9: not a pixel format, encodes nothing)
    b = capi.Batch(variant, len(monitors))
    outs = [torch.zeros(outh, outw, layout.bpp4fmt(f), dtype=torch.uint8) for f, _, _ in monitors]
    for i, (f, span, blend) in enumerate(monitors):
        b.set_monitor(i, outs[i], fmt=f, noise=3, blend=blend, scanlines=1, v_fac=(span - outh) % (1 << 32))
    b.commit_monitors()
    for it in range(2):
        for i in range(len(monitors)):
            if nes:
                img = torch.from_numpy(S.nes_image(seed=40 + i))
                b.set_source(i, img, dot_crawl_offset=i % 3, reinit=int(it == 0))
            else:
                f = fmts[(i + it) % len(fmts)]
                img = torch.from_numpy(S.rand_image(256, 224, bpp=layout.bpp4fmt(f) or 4, seed=40 + i))
                b.set_source(i, img, format=f, as_color=(i + it) & 1, field=it & 1, frame=0, do_aberration=i & 1)
        ran, counts = counted(b, b.modulate)
        assert ran == counts and ran > 0, ("modulate", it, ran, counts)
        ran, counts = counted(b, b.demodulate)
        assert ran == counts and ran > 0, ("demodulate", it, ran, counts)
    host = [torch.zeros(outh, outw, layout.bpp4fmt(f), dtype=torch.uint8) for f, _, _ in monitors]
    ran, counts = counted(b, lambda: b.frames_host([h.data_ptr() for h in host]))
    assert ran == counts and ran > 0, ("frames_host", ran, counts)
    b.close()

    # the drop-in interface against a one-monitor context, both after one field that uploads the configuration
    img = S.nes_image(seed=50) if nes else S.rand_image(256, 224, seed=50)
    kw = dict(dot_crawl_offset=1) if nes else dict(format=layout.PIX_BGRA, as_color=1, field=0, frame=0)
    e = S.ProductEngine(variant, 320, 240)
    e.set(blend=1, scanlines=1)
    one = capi.Batch(variant, 1)
    one.set_monitor(0, torch.zeros(240, 320, 4, dtype=torch.uint8), noise=3, blend=1, scanlines=1)
    one.commit_monitors()
    one.set_source(0, torch.from_numpy(img), **kw)
    pair = []
    for _ in range(2):
        ran = lib.simt_launches()
        e.modulate(img, **kw)
        e.demodulate(3)
        dropin = lib.simt_launches() - ran
        ran, counts = counted(one, lambda: (one.modulate(), one.demodulate()))
        assert ran == counts
        pair.append((dropin, counts))
    assert pair[1][0] + (2 if spec.system == layout.SYS_VHS else 0) == pair[1][1], pair
    one.close()


@pytest.mark.skipif(os.environ.get("SIMT_SCHEDULE") is not None, reason="already running under an alternative schedule")
@pytest.mark.parametrize("schedule", ["random:7"])
def test_other_thread_schedules(schedule):
    """Any order in which the runnable threads of a block are resumed is a legal interleaving.  The kernels newest to
    the tree (and a few of the long-standing ones) must give the same bits when the interpreter resumes them in
    reverse or in a freshly shuffled order every round -- an accidental "lower threads ran first" dependence, which a
    GPU would expose as a race, fails here."""
    import subprocess
    env = dict(os.environ, SIMT_SCHEDULE=schedule)
    sel = ("(parity_batch_matches_the_oracle and not snes and not conv and not vhs) or wire_ppm or wire_fade or fullsize"
           " or vfac_batch or vhs_batch_many_generator_states or (bfuzz_random_batches and ntsc_seed1)")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-k", sel, "-p", "no:cacheprovider"],
                       env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, cwd=S.ROOT)
    assert r.returncode == 0, r.stdout[-3000:]


@pytest.mark.parametrize("variant", ["ntsc", "pv1k"])
def test_bench_product_arm_dry_run(variant):
    """bench.py's product arm, every line of it, against the current libraries (tests/simt/bench_dry_run.py): the JSON
    line must carry the contract's keys and count the launches of the timed steps"""
    import json
    import subprocess
    r = subprocess.run([sys.executable, os.path.join(S.ROOT, "tests", "simt", "bench_dry_run.py"), "--variant", variant, "--batch", "4",
                        "--steps", "2", "--warmup", "1", "--e2e-batch", "8", "--no-cpu-baseline", "--config4-frames", "8",
                        "--config4-segments", "2", "--sustained-seconds", "0.001"],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, cwd=S.ROOT, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
                "dtype", "data", "config", "e2e", "gpu_launches", "roofline", "clocks"):
        assert key in line, key
    assert line["steps"] == 2 and line["warmup"] >= 3 and line["gpu_launches"] >= 2 * 4
    assert line["e2e"]["h2d_bytes_per_step"] > 0 and line["e2e"]["d2h_bytes_per_step"] > 0
    assert set(("bound", "achieved", "peak", "unit", "frac", "traffic")) <= set(line["roofline"])
    assert line["dropin"]["value"] > 0 and line["dropin"]["pairs"] >= 8, line["dropin"]
    assert line["sustained"]["steps"] >= 2 and "demodulate" in line["roofline"] and line["roofline"]["demodulate"]["frac"] > 0
    assert line["config"]["workload"] == __import__("bench").workload_name() or variant != "ntsc"
    if variant == "ntsc":  # BASELINE configs[3] in miniature: bit-identical to the sequential loop
        assert line["config4"]["bit_identical_to_sequential_loop"] is True and line["config4"]["frames_checked"] == 8


def test_interpreter_selftest(tmp_path):
    """tests/simt/selftest.cpp: the interpreter against known answers from the documented semantics of what it stands
    in for (shuffles with widths, ballots, block barriers with a predicate, the SIMD video intrinsics, byte
    permutes, three phases on one mbarrier with deferred bulk copies)"""
    import subprocess
    here = os.path.join(S.ROOT, "tests", "simt")
    exe = str(tmp_path / "selftest")
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-fwrapv", "-fno-strict-aliasing", "-Wno-unknown-pragmas", "-Wno-attributes",
           "-fsanitize=alignment", "-fsanitize-undefined-trap-on-error", "-I" + here, "-I" + os.path.join(S.ROOT, "include"),
           "-DCRT_SYSTEM=0", os.path.join(here, "selftest.cpp"), os.path.join(here, "simt_runtime.cpp"), "-o", exe]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0 and "selftest ok" in r.stdout, r.stdout[-2000:]


def test_packed_byte_helpers(tmp_path):
    """tests/simt/helpers_check.cpp: clamp127_4 / abs127_4 / max127_4 (crt_sync.cuh: max(b, -127), |b| and the larger of two
    values on four packed bytes with plain integer instructions) against their byte-wise definitions, exhaustively per pair
    of bytes and positions.  Picture content never produces the -128 that clamp127_4 exists for, and a too small maximum
    would only show on a monitor at the edge of the fast equaliser's range: both get their own check here."""
    import subprocess
    from simt import build as B  # noqa: F401  (the prepared copy of the product sources: tests/simt/_build/src)
    here = os.path.join(S.ROOT, "tests", "simt")
    src = os.path.join(here, "_build", "src")
    B.prepare(src)
    exe = str(tmp_path / "helpers_check")
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-fwrapv", "-fno-strict-aliasing", "-Wno-unknown-pragmas", "-Wno-attributes",
           "-I" + src, "-I" + os.path.join(S.ROOT, "include"), "-DCRT_SYSTEM=0",
           os.path.join(here, "helpers_check.cpp"), os.path.join(src, "simt_runtime.cpp"), "-o", exe]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0 and "helpers ok" in r.stdout, r.stdout[-2000:]
