"""TEST INFRASTRUCTURE: spot-check of the NES border colour on chroma pattern 1 (csrc/Makefile `custom`:
NAME=nes_p1_border DEFS="-DCRT_SYSTEM=1 -DCRT_CHROMA_PATTERN=1 -DNES_BORDER=1"), which is not in the test suite.

The kernel sources are built for the SIMT interpreter with those defines, the REFERENCE is built from a scratch copy with
NES_BORDER 1 and CRT_CHROMA_PATTERN 1 (unguarded #defines there, crt_nes.c:69, crt_nes.h:30), and both are driven
through the drop-in interface with the border colour, dot crawl and picture offsets changing between fields: every state
array must be identical.  Needs the reference sources.      python tests/simt/check_nes_border.py [reference dir]
"""
import dataclasses
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.chdir(ROOT)
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tests", "simt"))
import build as B  # noqa: E402
import support as S  # noqa: E402
from ntsc_crt_b200 import layout  # noqa: E402

REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
NAME, DEFS = "nes_p1_border", ["-DCRT_SYSTEM=1", "-DCRT_CHROMA_PATTERN=1", "-DNES_BORDER=1"]

srcdir = os.path.join(B.OUT, "src")
B.prepare(srcdir)
lib = os.path.join(B.OUT, "combo_libcrt_simt_%s.so" % NAME)
subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-fwrapv", "-fno-strict-aliasing", "-Wno-unknown-pragmas",
                "-Wno-attributes", "-I" + srcdir, "-I" + os.path.join(ROOT, "include")] + DEFS + ["-o", lib]
               + [os.path.join(srcdir, f) for f in ("crtx.cpp", "crt_dropin.cpp", "simt_runtime.cpp")], check=True)
T = tempfile.mkdtemp()
try:
    for f in ("crt_core.c", "crt_core.h", "crt_nes.c", "crt_nes.h"):
        shutil.copy(os.path.join(REF, f), T)
    for f, a, b in (("crt_nes.c", "#define NES_BORDER    0", "#define NES_BORDER    1"),
                    ("crt_nes.h", "#define CRT_CHROMA_PATTERN 2", "#define CRT_CHROMA_PATTERN 1")):
        txt = open(os.path.join(T, f)).read()
        assert a in txt, (f, a)
        open(os.path.join(T, f), "w").write(txt.replace(a, b, 1))
    reflib = os.path.join(B.OUT, "combo_libref_%s.so" % NAME)
    subprocess.run(["gcc", "-O3", "-fPIC", "-w", "-shared", "-DCRT_SYSTEM=1", "-I" + T, "-o", reflib,
                    os.path.join(T, "crt_core.c"), os.path.join(T, "crt_nes.c"), "oracle/ref_shim.c"], check=True)
finally:
    shutil.rmtree(T)

layout.SPECS[NAME] = dataclasses.replace(layout.SPECS["nes_p1"], name=NAME, border=True)
ok = True
for outw, outh in [(640, 480), (333, 250)]:
    img = S.nes_image(seed=3)
    gpu, ref = S.CEngine(lib, NAME, outw, outh), S.CEngine(reflib, NAME, outw, outh)
    for e in (gpu, ref):
        e.set(blend=1, scanlines=1, black_point=2, white_point=95)
        for it in range(5):
            e.modulate(img, dot_crawl_offset=it % 3, hue=20 * it, border_color=0x22 + 0x61 * it, xoffset=7 * it, yoffset=2 * it,
                       **(dict(field_initialized=0) if it == 3 else {}))
            e.demodulate(5 * it)
    try:
        S.assert_same_state(gpu.state(), ref.state(), NAME)
    except AssertionError as ex:
        ok = False
        print(NAME, "MISMATCH", str(ex)[:200])
print(NAME, "identical to the reference built the same way" if ok else "FAILED")
sys.exit(0 if ok else 1)
