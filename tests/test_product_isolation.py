"""The oracle is test infrastructure: nothing under ntsc-crt_b200/ (Python or CUDA sources), tools/ or include/ may
import, include, link or load anything from oracle/ or tests/, and the built libraries must not depend on the
oracle library."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRODUCT_DIRS = ["ntsc-crt_b200", "tools", "include"]
FORBIDDEN = re.compile(r"(crt_oracle|libcrt_oracle|oracle/|oracle\\|import support|from support|mock_crtx|mock_batch|_ref/libref|simt|libcrt_simt)")


def product_sources():
    for d in PRODUCT_DIRS:
        for base, _, files in os.walk(os.path.join(ROOT, d)):
            if "__pycache__" in base or os.sep + "lib" in base or os.sep + "bin" in base:
                continue
            for f in files:
                if f.endswith((".py", ".cu", ".cuh", ".h", ".c", "Makefile")):
                    yield os.path.join(base, f)


def test_product_sources_do_not_reference_the_oracle():
    bad = []
    for path in product_sources():
        for no, line in enumerate(open(path, errors="replace"), 1):
            code = line.split("//")[0] if path.endswith((".cu", ".cuh", ".h", ".c")) else line.split("#")[0]
            # documentation may NAME the test files; code lines must not pull them in
            if FORBIDDEN.search(code) and re.search(r"(#include|import |dlopen|CDLL|-l|\.so)", code):
                bad.append("%s:%d: %s" % (os.path.relpath(path, ROOT), no, line.strip()))
    assert not bad, "\n".join(bad)


def test_built_libraries_do_not_link_the_oracle():
    libdir = os.path.join(ROOT, "ntsc-crt_b200", "lib")
    libs = [f for f in os.listdir(libdir) if f.endswith(".so")] if os.path.isdir(libdir) else []
    if not libs:
        pytest.skip("libraries not built")
    for f in libs:
        out = subprocess.run(["readelf", "-d", os.path.join(libdir, f)], stdout=subprocess.PIPE).stdout.decode()
        needed = re.findall(r"NEEDED.*\[(.*?)\]", out)
        assert not any("oracle" in n or "libref" in n or "simt" in n for n in needed), (f, needed)


def test_the_simt_interpreter_stays_out_of_the_product():
    """tests/simt/ (the CPU interpreter that runs the kernel sources for debugging) is test infrastructure like the
    oracle: no product loader knows its libraries, and the product libraries are real sm_90a CUDA binaries."""
    from ntsc_crt_b200 import capi
    for v in capi.VARIANTS:
        assert "simt" not in capi.lib_path(v) and os.sep + "tests" + os.sep not in capi.lib_path(v)
    libdir = os.path.join(ROOT, "ntsc-crt_b200", "lib")
    libs = [f for f in os.listdir(libdir) if f.endswith(".so")] if os.path.isdir(libdir) else []
    if not libs:
        pytest.skip("libraries not built")
    for f in libs:
        out = subprocess.run(["readelf", "-d", os.path.join(libdir, f)], stdout=subprocess.PIPE).stdout.decode()
        assert "libcudart" in out or "cudart" in subprocess.run(["strings", "-n", "8", os.path.join(libdir, f)], stdout=subprocess.PIPE).stdout.decode(), f
        syms = subprocess.run(["nm", "-D", "--defined-only", os.path.join(libdir, f)], stdout=subprocess.PIPE).stdout.decode()
        assert "simt_launches" not in syms, f
