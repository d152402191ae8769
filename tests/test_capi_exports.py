"""CPU-side checks of the boundary: every symbol include/*.h declares is exported by every
library variant, every library reports the build its variant names, struct layouts equal the reference's, and the
host-only entry points (crt_bpp4fmt, crt_sincos14) agree with the oracle.  No compute calls: there is no GPU here."""
import ctypes as C
import os
import re

import pytest

import support as S
from ntsc_crt_b200 import capi, layout

ROOT = S.ROOT


def declared(header):
    text = open(os.path.join(ROOT, "include", header)).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(crtx?_[a-z0-9_]+)\s*\(", text)))


@pytest.mark.parametrize("variant", capi.ALL_VARIANTS)
def test_every_declared_symbol_is_exported(variant):
    if not os.path.exists(capi.lib_path(variant)):
        pytest.fail("library not built: run __graft_entry__.build()")
    lib = C.CDLL(capi.lib_path(variant))
    names = declared("crt_b200.h") + declared("crtx_batch.h")
    assert set(capi.CRT_EXPORTS) <= set(names) and set(capi.CRTX_EXPORTS) <= set(names)
    for name in names:
        assert hasattr(lib, name), "%s missing from %s" % (name, variant)


def test_variant_groups_are_disjoint():
    """the stock builds, the border builds and the sync-switch builds are three separate groups, ALL_VARIANTS all three,
    and each variant's spec puts it in its group"""
    assert capi.ALL_VARIANTS == capi.VARIANTS + capi.BORDER_VARIANTS + capi.SYNC_VARIANTS
    assert len(set(capi.ALL_VARIANTS)) == len(capi.ALL_VARIANTS)
    for variant in capi.ALL_VARIANTS:
        spec = layout.system_spec(variant)
        group = (capi.BORDER_VARIANTS if spec.border else capi.VARIANTS if spec.do_vsync and spec.do_hsync
                 else capi.SYNC_VARIANTS)
        assert variant in group, variant


@pytest.mark.parametrize("variant", capi.ALL_VARIANTS)
def test_geometry_and_host_only_entry_points(variant):
    """the library reports its system, timing, border switch and sync switches as its variant's spec has them (every
    stock library: no border, both sync searches on)"""
    lib = capi.load(variant)
    spec = layout.system_spec(variant)
    assert (lib.crtx_system(), lib.crtx_chroma_pattern(), lib.crtx_hres(), lib.crtx_input_size(),
            lib.crtx_lines(), lib.crtx_cc_vper(), lib.crtx_nes_border(), lib.crtx_do_vsync(), lib.crtx_do_hsync()) == (
        spec.system, spec.pattern, spec.hres, spec.input_size, spec.lines, spec.vper, int(spec.border),
        int(spec.do_vsync), int(spec.do_hsync))
    ora = S.oracle_lib()
    s1, c1, s2, c2 = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    for n in range(-17000, 34000, 13):
        lib.crt_sincos14(C.byref(s1), C.byref(c1), n)
        ora.ocrt_sincos14(C.byref(s2), C.byref(c2), n)
        assert (s1.value, c1.value) == (s2.value, c2.value)
    for f in range(-1, 8):
        assert lib.crt_bpp4fmt(f) == ora.ocrt_bpp(f)


def test_header_compiles_as_c89_and_matches_reference_layout(tmp_path):
    """include/crt_b200.h is C89 and lays struct CRT / NTSC_SETTINGS out like the reference."""
    src = tmp_path / "probe.c"
    src.write_text('#include <stdio.h>\n#include "crt_b200.h"\n'
                   'int main(void){printf("%d %d %d %d %d\\n",(int)sizeof(struct CRT),'
                   '(int)sizeof(struct NTSC_SETTINGS),CRT_HRES,AV_LEN,CRT_CC_VPER);return 0;}\n')
    import subprocess
    for variant, defs in (("ntsc", ["-DCRT_SYSTEM=0"]), ("vhs", ["-DCRT_SYSTEM=5"]),
                          ("nes", ["-DCRT_SYSTEM=1"]), ("nes_p0", ["-DCRT_SYSTEM=1", "-DCRT_CHROMA_PATTERN=0"])):
        exe = tmp_path / ("probe_" + variant)
        subprocess.check_call(["gcc", "-std=c89", "-pedantic", "-Wall", "-Werror", "-I",
                               os.path.join(ROOT, "include")] + defs + [str(src), "-o", str(exe)])
        got = subprocess.check_output([str(exe)]).split()
        spec = layout.system_spec(variant)
        assert [int(x) for x in got] == [C.sizeof(layout.crt_struct(spec)),
                                         C.sizeof(layout.settings_struct(spec)), spec.hres,
                                         spec.av_len, spec.vper], variant
