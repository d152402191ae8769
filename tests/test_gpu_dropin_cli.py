"""The reference's own, UNMODIFIED command-line driver (crt_main.c) linked against the CUDA library
instead of crt_core.c + crt_ntsc.c (oracle/Makefile target cli_b200_ntsc; include/compat/crt_core.h
stands in for the reference header) must write byte-identical files to the all-reference build.
The binaries are built where /root/reference is mounted and travel under oracle/_ref."""
import os
import subprocess

import numpy as np
import pytest

import support as S

pytestmark = pytest.mark.gpu

REF_CLI = os.path.join(S.REF_DIR, "cli_ref_ntsc")
B200_CLI = os.path.join(S.REF_DIR, "cli_b200_ntsc")


@pytest.mark.skipif(not (os.path.exists(REF_CLI) and os.path.exists(B200_CLI)), reason="driver binaries not built")
@pytest.mark.parametrize("flags,noise,hue", [("-op", 0, 0), ("-o", 12, 0), ("-om", 24, 30), ("-opr", 0, 90), ("-opa", 0, 0)])
def test_unmodified_cli_driver_is_byte_identical(tmp_path, flags, noise, hue):
    rgb = S.bars_image(320, 240, fmt=S.layout.PIX_RGB)[..., :3].copy()
    src = tmp_path / "in.ppm"
    S.write_ppm(str(src), rgb)
    outs = []
    for exe, name in ((REF_CLI, "ref.ppm"), (B200_CLI, "b200.ppm")):
        out = tmp_path / name
        subprocess.run([exe, flags, "832", "624", str(noise), str(hue), str(src), str(out)],
                       check=True, stdout=subprocess.DEVNULL, timeout=120)
        outs.append(open(out, "rb").read())
    assert len(outs[0]) > 1000
    assert outs[0] == outs[1]


@pytest.mark.parametrize("system", ["pv1k", "template", "snes", "vhs"])
@pytest.mark.parametrize("flags,noise,hue", [("-o", 12, 0), ("-opm", 0, 45), ("-opa", 0, 0)])
def test_unmodified_cli_driver_other_systems(tmp_path, system, flags, noise, hue):
    """crt_main.c also builds for the other RGB systems (CRT_SYSTEM 2, 3, 4, 5; it has no NES / NES-RGB build): the same
    source linked against libcrt_b200_<system>.so through include/compat/crt_core.h writes the all-reference build's
    bytes.  (VHS draws its noise from libc rand(), never seeded by the driver: same stream in both builds.)"""
    ref_cli, b200_cli = (os.path.join(S.REF_DIR, "cli_%s_%s" % (k, system)) for k in ("ref", "b200"))
    if not (os.path.exists(ref_cli) and os.path.exists(b200_cli)):
        pytest.skip("driver binaries not built")
    rgb = S.bars_image(320, 240, fmt=S.layout.PIX_RGB)[..., :3].copy()
    src = tmp_path / "in.ppm"
    S.write_ppm(str(src), rgb)
    outs = []
    for exe, name in ((ref_cli, "ref.ppm"), (b200_cli, "b200.ppm")):
        out = tmp_path / name
        subprocess.run([exe, flags, "640", "480", str(noise), str(hue), str(src), str(out)],
                       check=True, stdout=subprocess.DEVNULL, timeout=300)
        outs.append(open(out, "rb").read())
    assert len(outs[0]) > 1000
    assert outs[0] == outs[1]
