"""tools/crtx_video.c without a GPU: the driver is linked against tests/mock_crtx.c -- the crtx_* entry points it
uses, implemented with the oracle on the CPU -- so its host logic (segments, halo, speculated sync state,
verification of every seam, repair of a failed segment, BMP reading and writing) is exercised in the CPU suite,
including the repair path that well-behaved inputs never reach.  The GPU suite runs the same program against
the real library (tests/test_gpu_video_driver.py)."""
import os
import subprocess

import numpy as np
import pytest

import support as S
from ntsc_crt_b200 import layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    d = tmp_path_factory.mktemp("mock_driver")
    lib = d / "libcrt_b200_ntsc.so"
    exe = d / "crtx_video"
    inc = ["-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "oracle")]
    subprocess.run(["gcc", "-O2", "-fPIC", "-fwrapv", "-shared", "-o", str(lib), os.path.join(ROOT, "tests", "mock_crtx.c"),
                    os.path.join(ROOT, "oracle", "crt_oracle.c")] + inc, check=True)
    subprocess.run(["gcc", "-std=c89", "-pedantic", "-O2", "-pthread", "-o", str(exe), os.path.join(ROOT, "tools", "crtx_video.c"),
                    "-I" + os.path.join(ROOT, "include"), "-L" + str(d), "-lcrt_b200_ntsc", "-Wl,-rpath," + str(d)], check=True)
    return str(exe)


def frames_for(n, w, h, wild):
    rng = np.random.default_rng(5)
    base = S.bars_image(w, h)
    out = []
    for k in range(n):
        f = np.roll(base, 5 * k, axis=1).copy()
        if wild and k % 5 == 3:
            f[..., :3] = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)  # a scene cut to noise
        f[..., 3] = 255
        out.append(f)
    return out


@pytest.mark.parametrize("flags,noise,segments,n,wild", [
    ([], 0, 4, 14, False),
    ([], 3, 2, 23, False),           # many steps: the reader / writer threads cycle through both buffer sets
    (["-m"], 9, 14, 14, False),      # one image per segment: every seam is a halo seam
    (["-a"], 255, 5, 16, True),      # noise far beyond what the speculated sync state survives
    (["-p"], 200, 3, 10, True),
])
def test_driver_logic_against_the_sequential_loop(tmp_path, driver, flags, noise, segments, n, wild):
    w, h, outw, outh = 160, 240, 320, 240
    frames = frames_for(n, w, h, wild)
    os.mkdir(tmp_path / "frames")
    os.mkdir(tmp_path / "output")
    for k in range(n):
        S.write_bmp(str(tmp_path / "frames" / ("%06d.bmp" % (k + 1))), frames[k], 24)
    res = subprocess.run([driver] + flags + ["-S", str(segments), str(n + 1), str(outw), str(outh), str(noise)],
                         cwd=str(tmp_path), stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=600)
    assert res.returncode == 0, res.stderr.decode()
    ora = S.OracleEngine("ntsc", outw, outh)
    ora.set(blend=0, scanlines=0 if "-a" in flags else 1, saturation=10)
    for k in range(n):
        field, frame = (0, 0) if "-p" in flags else (k & 1, (k >> 1) & 1)
        ora.modulate(frames[k], format=layout.PIX_BGRA, as_color=0 if "-m" in flags else 1, field=field, frame=frame)
        ora.demodulate(noise)
        got = S.read_bmp32(str(tmp_path / "output" / ("%06d.bmp" % (k + 1))))
        assert np.array_equal(got, ora.out), "image %d: %s\n%s" % (k + 1, S.diff_report("image", got, ora.out),
                                                                   res.stdout.decode()[-200:])
    tail = res.stdout.decode().strip().splitlines()[-1]
    assert "done:" in tail
    if noise == 0:
        assert " 0 redone" in tail
    if noise >= 200:  # the point of these cases: the speculation fails and the repair path must produce the images
        assert " 0 redone" not in tail, tail
