"""At noise 0 k_sync does not write inp[] of the monitors k_lines2 decodes: k_lines2 reads its windows from analog[]
(clamped to -127), and inp[] is made from analog[] when it is handed out.  Every state the batch interface hands out --
analog[], inp[] (crtx_read_signal right after the demodulate), the image, the sync state -- must stay the CPU model's."""
import numpy as np
import pytest

import support as S
from ntsc_crt_b200 import layout

pytestmark = pytest.mark.gpu

BGRA, RGB = layout.PIX_BGRA, layout.PIX_RGB


def _fields(rig, n, fields, seed=0):
    imgs = [S.rand_image(320, 240, seed=seed + i) for i in range(n)]
    for f in range(fields):
        for i in range(n):
            rig.source(i, imgs[i], format=BGRA, as_color=1, field=f & 1, frame=(f >> 1) & 1)
        rig.modulate()
        before = rig.b.lines2_launches
        rig.demodulate()
        assert rig.b.lines2_launches > before, "k_lines2 did not run: the case does not reach the path under test"
        yield f


def _check(rig, what):
    """analog, inp (crtx_read_signal right after the demodulate), out and the sync state of every monitor"""
    for i, o in enumerate(rig.oras):
        S.assert_same_state(S.monitor_state(rig.b, i, rig.outs[i]), o.state(), "%s, monitor %d %r" % (what, i, rig.mons[i]))


def test_whole_batch_at_noise_0():
    n = 264
    rig = S.BatchRig("ntsc", [dict(outw=640, outh=480, fmt=BGRA, noise=0, knobs=dict(blend=1, scanlines=1)) for _ in range(n)])
    try:
        for f in _fields(rig, n, 3):
            for i in (0, 1, 131, 262, 263):  # (the oracle's whole state is checked on a sample of the batch)
                o = rig.oras[i]
                S.assert_same_state(S.monitor_state(rig.b, i, rig.outs[i]), o.state(), "field %d, monitor %d" % (f, i))
    finally:
        rig.close()


def test_mixed_batch():
    """noise 0 beside noise > 0, a monitor on the wrap-exact equaliser (brightness 5000), an odd count (the last k_lines2
    CTA has one monitor) and a 3-byte run (k_lines, which reads inp[] written by k_sync)"""
    mons = []
    for i in range(7):
        knobs = dict(blend=1, scanlines=i & 1)
        if i == 2:
            knobs["brightness"] = 5000
        mons.append(dict(outw=640, outh=480, fmt=BGRA, noise=(0 if i % 3 != 1 else 9), knobs=knobs))
    mons += [dict(outw=640, outh=480, fmt=RGB, noise=0, knobs=dict(blend=1, scanlines=1)) for _ in range(2)]
    mons.append(dict(outw=640, outh=480, fmt=BGRA, noise=0, knobs=dict(blend=0, scanlines=0)))
    rig = S.BatchRig("ntsc", mons)
    try:
        for i in (0, 4):  # a raw pointer to inp[] handed out: k_sync writes it on every demodulate from then on
            assert rig.b.inp_ptr(i)
        for f in _fields(rig, len(mons), 4, seed=20):
            _check(rig, "mixed batch, field %d" % f)
    finally:
        rig.close()


def test_poked_minus_128():
    """analog[] holding -128 (possible only by writing the signal): inp[] and the decode take it as -127"""
    rig = S.BatchRig("ntsc", [dict(outw=640, outh=480, fmt=BGRA, noise=0, knobs=dict(blend=1, scanlines=1)) for _ in range(2)])
    try:
        for f in _fields(rig, 2, 1, seed=40):
            _check(rig, "field %d" % f)
        rng = np.random.default_rng(3)
        for i in range(2):
            sig = rig.b.signal(i, "analog").copy()
            at = rng.choice(sig.size, size=sig.size // 50, replace=False)
            sig[at] = -128
            sig[-1] = -128
            rig.b.write_signal(i, sig, "analog")
            np.ctypeslib.as_array(rig.oras[i].mon.analog, shape=(sig.size,))[:] = sig
        before = rig.b.lines2_launches
        rig.demodulate()
        assert rig.b.lines2_launches > before
        _check(rig, "poked -128")
        for i in range(2):
            assert (rig.b.signal(i, "inp") >= -127).all()
    finally:
        rig.close()


def test_inp_after_a_later_modulate():
    """inp[] left unwritten is made from analog[]: once a modulate has rewritten analog[] it is gone, and reading it is an
    error that says so rather than a wrong signal, also after its pointer is taken then; a monitor whose inp[] pointer was
    taken before keeps it"""
    from ntsc_crt_b200 import capi
    rig = S.BatchRig("ntsc", [dict(outw=640, outh=480, fmt=BGRA, noise=0, knobs=dict(blend=1, scanlines=1)) for _ in range(2)])
    try:
        assert rig.b.inp_ptr(1)
        for f in _fields(rig, 2, 2, seed=60):
            _check(rig, "field %d" % f)
        rig.modulate()
        rig.demodulate()  # (inp[] not read before the next modulate)
        want = [o.state()["inp"].copy() for o in rig.oras]
        rig.modulate()
        with pytest.raises(capi.CrtxError, match="monitor 0: inp"):
            rig.b.signal(0, "inp")
        assert np.array_equal(rig.b.signal(1, "inp"), want[1])
        assert rig.b.inp_ptr(0)  # (pinned from now on, but what it points at is still gone)
        with pytest.raises(capi.CrtxError, match="monitor 0: inp"):
            rig.b.signal(0, "inp")
        rig.demodulate()
        _check(rig, "after the next demodulate")
    finally:
        rig.close()
