"""The knob-domain table of tests/knob_domain.py through the CUDA library: the picture knobs, the noise and the source
settings on the edges of their arithmetic, drop-in and batch interface, against the oracle and, where oracle/_ref is
built, the compiled reference.  tests/test_oracle_knob_domain.py pins the oracle to the reference on the same cases.

The batch runs one edge per monitor, so one launch mixes wrapped, clamped and stock monitors: with k_lines2 on and off,
with every monitor forced onto the wrap-exact equaliser (generic_eq) and with the staged encoder off (mod_staged 0).
Each run asserts the paths it expects (crtx_get_paths, the k_lines2 launches), so no case passes on the other kernel.
The noise edges put the LCG systems' fused noise of k_sync (noise_word, noisy_apply) above 255 and below 0."""
import numpy as np
import pytest

import knob_domain as K
import support as S
from ntsc_crt_b200 import layout
from support import run_all, trio
from test_gpu_vhs import libc_srand

pytestmark = pytest.mark.gpu

GEN, STAGED = 1, 2  # Batch.PATH_GENERIC_EQ, Batch.PATH_STAGED_MOD
# the variants of each encoder and decoder family; tests/test_oracle_knob_domain.py covers every variant on the oracle
VARIANTS = ["ntsc", "ntsc_conv", "vhs", "nes", "nes_p0", "snes", "nesrgb", "template", "pv1k", "ntsc_bloom", "nes_border",
            "ntsc_nosync", "nes_nosync"]
BATCH_VARIANTS = ["ntsc", "nes", "pv1k", "ntsc_conv", "vhs"]
LINES2_VARIANTS = ("ntsc", "nes", "vhs")  # (k_lines2 takes 4 samples per carrier cycle and the stock equaliser)
CASES = None  # all of a variant's cases; a number: every so many-th of them (the interpreter's runs)


def table(variant):
    cases = K.cases(variant)
    return cases if CASES is None else cases[::CASES]


def batch_settings(variant, src, it):
    """a field's source settings in the batch: the NES systems' first field writes the sync skeleton, as the drop-in's
    first call does (reinit)"""
    kw = K.modulate_settings(src, it)
    if layout.system_spec(variant).system in (layout.SYS_NES, layout.SYS_NESRGB):
        kw["reinit"] = int(it == 0)
    return kw


@pytest.mark.parametrize("variant", VARIANTS)
def test_dropin_knob_domain(variant):
    """every case through the reference's own interface, compared after every call; the caller's settings hold
    field & 1 and frame & 1 afterwards"""
    imgs = K.images(variant)
    for name, mon, src, noise in table(variant):
        what = "%s %s (monitor %r, source %r, noise %d)" % (variant, name, mon, src, noise)
        gpu, ora, ref = trio(variant, K.OUTW, K.OUTH, K.FMT)
        if variant == "vhs":  # the drop-in draws from the host's rand(), which the live reference would share
            ref = None
            libc_srand(1)  # (the oracle's replica is seeded with 1)
        run_all((gpu, ora, ref), lambda e: e.set(blend=1, scanlines=1, **mon))
        for it, img in enumerate(imgs):
            kw = K.modulate_settings(src, it)
            run_all((gpu, ora, ref), lambda e: e.modulate(img, **kw))
            S.check(gpu, ora, ref, "%s field %d modulate" % (what, it))
            if "field" in kw:
                assert (gpu.settings.field, gpu.settings.frame) == (kw["field"] & 1, kw["frame"] & 1), what
            run_all((gpu, ora, ref), lambda e: e.demodulate(noise))
            S.check(gpu, ora, ref, "%s field %d demodulate" % (what, it))


def _bright_limit(variant):
    """|bright| the fast equaliser admits (tests/test_gpu_guard_edges.py)"""
    return 2048 if layout.system_spec(variant).system == layout.SYS_PV1K else 4096


def _batch(variant, options, outw=640, outh=480):
    cases = table(variant)
    knobs = dict(K.STOCK_MONITOR, blend=1, scanlines=1)
    mons = [dict(outw=outw, outh=outh, fmt=K.FMT, noise=noise, knobs=dict(knobs, **mon)) for _, mon, _, noise in cases]
    if variant == "vhs":
        for i, m in enumerate(mons):
            m["seed"] = 1 + i
    return S.BatchRig(variant, mons, options=options), cases


@pytest.mark.parametrize("lines2,generic,staged", [(1, 0, 1), (0, 0, 1), (1, 1, 1), (1, 0, 0)],
                         ids=["lines2", "no_lines2", "generic_eq", "no_mod_staged"])
@pytest.mark.parametrize("variant", BATCH_VARIANTS)
def test_batch_knob_domain(variant, lines2, generic, staged):
    """one monitor per case in one batch, three fields, every monitor's state against its CPU model after every call"""
    rig, cases = _batch(variant, [("lines2", lines2), ("generic_eq", generic), ("mod_staged", staged)])
    imgs = K.images(variant)
    rgb = layout.system_spec(variant).system not in (layout.SYS_NES, layout.SYS_NESRGB)
    try:
        for it, img in enumerate(imgs):
            for i, (_, _, src, _) in enumerate(cases):
                rig.source(i, img, **batch_settings(variant, src, it))
            rig.modulate()
            rig.check("%s %s field %d modulate" % (variant, dict(lines2=lines2, generic=generic, staged=staged), it))
            before = rig.b.lines2_launches
            rig.demodulate()
            rig.check("%s field %d demodulate" % (variant, it))
            paths = list(rig.b.paths())
            assert (rig.b.lines2_launches > before) == bool(lines2 and variant in LINES2_VARIANTS), (
                variant, lines2, rig.b.lines2_launches - before)
            for i, (name, mon, src, noise) in enumerate(cases):
                what = "%s field %d %s: paths %d" % (variant, it, name, paths[i])
                if rgb:
                    assert bool(paths[i] & STAGED) == bool(staged), what
                bright = K.wrap32(mon.get("brightness", 0) - (layout.system_spec(variant).black + mon.get("black_point", 0)))
                if generic or abs(bright) > _bright_limit(variant):
                    assert paths[i] & GEN, what
    finally:
        rig.close()


def test_frames_host_knob_edges(monkeypatch):
    """crtx_frames_host on a batch of a stock monitor, a wrapped white scale, a wrapped brightness and a noise past a
    byte: the host images equal the CPU models'"""
    import torch
    monkeypatch.setenv("SIMT_HOST_MAPPED", "1")  # (only the CPU interpreter build of the library reads this)
    variant = "ntsc"
    knobs = [dict(), dict(white_point=21474837), dict(brightness=K.INT_MIN), dict(saturation=1 << 30)]
    noises = [K.STOCK_NOISE, K.STOCK_NOISE, K.STOCK_NOISE, 1 << 16]
    mons = [dict(outw=K.OUTW, outh=K.OUTH, fmt=K.FMT, noise=z, knobs=dict(K.STOCK_MONITOR, blend=1, scanlines=1, **k))
            for k, z in zip(knobs, noises)]
    rig = S.BatchRig(variant, mons)
    host = [torch.zeros((K.OUTH, K.OUTW, 4), dtype=torch.uint8).pin_memory() for _ in mons]
    src = K.stock_source(variant, K.SRC_W, K.SRC_H)
    try:
        for it, img in enumerate(K.images(variant)):
            for i in range(len(mons)):
                rig.source(i, img, **batch_settings(variant, src, it))
            rig.frames_host([h.data_ptr() for h in host])
            torch.cuda.synchronize()
            for i, o in enumerate(rig.oras):
                got = host[i].numpy()
                assert np.array_equal(got, o.out), "field %d monitor %r: %s" % (it, knobs[i], S.diff_report("host", got, o.out))
            rig.check("frames_host field %d" % it)
    finally:
        rig.close()
