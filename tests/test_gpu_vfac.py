"""v_fac, the vertical stretch of struct CRT (crt_core.h:86), through the CUDA library: drop-in and batch interface
against the oracle and the compiled reference.

v_fac decides which output rows every decoded line owns (crt_core.c:428-432), which is exactly what the line kernels
spread over threads.  The reference computes outh + v_fac and the products in 32-bit unsigned arithmetic, so a
"negative" v_fac makes lines share rows (applied in order: blended or overwritten), and a span whose products wrap
makes lines far apart write the same rows.  The edge cases are those of tests/test_oracle_vfac.py, where the oracle is
pinned to the reference on them."""
import numpy as np
import pytest

import support as S
import test_oracle_vfac as V
from ntsc_crt_b200 import layout
from test_gpu_lineshard import decode_one_image_in_blocks
from test_gpu_parity import check, run_all, trio

pytestmark = pytest.mark.gpu

M32 = 1 << 32
EDGE = (M32 - 1) // 240  # the largest span at which no product wraps (every library here decodes 240 lines)


def vfac_of_span(span, outh):
    return (span - outh) % M32


@pytest.mark.parametrize("variant,outw,outh,fmt", [
    ("ntsc", 640, 200, layout.PIX_BGRA),   # k_lines2's width range when each line owns its rows
    ("ntsc", 640, 480, layout.PIX_BGRA),
    ("ntsc", 320, 480, layout.PIX_RGB),    # below k_lines2's range; 3-byte pixels
    ("ntsc_conv", 400, 200, layout.PIX_BGRA),  # k_lines_fir
    ("ntsc_conv", 400, 480, layout.PIX_BGR),
    ("ntsc_bloom", 400, 200, layout.PIX_BGRA),  # k_lines_bloom
    ("nes", 640, 480, layout.PIX_BGRA),
    ("pv1k", 400, 200, layout.PIX_BGRA),
    ("pv1k", 400, 480, layout.PIX_ARGB),
])
def test_dropin_vfac_edges(variant, outw, outh, fmt):
    """every edge of tests/test_oracle_vfac.py through the reference's own interface, compared after every call"""
    lines = layout.system_spec(variant).lines
    for name, v_fac in V.vfac_cases(lines, outh):
        gpu, ora, ref = trio(variant, outw, outh, fmt)
        run_all((gpu, ora, ref), lambda e: e.set(v_fac=v_fac))
        for it, call in enumerate(V.CALLS):
            img, kw = V.source(variant, it)
            run_all((gpu, ora, ref), lambda e: e.set(blend=call["blend"], scanlines=call["scanlines"]))
            run_all((gpu, ora, ref), lambda e: e.modulate(img, **V.modulate_kw(variant, call, kw)))
            run_all((gpu, ora, ref), lambda e: e.demodulate(call["noise"]))
            check(gpu, ora, ref, "%s %dx%d v_fac %s (%d) call %d" % (variant, outw, outh, name, v_fac, it))


# one batch, monitors of one size with different v_fac (part of the launch-geometry key: one run of launches each)
BATCH_SPANS = [200, 240, 100, 0, 241, EDGE, EDGE + 1, (1 << 31) + 200, 239, 3 * 200 + 200]


@pytest.mark.parametrize("variant", ["ntsc", "pv1k"])
def test_batch_of_mixed_vfac_matches_the_oracles_line_table(variant):
    """per monitor, crtx_get_lines equals the oracle's sync_pass table (skip / beg / end) and the image the oracle's"""
    import torch
    from ntsc_crt_b200 import capi
    outw, outh = 400, 200
    n = len(BATCH_SPANS)
    b = capi.Batch(variant, n)
    outs = [torch.zeros(outh, outw, 4, dtype=torch.uint8, device="cuda") for _ in range(n)]
    img = S.rand_image(256, 220, seed=70)
    dimg = torch.from_numpy(img).cuda()
    oras = []
    for i, span in enumerate(BATCH_SPANS):
        v_fac = vfac_of_span(span, outh)
        blend, scanlines, noise = (i + 1) & 1, (i >> 1) & 1, 3 * (i % 3)
        b.set_monitor(i, outs[i], fmt=layout.PIX_BGRA, noise=noise, blend=blend, scanlines=scanlines, v_fac=v_fac)
        o = S.OracleEngine(variant, outw, outh)
        o.set(blend=blend, scanlines=scanlines, v_fac=v_fac)
        oras.append((o, noise))
    b.commit_monitors()
    for it in range(3):
        kw = dict(format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=0)
        for i in range(n):
            b.set_source(i, dimg, **kw)
        b.modulate()
        b.demodulate()
        torch.cuda.synchronize()
        for i, (o, noise) in enumerate(oras):
            o.modulate(img, **kw)
            o.noise_pass(noise)
            _, table = o.sync_pass()
            o.line_pass(table)
            got = b.get_lines(i)
            what = "%s span %d field %d monitor %d" % (variant, BATCH_SPANS[i], it, i)
            for k, (g, w) in enumerate(zip(got, table)):
                assert (g.beg < 0) == bool(w.skip), "%s line %d: skip %d, beg %d" % (what, k, w.skip, g.beg)
                if not w.skip:
                    assert (g.beg, g.end) == (w.beg, w.end), "%s line %d" % (what, k)
            image = outs[i].cpu().numpy()
            assert np.array_equal(image, o.out), "%s: %s" % (what, S.diff_report("image", image, o.out))
    b.close()


@pytest.mark.parametrize("variant", ["ntsc", "pv1k"])
def test_frames_host_rows_only_with_vfac(variant, monkeypatch):
    """crtx_frames_host with page-locked 16-byte granular host images and v_fac set.  A stretching v_fac (every line
    owns its rows) takes the rows-only copy: the rows the fields wrote equal the oracle's, the others keep the 0xA5
    sentinel.  A v_fac that wraps outh + v_fac to fewer rows than lines, and one whose products wrap, take the whole
    image: the host image equals the oracle's everywhere."""
    import torch
    from ntsc_crt_b200 import capi
    monkeypatch.setenv("SIMT_HOST_MAPPED", "1")  # (only the CPU interpreter build of the library reads this)
    outw, outh = 640, 400
    v_facs = [300, vfac_of_span(150, outh), vfac_of_span(EDGE + 7, outh)]  # stretching, shrinking (wrapped), wrapping products
    rows_only = [True, False, False]
    n = len(v_facs)
    b = capi.Batch(variant, n)
    b.set_option("host_rows", 1)
    outs = [torch.zeros(outh, outw, 4, dtype=torch.uint8, device="cuda") for _ in range(n)]
    host = [torch.full((outh, outw, 4), 0xA5, dtype=torch.uint8).pin_memory() for _ in range(n)]
    oras = []
    for i in range(n):
        b.set_monitor(i, outs[i], fmt=layout.PIX_BGRA, noise=2 * i, blend=1, scanlines=1, v_fac=v_facs[i])
        o = S.OracleEngine(variant, outw, outh)
        o.set(blend=1, scanlines=1, v_fac=v_facs[i])
        oras.append(o)
    b.commit_monitors()
    written = [np.zeros(outh, dtype=bool) for _ in range(n)]
    for it in range(3):
        imgs = [torch.from_numpy(S.rand_image(640 - 64 * i, 400 - 50 * i, seed=80 + i + it)).pin_memory() for i in range(n)]
        for i in range(n):
            kw = dict(format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=0)
            b.sources[i].data = imgs[i].data_ptr()
            b.sources[i].h, b.sources[i].w = imgs[i].shape[0], imgs[i].shape[1]
            for k, v in kw.items():
                setattr(b.sources[i], k, v)
            oras[i].modulate(imgs[i].numpy(), **kw)
            oras[i].demodulate(2 * i)
        b.frames_host([h.data_ptr() for h in host])
        torch.cuda.synchronize()
        for i in range(n):
            got = host[i].numpy()
            what = "%s field %d v_fac %d" % (variant, it, v_facs[i])
            assert np.array_equal(outs[i].cpu().numpy(), oras[i].out), what
            if not rows_only[i]:
                assert np.array_equal(got, oras[i].out), "%s: %s" % (what, S.diff_report("host image", got, oras[i].out))
                continue
            for l in b.get_lines(i):
                if l.beg >= 0:
                    written[i][l.beg:l.beg + max(1, l.end - 1 - l.beg)] = True
            w = written[i]
            assert 0 < w.sum() < outh or it > 0
            assert np.array_equal(got[w], oras[i].out[w]), "%s: %s" % (what, S.diff_report("written rows", got[w], oras[i].out[w]))
            assert (got[~w] == 0xA5).all(), "%s: a row no field wrote changed on the host" % what
    b.close()


@pytest.mark.parametrize("variant,outw,outh,v_fac,world", [("ntsc", 640, 200, 100, 2), ("ntsc", 640, 180, 60, 3),
                                                            ("ntsc_conv", 400, 200, 40, 2)])
def test_blocks_with_vfac(variant, outw, outh, v_fac, world):
    """the scanline-block partition with a stretching v_fac on an image shorter than the line count: the blocks'
    rows come from outh + v_fac (sharding.block_rows), lines past the image are skipped"""
    decode_one_image_in_blocks(variant, outw, outh, 1, 1, world, v_fac=v_fac)


def test_launches_per_demodulate_by_span():
    """the line passes a demodulate launches (two kernels each: fast and wrap-exact equaliser) after k_sync: one for a
    span of at least one row per line -- the benchmark's geometry, v_fac = 0 -- one per position in a run of lines
    sharing a row when blending, one per level when the products wrap"""
    import torch
    from ntsc_crt_b200 import capi
    outw, outh = 832, 624
    img = torch.from_numpy(S.rand_image(832, 624, seed=3)).cuda()

    def launches(v_fac, blend=1):
        b = capi.Batch("ntsc", 2)
        outs = [torch.zeros(outh, outw, 4, dtype=torch.uint8, device="cuda") for _ in range(2)]
        for i in range(2):
            b.set_monitor(i, outs[i], fmt=layout.PIX_BGRA, noise=4, blend=blend, scanlines=1, v_fac=v_fac)
            b.set_source(i, img, format=layout.PIX_BGRA, as_color=1, field=0, frame=0)
        b.commit_monitors()
        b.modulate()
        before, l2 = b.launches, b.lines2_launches
        b.demodulate()
        torch.cuda.synchronize()
        got = (b.launches - before, b.lines2_launches - l2)
        b.close()
        return got

    assert launches(0) == (3, 1)  # k_sync, k_lines2, the wrap-exact k_lines pass
    assert launches(vfac_of_span(EDGE, outh)) == (3, 1)
    assert launches(vfac_of_span(120, outh)) == (1 + 2 * 3, 0)  # runs of two lines: positions 0, 1 and one spare
    assert launches(vfac_of_span(120, outh), blend=0) == (3, 0)
    assert launches(vfac_of_span(EDGE + 1, outh)) == (1 + 2 * 240, 0)
