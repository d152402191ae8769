"""The additive batch interface's contract around the compute calls (include/crtx_batch.h): argument checking with
an explanation in crtx_last_error(), empty ranges, option names, the launch counter and the per-kernel timers,
state round trips, monitor ranges that are configured and advanced independently."""
import ctypes as C

import numpy as np
import pytest

import support as S
from ntsc_crt_b200 import layout

pytestmark = pytest.mark.gpu


def test_argument_errors_are_reported_not_ignored():
    import torch
    from ntsc_crt_b200 import capi
    lib = capi.load("ntsc")
    ctx = C.c_void_p()
    assert lib.crtx_create(C.byref(ctx), 0) != 0 and b"crtx_create" in lib.crtx_last_error()
    b = capi.Batch("ntsc", 2)
    out = torch.zeros(48, 64, 4, dtype=torch.uint8, device="cuda")
    for name in ("no_such_option", "tma", "fused_noise", "mod_bulk", "lines2_stage", "pdl"):
        with pytest.raises(capi.CrtxError, match="unknown option"):
            b.set_option(name, 1)
    with pytest.raises(capi.CrtxError, match="range"):
        b.modulate(first=1, count=2)
    with pytest.raises(capi.CrtxError, match="range"):
        b.demodulate(first=-1, count=1)
    b.set_monitor(0, out, fmt=layout.PIX_BGRA)
    b.monitors[0].outw = 9000  # above the supported maximum
    with pytest.raises(capi.CrtxError, match="outw"):
        b.commit_monitors(0, 1)
    b.monitors[0].outw = 64
    b.monitors[0].out = out.data_ptr() + 1  # 4-byte pixels need a 4-byte aligned image
    with pytest.raises(capi.CrtxError, match="aligned"):
        b.commit_monitors(0, 1)
    b.close()


def test_empty_ranges_counters_timers_and_state_round_trip():
    import torch
    from ntsc_crt_b200 import capi
    n = 3
    b = capi.Batch("ntsc", n)
    outs = [torch.zeros(240, 320, 4, dtype=torch.uint8, device="cuda") for _ in range(n)]
    img = S.rand_image(256, 240, seed=9)
    dimg = torch.from_numpy(img).cuda()
    for i in range(n):
        b.set_monitor(i, outs[i], fmt=layout.PIX_BGRA, noise=3, blend=0, scanlines=0)
        b.set_source(i, dimg, format=layout.PIX_BGRA, as_color=1, field=0, frame=0)
    b.commit_monitors()
    b.set_option("timing", 1)
    before = b.launches
    b.modulate(first=0, count=0)   # nothing to do is not an error
    b.demodulate(first=2, count=0)
    assert b.launches == before
    # monitors 0 and 2 advance, monitor 1 stays where crtx_create left it
    for i in (0, 2):
        b.modulate(first=i, count=1)
        b.demodulate(first=i, count=1)
    torch.cuda.synchronize()
    assert b.launches > before
    t = b.timing()
    assert t["sync"][1] == 2 and t["lines"][1] >= 2 and all(ms >= 0 for ms, _ in t.values())
    ora = S.OracleEngine("ntsc", 320, 240)
    ora.set(blend=0, scanlines=0)
    ora.modulate(img, format=layout.PIX_BGRA, as_color=1, field=0, frame=0)
    ora.demodulate(3)
    st = b.get_state()
    for i in (0, 2):
        assert np.array_equal(outs[i].cpu().numpy(), ora.out), i
        assert (st[i].hsync, st[i].vsync, st[i].rn) == (ora.hsync, ora.vsync, ora.rn), i
    assert not outs[1].any() and (st[1].hsync, st[1].vsync, st[1].rn) == (0, 0, 194)  # crt_init's state (crt_core.c:250-269)
    assert not b.signal(1, "analog").any()
    # state written back is what the next call starts from: give monitor 1 monitor 0's state and signal, decode again
    b.set_state((capi.State * 1)(st[0]), first=1)
    b.write_signal(1, b.signal(0, "analog"), "analog")
    b.demodulate(first=1, count=1)
    ora.demodulate(3)
    torch.cuda.synchronize()
    assert np.array_equal(outs[1].cpu().numpy(), ora.out)
    lines = b.get_lines(1)
    assert len(lines) == 240 and all(l.beg >= 0 and l.end > l.beg for l in lines)
    b.close()


@pytest.mark.parametrize("variant,host_src", [("ntsc", 0), ("nes", 0), ("pv1k", 0), ("ntsc", 1)])
def test_frames_host_is_the_same_field_with_host_buffers(variant, host_src):
    """crtx_frames_host (what bench.py's e2e figure goes through): source images and decoded images are HOST buffers,
    the copies happen inside the call on the caller's stream.  Images of different sizes (the staging slots grow),
    several fields, outputs compared with the oracle's."""
    import torch
    n = 3
    nes = variant == "nes"
    # "host_src": page-locked source images are read in place by the encoder instead of being copied first
    rig = S.BatchRig(variant, [dict(outw=640, outh=480, fmt=layout.PIX_BGRA, noise=2 * i, knobs=dict(blend=1, scanlines=1))
                               for i in range(n)], options=(("host_src", 1),) if host_src else ())
    host_outs = [np.zeros((480, 640, 4), dtype=np.uint8) for _ in range(n)]
    pinned = []  # keeps page-locked copies alive
    for it in range(3):
        imgs = [S.nes_image(seed=40 + i + it) if nes else S.rand_image(200 + 150 * i + 64 * it, 120 + 100 * i, seed=40 + i + it)
                for i in range(n)]
        if host_src:  # the same images in page-locked memory (monitor 1 stays pageable: that one takes the copy)
            held = [torch.from_numpy(im).pin_memory() if i != 1 else torch.from_numpy(im) for i, im in enumerate(imgs)]
            pinned.append(held)
            imgs = [t.numpy() for t in held]
        for i in range(n):
            kw = dict(dot_crawl_offset=it % 3, hue=10 * i) if nes else dict(format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=0,
                                                                              dot_crawl_offset=it % 3)
            rig.source(i, imgs[i], reinit=int(nes and it == 0), **kw)
        rig.frames_host([h.ctypes.data for h in host_outs])  # HOST source images in, HOST images out
        rig.check("%s field %d" % (variant, it))
        for i in range(n):
            assert np.array_equal(host_outs[i], rig.oras[i].out), "%s field %d monitor %d: %s" % (
                variant, it, i, S.diff_report("host image", host_outs[i], rig.oras[i].out))
    rig.close()


@pytest.mark.parametrize("variant,raw", [("ntsc", 0), ("ntsc", 1), ("pv1k", 0), ("nes", 0), ("ntsc_conv", 0)])
def test_frames_host_moves_only_the_rows_a_field_touches(variant, raw, monkeypatch):
    """crtx_frames_host with page-locked, 16-byte granular host images: the source rows the field reads are gathered
    from the host image in place (crt_ntsc.c:258-266) and only the rows the field wrote are stored back into the host
    image (crt_core.c:428-432, 662-664).  The host image is the monitor's persistent `out`, as in the reference: rows a
    field does not write keep their previous bytes -- proven with a sentinel the device image never held -- and after
    every field the rows that WERE written equal the oracle's.  `host_rows` 0 restores whole-image copies."""
    import torch
    from ntsc_crt_b200 import capi
    monkeypatch.setenv("SIMT_HOST_MAPPED", "1")  # (only the CPU interpreter build of the library reads this)
    n, outw, outh = 3, 832, 624
    nes = variant == "nes"
    for host_rows in (1, 0):
        b = capi.Batch(variant, n)
        b.set_option("host_rows", host_rows)
        outs = [torch.zeros(outh, outw, 4, dtype=torch.uint8, device="cuda") for _ in range(n)]
        host = [torch.full((outh, outw, 4), 0xA5, dtype=torch.uint8).pin_memory() for _ in range(n)]  # sentinel 0xA5
        oras = []
        for i in range(n):
            b.set_monitor(i, outs[i], fmt=layout.PIX_BGRA, noise=3 * i, blend=1, scanlines=1)
            o = S.OracleEngine(variant, outw, outh)
            o.set(blend=1, scanlines=1)
            oras.append(o)
        b.commit_monitors()
        written = [np.zeros(outh, dtype=bool) for _ in range(n)]
        for it in range(3):
            if nes:
                imgs = [torch.from_numpy(S.nes_image(seed=60 + i + it).astype(np.int16)).pin_memory() for i in range(n)]
            elif raw:  # small images placed as they are (crt_ntsc.c:163-172): fewer rows than picture lines
                imgs = [torch.from_numpy(S.rand_image(320 + 64 * i, 100 + 60 * i, seed=60 + i + it)).pin_memory() for i in range(n)]
            else:
                imgs = [torch.from_numpy(S.rand_image(832 - 64 * i, 624 - 100 * i, seed=60 + i + it)).pin_memory() for i in range(n)]
            for i in range(n):
                if nes:
                    kw = dict(dot_crawl_offset=it % 3, hue=10 * i)
                else:
                    # (raw images shorter than the picture: an odd field would read the row one past the image in the
                    # reference, crt_ntsc.c:263 -- outside the reproduced domain, DESIGN.md section 2)
                    kw = dict(format=layout.PIX_BGRA, as_color=1, field=0 if raw else it & 1, frame=(it >> 1) & 1, raw=raw, dot_crawl_offset=it % 3)
                b.sources[i].reinit = 1 if (nes and it == 0) else 0
                b.sources[i].data = imgs[i].data_ptr()
                b.sources[i].h, b.sources[i].w = imgs[i].shape[0], imgs[i].shape[1]
                for k, v in kw.items():
                    setattr(b.sources[i], k, v)
                src_np = imgs[i].numpy().view(np.uint16) if nes else imgs[i].numpy()
                oras[i].modulate(src_np, **kw)
                oras[i].demodulate(3 * i)
            b.frames_host([h.data_ptr() for h in host])
            torch.cuda.synchronize()
            for i in range(n):
                got = host[i].numpy()
                assert np.array_equal(outs[i].cpu().numpy(), oras[i].out), (variant, it, i)
                if not host_rows:
                    assert np.array_equal(got, oras[i].out), "%s field %d monitor %d: %s" % (variant, it, i, S.diff_report("host image", got, oras[i].out))
                    continue
                for l in b.get_lines(i):
                    if l.beg >= 0:
                        written[i][l.beg:l.beg + max(1, l.end - 1 - l.beg)] = True
                w = written[i]
                assert 0 < w.sum() < outh or it > 0
                assert np.array_equal(got[w], oras[i].out[w]), "%s field %d monitor %d: %s" % (
                    variant, it, i, S.diff_report("written rows", got[w], oras[i].out[w]))
                assert (got[~w] == 0xA5).all(), "%s field %d monitor %d: a row no field wrote changed on the host" % (variant, it, i)
        b.close()


@pytest.mark.parametrize("variant", ["ntsc", "ntsc_conv", "template", "pv1k"])
@pytest.mark.parametrize("option,value", [("generic_eq", 1), ("mod_staged", 0), ("lines2", 0)])
def test_every_switch_of_the_library_gives_the_same_bits(variant, option, value):
    """the switches of crtx_set_option that force a path real inputs also take (the wrap-exact equaliser on every
    monitor, the gather encoder, k_lines in place of k_lines2): all of them must decode to the oracle's image"""
    import torch
    from ntsc_crt_b200 import capi
    b = capi.Batch(variant, 2)
    b.set_option(option, value)
    outs = [torch.zeros(300, 400, 4, dtype=torch.uint8, device="cuda") for _ in range(2)]
    imgs = [S.rand_image(320, 240, seed=60), S.bars_image(500, 260)]
    dimgs = [torch.from_numpy(im).cuda() for im in imgs]
    oras = []
    for i in range(2):
        b.set_monitor(i, outs[i], fmt=layout.PIX_BGRA, noise=6 * i, blend=1, scanlines=i, saturation=12)
        o = S.OracleEngine(variant, 400, 300)
        o.set(blend=1, scanlines=i, saturation=12)
        oras.append(o)
    b.commit_monitors()
    for it in range(3):
        for i in range(2):
            kw = dict(format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=0, dot_crawl_offset=it)
            b.set_source(i, dimgs[i], **kw)
            oras[i].modulate(imgs[i], **kw)
            oras[i].demodulate(6 * i)
        b.modulate()
        b.demodulate()
        torch.cuda.synchronize()
        for i in range(2):
            got = outs[i].cpu().numpy()
            assert np.array_equal(got, oras[i].out), "%s %s=%d field %d monitor %d: %s" % (
                variant, option, value, it, i, S.diff_report("out", got, oras[i].out))
            assert np.array_equal(b.signal(i, "analog"), oras[i].analog) and np.array_equal(b.signal(i, "inp"), oras[i].inp)
    b.close()


@pytest.mark.parametrize("variant", ["ntsc", "ntsc_conv", "pv1k", "ntsc_bloom"])
@pytest.mark.parametrize("out_skew,src_skew,src_fmt", [(4, 4, layout.PIX_BGRA), (8, 12, layout.PIX_ARGB), (12, 1, layout.PIX_RGB),
                                                       (4, 2, layout.PIX_BGR)])
def test_images_that_are_not_16_byte_aligned(variant, out_skew, src_skew, src_fmt):
    """Device images handed in at 4-, 8- or 12-byte offsets from a 16-byte boundary (views into larger buffers), 3-byte
    sources at odd addresses: the vector and bulk-copy paths must step aside for the per-lane ones, with no access that
    is misaligned for its type (the interpreter traps on those, the GPU faults)."""
    import torch
    from ntsc_crt_b200 import capi
    outw, outh = 400, 300
    b = capi.Batch(variant, 1)
    big = torch.zeros(outw * outh * 4 + 64, dtype=torch.uint8, device="cuda")
    base = (-big.data_ptr()) % 16  # bytes to the next 16-byte boundary
    out = big[base + out_skew: base + out_skew + outw * outh * 4].view(outh, outw, 4)
    assert out.data_ptr() % 16 == out_skew
    rgb = S.rand_image(320, 240, bpp=3, seed=90)
    img = S.pack_rgb(rgb, src_fmt)
    bpp = img.shape[2]
    sbig = torch.zeros(img.size + 64, dtype=torch.uint8, device="cuda")
    sbase = (-sbig.data_ptr()) % 16
    dimg = sbig[sbase + src_skew: sbase + src_skew + img.size].view(240, 320, bpp)
    dimg.copy_(torch.from_numpy(img))
    assert dimg.data_ptr() % 16 == src_skew % 16
    b.set_monitor(0, out, fmt=layout.PIX_BGRA, noise=3, blend=1, scanlines=1)
    b.commit_monitors()
    ora = S.OracleEngine(variant, outw, outh)
    ora.set(blend=1, scanlines=1)
    for it in range(3):
        kw = dict(format=src_fmt, as_color=1, field=it & 1, frame=0, dot_crawl_offset=it, xoffset=4 * (it & 1))
        b.set_source(0, dimg, **kw)
        ora.modulate(img, **kw)
        ora.demodulate(3)
        b.modulate()
        b.demodulate()
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        assert np.array_equal(got, ora.out), "%s field %d: %s" % (variant, it, S.diff_report("out", got, ora.out))
        assert np.array_equal(b.signal(0, "analog"), ora.analog)
    assert not big[:base + out_skew].any() and not big[base + out_skew + outw * outh * 4:].any(), "wrote outside the image"
    b.close()


@pytest.mark.parametrize("variant", ["ntsc", "vhs", "template"])
def test_picture_moved_into_the_skeleton_keeps_the_reference_order(variant):
    """crt_modulate writes the sync / blank / burst skeleton first and the picture over it (crt_ntsc.c:205-324); offsets
    move the picture into the skeleton's bytes (above CRT_TOP, left of AV_BEG, or -- xoffset >= 4 -- three bytes into the
    next line's porch), where that order decides the result.  A batch that mixes such pictures with ordinary ones, against
    the oracle, analog[] included."""
    import torch
    from ntsc_crt_b200 import capi
    n = 3
    offs = [(0, 0), (-12, -4), (8, 3)]
    b = capi.Batch(variant, n)
    outs = [torch.zeros(480, 640, 4, dtype=torch.uint8, device="cuda") for _ in range(n)]
    imgs = [S.rand_image(300, 200, seed=90 + i) for i in range(n)]
    dimgs = [torch.from_numpy(im).cuda() for im in imgs]
    oras = []
    for i in range(n):
        b.set_monitor(i, outs[i], fmt=layout.PIX_BGRA, noise=0 if variant == "vhs" else 5, blend=0, scanlines=0)
        o = S.OracleEngine(variant, 640, 480)
        o.set(blend=0, scanlines=0)
        oras.append(o)
    b.commit_monitors()
    for f in range(3):
        for i in range(n):
            kw = dict(format=layout.PIX_BGRA, as_color=1, field=f & 1, frame=(f >> 1) & 1, xoffset=offs[i][0], yoffset=offs[i][1],
                      dot_crawl_offset=f % 2)
            b.set_source(i, dimgs[i], **kw)
            oras[i].modulate(imgs[i], **kw)
        b.modulate()
        for i in range(n):
            assert np.array_equal(b.signal(i, "analog"), oras[i].analog), "%s field %d monitor %d: %s" % (
                variant, f, i, S.diff_report("analog", b.signal(i, "analog"), oras[i].analog))
        if variant != "vhs":  # (VHS noise comes from rand(): the stream comparison has its own tests)
            b.demodulate()
            torch.cuda.synchronize()
            for i in range(n):
                oras[i].demodulate(5)
                assert np.array_equal(outs[i].cpu().numpy(), oras[i].out), (variant, f, i)
    b.close()
