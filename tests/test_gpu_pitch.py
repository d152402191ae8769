"""Row-pitched images in the batch interface (include/crtx_batch.h: crtx_monitor::out_pitch, crtx_source::pitch).

Sources and outputs are windows of larger torch tensors whose padding holds a sentinel.  Every field must equal the
oracle's image bit for bit, no padding byte may change, the fast paths must still be taken for rows on 16-byte
boundaries (and the general ones, exactly, otherwise), a batch with one shared pitch must launch what the dense batch
launches, and a rejected pitch must leave the context as it was.

The same bodies run on the CPU through the SIMT interpreter (TestOnTheInterpreter, below)."""
import ctypes as C

import numpy as np
import pytest

import support as S
from ntsc_crt_b200 import capi, layout
from test_simt_kernels import simt_libs  # noqa: F401  (session fixture of the interpreter builds)
import test_simt_kernels as _simt

SENT = 0xA7


def _nes(variant):
    return layout.system_spec(variant).system == layout.SYS_NES


def _window(h, w, c, pad, off, fill=SENT, dtype=None):
    """a (h, w, c) -- or (h, w) when c is 0 -- view at column `off` of a canvas `pad` pixels wider, every byte `fill`"""
    import torch
    dtype = dtype or torch.uint8
    canvas = torch.full((h, w + pad, c) if c else (h, w + pad), fill, dtype=dtype, device="cuda")
    return canvas, canvas[:, off:off + w]


def _pixels(canvas, off, w):
    """(image region, padding) of a canvas as numpy arrays"""
    a = canvas.cpu().numpy()
    mask = np.ones(a.shape[1], dtype=bool)
    mask[off:off + w] = False
    return a[:, off:off + w], a[:, mask]


def _source(variant, w, h, fmt, seed):
    if _nes(variant):
        return S.nes_image(w, h, seed=seed).astype(np.int16)  # 9-bit PPU pixels in 2-byte elements
    return S.rand_image(w, h, bpp=layout.bpp4fmt(fmt), seed=seed)


def _put(t, img):
    import torch
    t.copy_(torch.from_numpy(img).to(t.device))


def _settings(variant, it, i, fmt):
    if _nes(variant):
        return dict(dot_crawl_offset=(it + i) % 3, hue=10 * i)
    return dict(format=fmt, as_color=1, field=it & 1, frame=(it >> 1) & 1, dot_crawl_offset=(it + i) % 3)


def _oracle_src(img):
    return img.view(np.uint16) if img.dtype == np.int16 else img


# ---- 1. every variant, pitched in and out --------------------------------------------------------------------------
# (outw, outh, output format, canvas pad in pixels, column offset), (source w, h, format, pad, offset)
CASES = [((397, 250, layout.PIX_BGRA, 5, 3), (203, 180, layout.PIX_BGRA, 3, 1)),
         ((301, 246, layout.PIX_BGR, 7, 2), (150, 120, layout.PIX_RGB, 5, 2))]


def check_every_variant(variant):
    import torch
    nes = _nes(variant)
    b = capi.Batch(variant, len(CASES))
    outs, srcs, oras, imgs = [], [], [], []
    for i, ((outw, outh, fmt, pad, off), (w, h, sfmt, spad, soff)) in enumerate(CASES):
        canvas, view = _window(outh, outw, layout.bpp4fmt(fmt), pad, off)
        view.zero_()  # (the oracle's image starts black; blend reads it)
        b.set_monitor(i, view, fmt=fmt, noise=5 + 4 * i, blend=1, scanlines=i)
        assert b.monitors[i].out_pitch == (outw + pad) * layout.bpp4fmt(fmt)
        outs.append((canvas, off, outw))
        o = S.OracleEngine(variant, outw, outh, fmt=fmt)
        o.set(blend=1, scanlines=i)
        oras.append(o)
        if nes:
            w, h = 256 - 40 * i, 240 - 50 * i
        scanvas, sview = _window(h, w, 0 if nes else layout.bpp4fmt(sfmt), spad, soff, fill=0x5A,
                                 dtype=torch.int16 if nes else None)
        srcs.append((scanvas, sview, sfmt))
    b.commit_monitors()
    for it in range(3):
        for i, (scanvas, sview, sfmt) in enumerate(srcs):
            img = _source(variant, sview.shape[1], sview.shape[0], sfmt, seed=10 * it + i)
            _put(sview, img)
            kw = _settings(variant, it, i, sfmt)
            b.set_source(i, sview, **kw)
            b.sources[i].reinit = 1 if it == 0 else 0  # (NES and NES-RGB: the first field writes the sync template)
            oras[i].modulate(_oracle_src(img), **kw)
            oras[i].demodulate(5 + 4 * i)
        b.modulate()
        b.demodulate()
        torch.cuda.synchronize()
        for i, (canvas, off, outw) in enumerate(outs):
            got, padding = _pixels(canvas, off, outw)
            assert np.array_equal(got, oras[i].out), "%s field %d monitor %d: %s" % (
                variant, it, i, S.diff_report("out", got, oras[i].out))
            assert (padding == SENT).all(), "%s field %d monitor %d: a byte between rows changed" % (variant, it, i)
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("variant", capi.VARIANTS)
def test_every_variant_decodes_pitched_images_exactly(variant):
    check_every_variant(variant)


# ---- 2. paths, and the launches of the dense batch ----------------------------------------------------------------
def _run_pair(variant, pad, src_pad, fields=2, n=2, outw=640, outh=480):
    """the same batch twice: pitched (`pad` extra pixels per output row, `src_pad` per source row) and dense.
    Returns the pitched run's outputs, paths and counters, and the dense run's."""
    import torch
    runs = []
    for pitched in (True, False):
        b = capi.Batch(variant, n)
        canv, views = [], []
        for i in range(n):
            if pitched:
                c, v = _window(outh, outw, 4, pad, 0)
            else:
                c = v = torch.full((outh, outw, 4), SENT, dtype=torch.uint8, device="cuda")  # (blend reads it)
            canv.append(c)
            views.append(v)
            b.set_monitor(i, v, fmt=layout.PIX_BGRA, noise=3 + i, blend=1, scanlines=1)
        b.commit_monitors()
        imgs = [S.rand_image(256, 240, seed=70 + i) for i in range(n)]
        dsrc = []
        for i in range(n):
            if pitched:
                _, sv = _window(240, 256, 4, src_pad, 0, fill=0)
                _put(sv, imgs[i])
            else:
                sv = torch.from_numpy(imgs[i]).cuda()
            dsrc.append(sv)
        l0, l2 = b.launches, b.lines2_launches
        for it in range(fields):
            for i in range(n):
                b.set_source(i, dsrc[i], format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=0)
            b.modulate()
            b.demodulate()
        torch.cuda.synchronize()
        got = [v.cpu().numpy().copy() for v in views]
        pads = [_pixels(c, 0, outw)[1] if pitched else None for c in canv]
        runs.append(dict(out=got, pad=pads, paths=b.paths(), launches=b.launches - l0, lines2=b.lines2_launches - l2))
        b.close()
    return runs


def check_paths(variant):
    # rows on 16-byte boundaries: 648- and 260-pixel canvases (2592- and 1040-byte pitches)
    fast, dense = _run_pair(variant, pad=8, src_pad=4)
    for i in range(2):
        assert np.array_equal(fast["out"][i], dense["out"][i]), (variant, i)
        assert (fast["pad"][i] == SENT).all(), (variant, i)
    assert fast["launches"] == dense["launches"] and fast["lines2"] == dense["lines2"], (fast, dense)
    for p, q in zip(fast["paths"], dense["paths"]):
        assert p == q, (variant, fast["paths"], dense["paths"])
        if variant in ("ntsc", "ntsc_conv", "pv1k"):
            assert p & capi.Batch.PATH_STAGED_MOD and p & capi.Batch.PATH_ROW16, (variant, p)
    if variant == "ntsc":
        assert fast["lines2"] > 0
    # pitches 4 bytes past a multiple of 16 (641- and 257-pixel canvases): the general paths, the same bits
    slow, dense2 = _run_pair(variant, pad=1, src_pad=1)
    for i in range(2):
        assert np.array_equal(slow["out"][i], dense2["out"][i]), (variant, i)
        assert (slow["pad"][i] == SENT).all(), (variant, i)
    for p in slow["paths"]:
        assert not p & capi.Batch.PATH_ROW16, (variant, p)
        if variant in ("ntsc", "ntsc_conv", "pv1k"):
            assert p & capi.Batch.PATH_STAGED_MOD  # (the staged encoder needs 4-byte aligned rows only)
    if variant == "ntsc":
        assert slow["lines2"] == 0 and dense2["lines2"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["ntsc", "ntsc_conv", "pv1k", "ntsc_bloom"])
def test_fast_paths_need_rows_on_16_byte_boundaries(variant):
    check_paths(variant)


# ---- 3. a mosaic: monitors decode into side-by-side tiles of one tensor ---------------------------------------------
def check_mosaic(variant, line_window):
    import torch
    n, tw, th = 4, 320, 240
    canvas = torch.full((th, n * tw + 16, 4), SENT, dtype=torch.uint8, device="cuda")
    imgs = [S.rand_image(200 + 20 * i, 150, seed=90 + i) for i in range(n)]
    dimgs = [torch.from_numpy(im).cuda() for im in imgs]
    tiled = capi.Batch(variant, n)
    singles = [capi.Batch(variant, 1) for _ in range(n)]
    alone = [torch.full((th, tw, 4), SENT, dtype=torch.uint8, device="cuda") for _ in range(n)]  # (rows a window skips)
    for b in [tiled] + singles:
        if line_window:
            b.set_option("line_lo", line_window[0])
            b.set_option("line_hi", line_window[1])
    for i in range(n):
        knobs = dict(noise=4 * i, blend=1, scanlines=i & 1, hue=7 * i)
        tiled.set_monitor(i, canvas[:, 8 + i * tw: 8 + (i + 1) * tw], fmt=layout.PIX_BGRA, **knobs)
        singles[i].set_monitor(0, alone[i], fmt=layout.PIX_BGRA, **knobs)
        singles[i].commit_monitors()
    tiled.commit_monitors()
    for it in range(3):
        for i in range(n):
            kw = dict(format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=0, dot_crawl_offset=it % 3)
            tiled.set_source(i, dimgs[i], **kw)
            singles[i].set_source(0, dimgs[i], **kw)
            singles[i].modulate()
            singles[i].demodulate()
        tiled.modulate()
        tiled.demodulate()
        torch.cuda.synchronize()
        a = canvas.cpu().numpy()
        for i in range(n):
            assert np.array_equal(a[:, 8 + i * tw: 8 + (i + 1) * tw], alone[i].cpu().numpy()), (variant, line_window, it, i)
        assert (a[:, :8] == SENT).all() and (a[:, 8 + n * tw:] == SENT).all()
    for b in [tiled] + singles:
        b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["ntsc", "ntsc_conv"])
@pytest.mark.parametrize("line_window", [None, (37, 181)])
def test_mosaic_tiles_decode_like_separate_images(variant, line_window):
    check_mosaic(variant, line_window)


# ---- 4. crtx_frames_host with host rows padded to 16 bytes --------------------------------------------------------
def check_frames_host(variant, host_src):
    import torch
    n, outw, outh, opitch = 2, 1366, 600, 5472  # 5464-byte rows padded to 5472
    b = capi.Batch(variant, n)
    if host_src:
        b.set_option("host_src", 1)
    outs = [torch.zeros(outh * opitch, dtype=torch.uint8, device="cuda") for _ in range(n)]
    host = [torch.full((outh * opitch,), SENT, dtype=torch.uint8).pin_memory() for _ in range(n)]
    oras = []
    for i in range(n):
        view = outs[i].as_strided((outh, outw, 4), (opitch, 4, 1))
        b.set_monitor(i, view, fmt=layout.PIX_BGRA, noise=3 + i, blend=1, scanlines=1)
        assert b.monitors[i].out_pitch == opitch
        o = S.OracleEngine(variant, outw, outh)
        o.set(blend=1, scanlines=1)
        oras.append(o)
    b.commit_monitors()
    written = [np.zeros(outh, dtype=bool) for _ in range(n)]
    spitch = 1376  # 341 BGRA pixels = 1364 bytes, padded to 1376
    keep = []
    for it in range(3):
        for i in range(n):
            img = S.rand_image(341, 200 + 20 * i, seed=30 + it + i)
            src = torch.full((img.shape[0] * spitch,), 0, dtype=torch.uint8).pin_memory()
            src.as_strided(img.shape, (spitch, 4, 1)).copy_(torch.from_numpy(img))
            keep.append(src)
            kw = dict(format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=0, dot_crawl_offset=it % 3)
            s = b.sources[i]
            s.data, s.h, s.w, s.pitch = src.data_ptr(), img.shape[0], img.shape[1], spitch
            for k, v in kw.items():
                setattr(s, k, v)
            oras[i].modulate(img, **kw)
            oras[i].demodulate(3 + i)
        b.frames_host([h.data_ptr() for h in host])
        torch.cuda.synchronize()
        for i in range(n):
            full = host[i].numpy().reshape(outh, opitch)
            got, padding = full[:, :outw * 4].reshape(outh, outw, 4), full[:, outw * 4:]
            assert (padding == SENT).all(), (variant, host_src, it, i)
            assert np.array_equal(outs[i].cpu().numpy().reshape(outh, opitch)[:, :outw * 4].reshape(outh, outw, 4), oras[i].out)
            written[i] |= S.written_rows(b.get_lines(i), outh, 1)
            w = written[i]
            assert 0 < w.sum() < outh or it > 0
            assert np.array_equal(got[w], oras[i].out[w]), (variant, host_src, it, i, S.diff_report("rows", got[w], oras[i].out[w]))
            assert (got[~w] == SENT).all(), "%s: a row no field wrote changed on the host (the rows-only path did not run)" % variant
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("variant,host_src", [("ntsc", 0), ("ntsc", 1), ("pv1k", 0)])
def test_frames_host_moves_only_the_rows_of_padded_host_images(variant, host_src):
    check_frames_host(variant, host_src)


# ---- 5. the error contract -----------------------------------------------------------------------------------------
def check_rejected_pitches(variant):
    import torch
    nes = _nes(variant)
    fmt = layout.PIX_BGRA
    outw, outh = 320, 240
    img = _source(variant, 256, 240, fmt, seed=5)
    dimg = torch.from_numpy(img).cuda()

    def field(b, out):
        b.set_source(0, dimg, **_settings(variant, 0, 0, fmt))
        b.sources[0].reinit = 1
        b.modulate()
        b.demodulate()
        torch.cuda.synchronize()
        return out.cpu().numpy().copy(), b.signal(0, "analog")

    fresh_out = torch.zeros(outh, outw, 4, dtype=torch.uint8, device="cuda")
    fresh = capi.Batch(variant, 1)
    fresh.set_monitor(0, fresh_out, fmt=fmt, noise=4, blend=1)
    fresh.commit_monitors()
    want = field(fresh, fresh_out)
    fresh.close()

    out = torch.zeros(outh, outw, 4, dtype=torch.uint8, device="cuda")
    b = capi.Batch(variant, 1)
    b.set_monitor(0, out, fmt=fmt, noise=4, blend=1)
    b.commit_monitors()
    for bad, rule in ((outw * 4 - 4, "below"), (-outw * 4, "negative"), (outw * 4 + 2, "multiple of 4")):
        b.monitors[0].out_pitch = bad
        with pytest.raises(capi.CrtxError, match="monitor 0: .*%s" % rule):
            b.commit_monitors()
    b.monitors[0].out_pitch = 0  # 0: dense
    b.commit_monitors()
    row = 256 * (2 if nes else 4)
    bads = [(row - 2, "below"), (-row, "negative")] + ([(row + 1, "odd")] if nes else [(row + 2, "multiple of 4")])
    for bad, rule in bads:
        b.set_source(0, dimg, **_settings(variant, 0, 0, fmt))
        b.sources[0].pitch = bad
        with pytest.raises(capi.CrtxError, match="monitor 0: .*%s" % rule):
            b.modulate()
        with pytest.raises(capi.CrtxError, match="monitor 0: .*%s" % rule):
            b.frames_host([None])
    got = field(b, out)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), variant
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["ntsc", "nes", "snes"])
def test_rejected_pitches_leave_the_context_as_it_was(variant):
    check_rejected_pitches(variant)


# ---- 6. the binding ------------------------------------------------------------------------------------------------
def check_binding():
    import torch
    b = capi.Batch("ntsc", 2)
    dense = torch.zeros(48, 64, 4, dtype=torch.uint8, device="cuda")
    b.set_monitor(0, dense)
    assert b.monitors[0].out_pitch == 64 * 4
    canvas = torch.zeros(48, 200, 4, dtype=torch.uint8, device="cuda")
    b.set_monitor(1, canvas[:, 10:74])
    assert b.monitors[1].out_pitch == 200 * 4 and b.monitors[1].outw == 64
    nes = torch.zeros(40, 300, dtype=torch.int16, device="cuda")
    b.set_source(0, nes[:, 8:264])
    assert b.sources[0].pitch == 600 and b.sources[0].w == 256
    b.set_source(1, canvas)
    assert b.sources[1].pitch == 800
    for bad in (canvas[:, ::2], canvas.permute(1, 0, 2), canvas[:, :, :3].transpose(0, 1), nes[:, ::2], nes.t()):
        with pytest.raises(ValueError):
            b.set_monitor(0, bad)
        with pytest.raises(ValueError):
            b.set_source(0, bad)
    # source_table follows the structure: its dtype has the pitch column
    t = capi.source_table(b.sources)
    assert "pitch" in t.dtype.names and list(t["pitch"]) == [600, 800]
    b.close()


@pytest.mark.gpu
def test_binding_takes_the_pitch_from_the_tensor():
    check_binding()


# ---- the same bodies on the CPU, through the SIMT interpreter ------------------------------------------------------
class TestOnTheInterpreter:
    simt_backend = staticmethod(_simt.simt_backend)  # autouse within this class: the interpreter builds, host "device" tensors

    @pytest.mark.parametrize("variant", capi.VARIANTS)
    def test_every_variant(self, variant):
        check_every_variant(variant)

    @pytest.mark.parametrize("variant", ["ntsc", "ntsc_conv", "pv1k", "ntsc_bloom"])
    def test_paths(self, variant):
        check_paths(variant)

    @pytest.mark.parametrize("line_window", [None, (37, 181)])
    def test_mosaic(self, line_window):
        check_mosaic("ntsc", line_window)

    @pytest.mark.parametrize("host_src", [0, 1])
    def test_frames_host(self, host_src, monkeypatch):
        monkeypatch.setenv("SIMT_HOST_MAPPED", "1")  # (only the interpreter build of the library reads this)
        check_frames_host("ntsc", host_src)

    @pytest.mark.parametrize("variant", ["ntsc", "nes"])
    def test_rejected_pitches(self, variant):
        check_rejected_pitches(variant)

    def test_binding(self):
        check_binding()
