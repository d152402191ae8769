"""The NES border colour: the libraries built with NES_BORDER 1 (crt_nes.c:64-69; libcrt_b200_nes_border.so on the
stock timing, libcrt_b200_nes_p0_border.so on chroma pattern 0) draw lines CRT_TOP .. CRT_BOT + 2 from LAV_BEG on in
settings.border_color on every call, the picture over it (crt_nes.c:138-161).  Every field is compared bit for bit with
the CPU model of the border (tests/nes_border_oracle.py, the stock oracle plus the border bytes) and, where it is built,
with the reference compiled with the switch on (oracle/_ref/libref_*_border.so, oracle/nes_border.mk):
batches that span the border colours, dot crawl, black and white points, picture offsets and re-initialisations; the
drop-in interface; crtx_frames_host; a line-block split.  The stock NES library ignores the field, as the reference does.

The same bodies run on the CPU through the SIMT interpreter (TestOnTheInterpreter, below)."""
import numpy as np
import pytest

import support as S
from nes_border_oracle import BORDER_VARIANTS, COLOURS, XMAX, oracle_engine
from ntsc_crt_b200 import capi, layout, sharding
from test_simt_kernels import simt_libs  # noqa: F401  (session fixture of the interpreter builds)
import test_simt_kernels as _simt

# monitor knobs: (black_point, white_point, hue, blend, scanlines)
KNOBS = [(0, 100, 0, 1, 1), (6, 90, 20, 0, 1), (-4, 115, -30, 1, 0), (12, 80, 75, 0, 0)]

BATCH, FIELDS = 64, 9  # every colour in COLOURS at least once across the batch's fields
OUTW, OUTH = 400, 300


def _settings(variant, it, i, n):
    return dict(dot_crawl_offset=(i + it) % 3, hue=(37 * i + 11 * it) % 360, xoffset=(7 * i + 3 * it) % (XMAX[variant] + 1),
                yoffset=(i + it) % 8, border_color=COLOURS[(it * n + i) % len(COLOURS)])


def _reinit(it, i):
    """the first field writes the sync template, and every other monitor writes it again in field 3"""
    return it == 0 or (it == 3 and i % 2 == 1)


def check_batch(variant, n=None, fields=None):
    """n monitors for `fields` consecutive fields, every field's whole state against the oracle"""
    n, fields = n or BATCH, fields or FIELDS
    mons = []
    for i in range(n):
        bp, wp, hue, blend, scan = KNOBS[i % len(KNOBS)]
        mons.append(dict(outw=OUTW, outh=OUTH, fmt=layout.PIX_BGRA, noise=(5 * i) % 17,
                         knobs=dict(blend=blend, scanlines=scan, black_point=bp, white_point=wp, hue=hue)))
    rig = S.BatchRig(variant, mons, oracle=oracle_engine)
    imgs = [S.nes_image(seed=300 + i, rainbow=(i % 5 == 4)) for i in range(n)]
    for it in range(fields):
        for i in range(n):
            rig.source(i, imgs[i], reinit=int(_reinit(it, i)), **_settings(variant, it, i, n))
        rig.modulate()
        rig.demodulate()
        rig.check("%s field %d" % (variant, it))
    rig.close()


def check_dropin(variant, fields=8):
    """the drop-in interface (crt_modulate / crt_demodulate, NTSC_SETTINGS.border_color), after every call; the settings
    are re-initialised once more half way"""
    gpu, ora, ref = S.trio(variant, 832, 624, oracle=oracle_engine)
    S.run_all((gpu, ora, ref), lambda e: e.set(blend=1, scanlines=1, black_point=3, white_point=93))
    img = S.nes_image(seed=21)
    for it in range(fields):
        kw = dict(border_color=[0x22, 0x0f, 0x1ff, 0x2d, 0x30, 0x100 | 0x16, 0x0d, 0x222][it % 8], dot_crawl_offset=it % 3,
                  hue=(it * 40) % 360, xoffset=[0, XMAX[variant], 16, 7, 3, 28, 12, 1][it % 8], yoffset=it % 8)
        if it == fields // 2:
            kw["field_initialized"] = 0
        S.run_all((gpu, ora, ref), lambda e: e.modulate(img, **kw))
        S.check(gpu, ora, ref, "%s drop-in mod %d" % (variant, it))
        S.run_all((gpu, ora, ref), lambda e: e.demodulate(3 * it))
        S.check(gpu, ora, ref, "%s drop-in demod %d" % (variant, it))


def check_frames_host(variant, n=3, fields=4):
    """crtx_frames_host: host source images in, host images out; the whole state, and the output rows the fields write
    in the host images, equal the oracle's"""
    import torch
    outw, outh = 640, 480
    rig = S.BatchRig(variant, [dict(outw=outw, outh=outh, fmt=layout.PIX_BGRA, noise=2 + i,
                                    knobs=dict(blend=1, scanlines=1, black_point=i, white_point=100 - 5 * i)) for i in range(n)],
                     oracle=oracle_engine)
    host = [torch.zeros(outh, outw, 4, dtype=torch.uint8).pin_memory() for _ in range(n)]
    srcs = [torch.from_numpy(S.nes_image(256, 240 - 16 * i, seed=60 + i).astype(np.int16)).pin_memory() for i in range(n)]
    imgs = [s.numpy().view(np.uint16) for s in srcs]  # (the page-locked images themselves)
    for it in range(fields):
        for i in range(n):
            rig.source(i, imgs[i], reinit=int(it == 0), dot_crawl_offset=(it + i) % 3, hue=15 * i,
                       xoffset=(9 * it + 5 * i) % (XMAX[variant] + 1), yoffset=(it + 2 * i) % 8,
                       border_color=(0x22 + 0x41 * it + 0x9 * i) & 0x1ff)
        rig.frames_host([h.data_ptr() for h in host])
        rig.check("%s frames_host field %d" % (variant, it))
        for i in range(n):
            got, want = host[i].numpy(), rig.oras[i].out
            rows = np.zeros(outh, dtype=bool)
            for l in rig.b.get_lines(i):
                if l.beg >= 0:
                    rows[l.beg:l.beg + max(1, l.end - 1 - l.beg)] = True
            assert rows.any()
            assert np.array_equal(got[rows], want[rows]), (variant, it, i, S.diff_report("rows", got[rows], want[rows]))
    rig.close()


def check_line_blocks(variant, world=2, outw=832, outh=624, fields=5):
    """two contexts each decode their own block of lines (crtx_set_option line_lo / line_hi, sharding.ImageSharder);
    the merged image equals the oracle's sequential decode"""
    import torch
    img = S.nes_image(seed=77)
    dimg = torch.from_numpy(img.astype(np.int16)).cuda()
    ora = oracle_engine(variant, outw, outh)
    ora.set(blend=1, scanlines=1)
    ranks = []
    for r in range(world):
        b = capi.Batch(variant, 1)
        out = torch.zeros(outh, outw, 4, dtype=torch.uint8, device="cuda")
        b.set_monitor(0, out, fmt=layout.PIX_BGRA, noise=4, blend=1, scanlines=1)
        b.commit_monitors()
        part = sharding.ImageSharder(out, b.spec.lines, rank=r, world=world)
        part.apply(b)
        ranks.append((b, out, part))
    for it in range(fields):
        kw = dict(dot_crawl_offset=it % 3, border_color=(0x22 * (it + 1)) & 0x1ff, xoffset=4 * it, yoffset=it)
        ora.modulate(img, field_initialized=int(it != 0), **kw)
        ora.demodulate(4)
        ends = []
        for r in range(world - 1):  # the halo rows ImageSharder.fetch_halo_rows hands over before the field
            (_, dst, ps), (_, src, pn) = ranks[r], ranks[r + 1]
            cnt = ps._halo_count(r)
            if cnt:
                dst[ps.r1:ps.r1 + cnt].copy_(src[pn.r0:pn.r0 + cnt])
        for b, out, part in ranks:
            b.set_source(0, dimg, **kw)
            b.sources[0].reinit = int(it == 0)
            b.modulate()
            b.demodulate()
            last = b.get_lines(0)[part.hi - 1]
            ends.append(0 if last.beg < 0 else max(last.beg + 1, last.end - 1))
        torch.cuda.synchronize()
        for r in range(world - 1):  # the spill rows ImageSharder.exchange_spill_rows hands on after it
            (_, src, ps), (_, dst, pd) = ranks[r], ranks[r + 1]
            cnt = max(0, min(ends[r], outh, ps.r1 + ps.max_spill()) - ps.r1)
            if cnt and pd.r0 == ps.r1:
                dst[pd.r0:pd.r0 + cnt].copy_(src[ps.r1:ps.r1 + cnt])
    full = np.zeros((outh, outw, 4), dtype=np.uint8)
    for b, out, part in ranks:
        full[part.r0:part.r1] = out[part.r0:part.r1].cpu().numpy()
        b.close()
    assert np.array_equal(full, ora.out), S.diff_report("merged image", full, ora.out)


def check_stock_ignores_the_border(variant="nes", fields=3):
    """the stock NES library gives the same bytes whatever border_color holds, as the reference's NES_BORDER 0 build does:
    one monitor with border_color 0, one with 0x22, in one batch and through the drop-in interface"""
    import torch
    b = capi.Batch(variant, 2)
    outs = [torch.zeros(240, 320, 4, dtype=torch.uint8, device="cuda") for _ in range(2)]
    for i in range(2):
        b.set_monitor(i, outs[i], fmt=layout.PIX_BGRA, noise=3, blend=1, scanlines=1)
    b.commit_monitors()
    dimg = torch.from_numpy(S.nes_image(seed=8).astype(np.int16)).cuda()
    ora = oracle_engine(variant, 320, 240)
    ora.set(blend=1, scanlines=1)
    for it in range(fields):
        for i in range(2):
            b.set_source(i, dimg, dot_crawl_offset=it % 3, xoffset=8, yoffset=2, border_color=(0, 0x22)[i])
            b.sources[i].reinit = int(it == 0)
        ora.modulate(S.nes_image(seed=8), dot_crawl_offset=it % 3, xoffset=8, yoffset=2, field_initialized=int(it != 0))
        ora.demodulate(3)
        b.modulate()
        b.demodulate()
        torch.cuda.synchronize()
        for which in ("analog", "inp"):
            assert np.array_equal(b.signal(0, which), b.signal(1, which)), (which, it)
            assert np.array_equal(b.signal(0, which), getattr(ora, which)), (which, it)
        assert np.array_equal(outs[0].cpu().numpy(), outs[1].cpu().numpy()), it
    b.close()
    img = S.nes_image(seed=9)
    states = []
    for colour in (0, 0x22):
        e = S.ProductEngine(variant, 320, 240)
        e.set(blend=1, scanlines=1)
        for it in range(fields):
            e.modulate(img, dot_crawl_offset=it % 3, border_color=colour)
            e.demodulate(2)
        states.append(e.state())
    S.assert_same_state(states[0], states[1], "%s border_color 0 vs 0x22" % variant)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", BORDER_VARIANTS)
def test_batch_spans_border_colours_offsets_and_reinit(variant):
    check_batch(variant)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", BORDER_VARIANTS)
def test_dropin_border(variant):
    check_dropin(variant)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", BORDER_VARIANTS)
def test_frames_host_border(variant):
    check_frames_host(variant)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", BORDER_VARIANTS)
def test_line_blocks_border(variant):
    check_line_blocks(variant)


@pytest.mark.gpu
def test_stock_nes_ignores_border_color():
    check_stock_ignores_the_border()


@pytest.mark.parametrize("variant", BORDER_VARIANTS)
def test_border_library_exports_and_geometry(variant):
    """every symbol the headers declare is exported, and the library reports its system, timing and border switch
    (capi.load checks crtx_nes_border against the variant too)"""
    import ctypes as C
    import test_capi_exports as X
    lib = C.CDLL(capi.lib_path(variant))
    for name in X.declared("crt_b200.h") + X.declared("crtx_batch.h"):
        assert hasattr(lib, name), "%s missing from %s" % (name, variant)
    lib = capi.load(variant)
    spec = layout.system_spec(variant)
    assert (lib.crtx_system(), lib.crtx_chroma_pattern(), lib.crtx_hres(), lib.crtx_nes_border()) == (
        layout.SYS_NES, spec.pattern, spec.hres, 1)
    assert capi.load("nes").crtx_nes_border() == 0 and capi.load("nes_p0").crtx_nes_border() == 0
    assert variant in capi.ALL_VARIANTS and variant not in capi.VARIANTS


# ---- the same bodies on the CPU, through the SIMT interpreter ------------------------------------------------------
class TestOnTheInterpreter:
    simt_backend = staticmethod(_simt.simt_backend)  # autouse within this class: the interpreter builds, host "device" tensors

    @pytest.mark.parametrize("variant", BORDER_VARIANTS)
    def test_batch(self, variant):
        check_batch(variant, n=6, fields=7)

    @pytest.mark.parametrize("variant", BORDER_VARIANTS)
    def test_every_border_colour(self, variant):
        """every colour of COLOURS through the interpreted encoder: analog only, 16 monitors per call"""
        import torch
        n = 16
        b = capi.Batch(variant, n)
        oras = []
        for i in range(n):
            bp, wp, hue, blend, scan = KNOBS[i % len(KNOBS)]
            b.set_monitor(i, torch.zeros(48, 64, 4, dtype=torch.uint8), fmt=layout.PIX_BGRA, black_point=bp, white_point=wp)
            o = oracle_engine(variant, 64, 48)
            o.set(black_point=bp, white_point=wp)
            oras.append(o)
        b.commit_monitors()
        img = S.nes_image(seed=4)
        dimg = torch.from_numpy(img.astype(np.int16))
        for it in range((len(COLOURS) + n - 1) // n):
            for i in range(n):
                kw = _settings(variant, it, i, n)
                b.set_source(i, dimg, **kw)
                b.sources[i].reinit = int(it == 0)
                oras[i].modulate(img, field_initialized=int(it != 0), **kw)
            b.modulate()
            for i in range(n):
                got = b.signal(i, "analog")
                assert np.array_equal(got, oras[i].analog), (variant, it, i, S.diff_report("analog", got, oras[i].analog))
        b.close()

    @pytest.mark.parametrize("variant", BORDER_VARIANTS)
    def test_dropin(self, variant):
        check_dropin(variant, fields=4)

    @pytest.mark.parametrize("variant", BORDER_VARIANTS)
    def test_frames_host(self, variant, monkeypatch):
        monkeypatch.setenv("SIMT_HOST_MAPPED", "1")  # (only the interpreter build of the library reads this)
        check_frames_host(variant, n=2, fields=3)

    def test_line_blocks(self):
        check_line_blocks("nes_border", outw=320, outh=240, fields=3)

    def test_stock_nes_ignores_border_color(self):
        check_stock_ignores_the_border(fields=2)
