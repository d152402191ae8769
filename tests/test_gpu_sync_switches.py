"""The decoder with its sync searches off: the libraries built with CRT_DO_VSYNC 0 and / or CRT_DO_HSYNC 0
(crt_core.h:71-72; capi.SYNC_VARIANTS).  With the vsync search off the field is taken from analog[] before any noise
and the lines are decoded from vsync -3 (crt_core.c:323-342); with the hsync search off hsync is 0 after every decoded
line (crt_core.c:446-450).  Every field is compared bit for bit with the CPU model of the switches (tests/sync_oracle.py,
the stock oracle with its own sync pass) and, where it is built, with the reference compiled with the switches off
(oracle/_ref/libref_*_no*sync.so, oracle/Makefile): mixed batches with noise up to 255, geometries on k_lines2 and on
k_lines, the generic equaliser and poked sync states; the drop-in interface; crtx_frames_host; a line-block split; the
reference's unmodified crt_main.c and extra/video_convert.c linked against the libraries.

The same bodies run on the CPU through the SIMT interpreter (TestOnTheInterpreter, below)."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import support as S
from ntsc_crt_b200 import capi, layout
from test_simt_kernels import simt_libs  # noqa: F401  (session fixture of the interpreter builds)
import test_simt_kernels as _simt

NOISES = (0, 12, 60, 255)
# poked (vsync, hsync) pairs, each set on some monitors before a field
POKES = ((130, 700), (-50, -50), (700, 130))


def libc_srand(seed):
    libc = C.CDLL(None)
    libc.srand.argtypes = [C.c_uint]
    libc.srand(seed)


def is_nes(variant):
    return layout.system_spec(variant).system == layout.SYS_NES


def source(variant, it, i=0, seed=0, aberration=False):
    """(numpy image, settings) of field `it` for monitor `i`: NES pixels or an RGB picture (pictures stay inside the
    field: yoffset <= 2).  aberration: VHS with do_aberration on every other field (on monitors with blend 0)"""
    if is_nes(variant):
        return S.nes_image(seed=300 + seed + i, rainbow=(i % 3 == 2)), dict(dot_crawl_offset=(i + it) % 3,
                                                                             hue=(37 * i + 11 * it) % 360,
                                                                             xoffset=4 * ((i + it) % 4), yoffset=(i + it) % 3)
    img = S.bars_image(320, 240) if (i + seed) % 2 else S.rand_image(256, 224, seed=70 + seed + i)
    kw = dict(format=layout.PIX_BGRA, as_color=int((i + it) % 4 != 3), field=it & 1, frame=(it >> 1) & 1, raw=0,
              hue=(37 * i + 11 * it) % 360, xoffset=4 * ((i + it) % 4), yoffset=(i + it) % 3)
    if layout.system_spec(variant).system == layout.SYS_VHS:
        kw["do_aberration"] = int(aberration and (i + it) % 2 == 0)
    return img, kw


def poke(rig, i, vsync, hsync):
    """set monitor i's vsync / hsync on both sides of a BatchRig (the rest of its state kept)"""
    st = rig.b.get_state(first=i, count=1)
    st[0].vsync, st[0].hsync = vsync, hsync
    rig.b.set_state(st, first=i)
    rig.oras[i].set(vsync=vsync, hsync=hsync)


def check_properties(variant, b, n):
    """what the switches promise: vsync -3 after every demodulate without the vsync search, hsync 0 on every decoded
    line without the hsync search"""
    spec = layout.system_spec(variant)
    states = b.get_state()
    for i in range(n):
        if not spec.do_vsync:
            assert states[i].vsync == -3, (variant, i, states[i].vsync)
        if not spec.do_hsync:
            lines = [l for l in b.get_lines(i) if l.beg >= 0]
            assert lines and all(l.hsync == 0 for l in lines), (variant, i)


def check_batch(variant, generic=0, fields=8, big=(832, 624), small=(400, 300), per_group=3):
    """`per_group` monitors on a geometry k_lines2 takes and as many on one it does not, noise 0 .. 255, knobs, VHS
    aberrations; vsync / hsync poked on some monitors before fields 2, 4 and 6; the whole state of every monitor after
    every field, against the CPU model and, where it is built, the reference with the switches off (each monitor's
    calls replayed on its own reference instance).  The two groups are demodulated one after the other so that each
    one's line kernel is seen."""
    mons = []
    for i in range(2 * per_group):
        w, h = big if i < per_group else small
        fmt = layout.PIX_BGRA if i < per_group else layout.PIX_RGB
        knobs = dict(blend=1, scanlines=1) if i < per_group else dict(blend=0, scanlines=1, hue=-20 + 15 * i, saturation=14,
                                                                      black_point=3, white_point=90, v_fac=3 * (i % 2))
        m = dict(outw=w, outh=h, fmt=fmt, noise=(NOISES + (100, 33))[i % 6], knobs=knobs)
        if layout.system_spec(variant).system == layout.SYS_VHS:
            m["seed"] = 100 + i
        mons.append(m)
    rig = S.BatchRig(variant, mons, options=(("generic_eq", generic),))
    imgs = [source(variant, 0, i)[0] for i in range(len(mons))]
    calls = [[] for _ in mons]  # per monitor and field: (poked (vsync, hsync) or None, settings, batch state after it)
    for it in range(fields):
        poked = {}
        if it in (2, 4, 6):
            vs, hs = POKES[it // 2 - 1]
            for i in range(it // 2 - 1, len(mons), 2):
                poke(rig, i, vs, hs)
                poked[i] = (vs, hs)
        for i in range(len(mons)):
            kw = source(variant, it, i, aberration=not mons[i]["knobs"]["blend"])[1]
            if is_nes(variant):
                kw["reinit"] = int(it == 0)
            rig.source(i, imgs[i], **kw)
        rig.modulate()
        before = rig.b.lines2_launches
        rig.demodulate(first=0, count=per_group)
        took_big = rig.b.lines2_launches - before
        rig.demodulate(first=per_group, count=per_group)
        took_small = rig.b.lines2_launches - before - took_big
        assert took_big > 0 and took_small == 0, (variant, it, took_big, took_small)
        rig.check("%s generic_eq %d field %d" % (variant, generic, it))
        check_properties(variant, rig.b, len(mons))
        for i in range(len(mons)):
            calls[i].append((poked.get(i), dict(rig._src[i][1]), S.monitor_state(rig.b, i, rig.outs[i])))
    rig.close()
    if not S.have_ref(variant):
        return
    for i, m in enumerate(mons):  # (one at a time: the VHS builds share the process's libc rand())
        ref = S.RefEngine(variant, m["outw"], m["outh"], m["fmt"], seed=m.get("seed", 1))
        ref.set(**m["knobs"])
        for it, (pk, kw, st) in enumerate(calls[i]):
            if pk:
                ref.set(vsync=pk[0], hsync=pk[1])
            ref.modulate(imgs[i], **kw)
            ref.demodulate(m["noise"])
            S.assert_same_state(st, dict(ref.state()), "%s generic_eq %d field %d monitor %d [batch vs reference]" % (
                variant, generic, it, i))


def check_dropin(variant, outw=832, outh=624, fields=8):
    """the drop-in interface after every call, against the CPU model; then the reference with the switches off, where it
    is built, through the same calls (VHS: libc rand() seeded alike for each)"""
    calls = []
    for it in range(fields):
        img, kw = source(variant, it, it % 2, seed=5)
        calls.append((POKES[it // 2 - 1] if it in (2, 4, 6) else None, img, kw, NOISES[it % 4] if it < 4 else (100, 255, 33, 60)[it % 4]))
    gpu, ora = S.ProductEngine(variant, outw, outh), S.oracle_engine(variant, outw, outh)
    libc_srand(1)
    got = []
    for e in (gpu, ora):
        e.set(blend=1, scanlines=1, hue=10)
    for it, (pk, img, kw, noise) in enumerate(calls):
        for e in (gpu, ora):
            if pk:
                e.set(vsync=pk[0], hsync=pk[1])
            e.modulate(img, **kw)
        S.assert_same_state(gpu.state(), ora.state(), "%s drop-in mod %d" % (variant, it))
        for e in (gpu, ora):
            e.demodulate(noise)
        S.assert_same_state(gpu.state(), ora.state(), "%s drop-in demod %d" % (variant, it))
        got.append(gpu.state())
    if not S.have_ref(variant):
        return
    ref = S.RefEngine(variant, outw, outh, seed=1)
    ref.set(blend=1, scanlines=1, hue=10)
    for it, (pk, img, kw, noise) in enumerate(calls):
        if pk:
            ref.set(vsync=pk[0], hsync=pk[1])
        ref.modulate(img, **kw)
        ref.demodulate(noise)
        S.assert_same_state(got[it], dict(ref.state()), "%s drop-in call %d [gpu vs reference]" % (variant, it))


def check_frames_host(variant, n=3, fields=4, outw=640, outh=480):
    """crtx_frames_host: host source images in, host images out; the whole state, and the rows the fields write in the
    host images, equal the CPU model's"""
    import torch
    mons = [dict(outw=outw, outh=outh, fmt=layout.PIX_BGRA, noise=(60, 255, 12)[i % 3],
                 knobs=dict(blend=1, scanlines=1, black_point=i, white_point=100 - 5 * i)) for i in range(n)]
    if layout.system_spec(variant).system == layout.SYS_VHS:
        for i, m in enumerate(mons):
            m["seed"] = 7 + i
    rig = S.BatchRig(variant, mons)
    host = [torch.zeros(outh, outw, 4, dtype=torch.uint8).pin_memory() for _ in range(n)]
    srcs = []
    for i in range(n):
        img = source(variant, 0, i, seed=9)[0]
        t = torch.from_numpy(img.astype(np.int16) if img.dtype == np.uint16 else img).pin_memory()
        srcs.append(t.numpy().view(np.uint16) if img.dtype == np.uint16 else t.numpy())  # (the page-locked images)
    for it in range(fields):
        for i in range(n):
            kw = source(variant, it, i, seed=9)[1]
            if is_nes(variant):
                kw["reinit"] = int(it == 0)
            rig.source(i, srcs[i], **kw)
        rig.frames_host([h.data_ptr() for h in host])
        rig.check("%s frames_host field %d" % (variant, it))
        for i in range(n):
            got, want = host[i].numpy(), rig.oras[i].out
            rows = S.written_rows(rig.b.get_lines(i), outh, 1)
            assert rows.any()
            assert np.array_equal(got[rows], want[rows]), (variant, it, i, S.diff_report("rows", got[rows], want[rows]))
    rig.close()


def check_line_blocks(variant, outw=832, outh=624, fields=5):
    """two contexts each decode their own block of lines (support.decode_in_blocks) at noise 60"""
    def field(it):
        img, kw = source(variant, it, 1, seed=3)
        return img, dict(kw, reinit=int(it == 0))
    S.decode_in_blocks(variant, outw, outh, 2, field, fields=fields, noise=60)


def check_video(noise=100, n=23, segments=5, outw=640, outh=480):
    """VideoConverter on ntsc_nosync: bit-identical to the sequential loop on the CPU model, and no segment recomputed
    (the sync state is a constant, so the speculation always holds)"""
    import torch
    from ntsc_crt_b200 import video
    frames = S.moving_bars(n, 320, 240)
    ora = S.oracle_engine("ntsc_nosync", outw, outh)
    ora.set(blend=0, scanlines=1, saturation=10)
    want = []
    for f in range(n):
        field, frame = video.frame_parity(f)
        ora.modulate(frames[f], format=layout.PIX_BGRA, as_color=1, field=field, frame=frame)
        ora.demodulate(noise)
        want.append(ora.out.copy())
    vc = video.VideoConverter("ntsc_nosync", outw, outh, noise=noise, scanlines=1, segments=segments)
    got = vc.convert(torch.from_numpy(frames).cuda()).cpu().numpy()
    vc.close()
    for f in range(n):
        assert np.array_equal(got[f], want[f]), "frame %d (recomputed segments: %d)" % (f, vc.recomputed)
    assert vc.recomputed == 0


@pytest.mark.gpu
@pytest.mark.parametrize("generic", [0, 1], ids=["fast_eq", "generic_eq"])
@pytest.mark.parametrize("variant", capi.SYNC_VARIANTS)
def test_batch_noise_geometries_and_poked_states(variant, generic):
    check_batch(variant, generic)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", capi.SYNC_VARIANTS)
def test_dropin(variant):
    check_dropin(variant)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", capi.SYNC_VARIANTS)
def test_frames_host(variant):
    check_frames_host(variant)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", capi.SYNC_VARIANTS)
def test_line_blocks(variant):
    check_line_blocks(variant)


@pytest.mark.gpu
def test_video_converter_never_recomputes():
    check_video()


@pytest.mark.gpu
def test_vhs_nosync_launches_what_vhs_launches():
    """the same fields on a vhs and a vhs_nosync batch (aberrations, both line kernels) count the same kernel launches:
    the switches change what k_sync computes, not what runs"""
    import torch
    counts = {}
    for variant in ("vhs", "vhs_nosync"):
        b = capi.Batch(variant, 2)
        outs = [torch.zeros(h, w, 4, dtype=torch.uint8, device="cuda") for w, h in ((832, 624), (400, 300))]
        for i in range(2):
            b.set_monitor(i, outs[i], fmt=layout.PIX_BGRA, noise=30, blend=1 - i, scanlines=1)
        b.commit_monitors()
        b.seed(5, first=0, count=2)
        img = torch.from_numpy(S.rand_image(256, 224, seed=4)).cuda()
        seen = []
        for it in range(4):
            for i in range(2):
                b.set_source(i, img, format=layout.PIX_BGRA, as_color=1, field=it & 1, do_aberration=int(i == 1 and it % 2 == 0))
            before = b.launches
            b.modulate()
            b.demodulate()
            seen.append(b.launches - before)
        torch.cuda.synchronize()
        counts[variant] = seen
        b.close()
    assert counts["vhs"] == counts["vhs_nosync"], counts


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["ntsc_nosync", "vhs_nosync"])
@pytest.mark.parametrize("flags,noise,hue", [("-o", 200, 0), ("-op", 60, 0), ("-om", 255, 30), ("-opa", 12, 0)])
def test_unmodified_cli_driver(tmp_path, variant, flags, noise, hue):
    """crt_main.c, unchanged, compiled with -DCRT_DO_VSYNC=0 -DCRT_DO_HSYNC=0 against our header and linked with
    libcrt_b200_<system>_nosync.so, writes the bytes of the reference build with the switches off.  (VHS draws its
    noise from libc rand(), never seeded by the driver: the same stream in both builds.)"""
    ref_cli, b200_cli = (os.path.join(S.REF_DIR, "cli_%s_%s" % (k, variant)) for k in ("ref", "b200"))
    if not (os.path.exists(ref_cli) and os.path.exists(b200_cli)):
        pytest.skip("driver binaries not built")
    rgb = S.bars_image(320, 240, fmt=layout.PIX_RGB)[..., :3].copy()
    src = tmp_path / "in.ppm"
    S.write_ppm(str(src), rgb)
    outs = []
    for exe, name in ((ref_cli, "ref.ppm"), (b200_cli, "b200.ppm")):
        out = tmp_path / name
        subprocess.run([exe, flags, "832", "624", str(noise), str(hue), str(src), str(out)],
                       check=True, stdout=subprocess.DEVNULL, timeout=300)
        outs.append(open(out, "rb").read())
    assert len(outs[0]) > 1000
    assert outs[0] == outs[1]


@pytest.mark.gpu
@pytest.mark.parametrize("flags,noise", [("-o", 100), ("-osp", 255)])
def test_unmodified_video_convert(tmp_path, flags, noise):
    """extra/video_convert.c, unchanged, against libcrt_b200_ntsc_nosync.so writes the bytes of the reference build with
    the switches off"""
    ref_exe, b200_exe = (os.path.join(S.REF_DIR, "video_%s_ntsc_nosync" % k) for k in ("ref", "b200"))
    if not (os.path.exists(ref_exe) and os.path.exists(b200_exe)):
        pytest.skip("video drivers not built")
    frames = S.moving_bars(8, 320, 240, seed=6)
    ref = S.run_video_convert(ref_exe, str(tmp_path / "ref"), frames, flags, 640, 480, noise)
    got = S.run_video_convert(b200_exe, str(tmp_path / "b200"), frames, flags, 640, 480, noise)
    for k, (a, b) in enumerate(zip(got, ref)):
        assert a == b, "output/%06d.bmp differs from the reference build's" % (k + 1)
    shutil.rmtree(str(tmp_path / "ref"))
    shutil.rmtree(str(tmp_path / "b200"))


# ---- the same bodies on the CPU, through the SIMT interpreter ------------------------------------------------------
class TestOnTheInterpreter:
    simt_backend = staticmethod(_simt.simt_backend)  # autouse within this class: the interpreter builds, host "device" tensors

    @pytest.mark.parametrize("variant", capi.SYNC_VARIANTS)
    def test_batch(self, variant):
        check_batch(variant, fields=4, big=(528, 400), small=(320, 240), per_group=2)

    def test_batch_generic_eq(self):
        check_batch("ntsc_nosync", generic=1, fields=3, big=(528, 400), small=(320, 240), per_group=1)

    @pytest.mark.parametrize("variant", capi.SYNC_VARIANTS)
    def test_dropin(self, variant):
        check_dropin(variant, outw=320, outh=240, fields=4)

    @pytest.mark.parametrize("variant", ["ntsc_nosync", "nes_nosync"])
    def test_frames_host(self, variant, monkeypatch):
        monkeypatch.setenv("SIMT_HOST_MAPPED", "1")  # (only the interpreter build of the library reads this)
        check_frames_host(variant, n=2, fields=3, outw=320, outh=240)

    def test_line_blocks(self):
        check_line_blocks("ntsc_nohsync", outw=320, outh=240, fields=3)

    def test_video_converter_never_recomputes(self):
        check_video(n=9, segments=3, outw=320, outh=240)
