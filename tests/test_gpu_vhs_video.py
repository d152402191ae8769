"""The VHS build's rand() replica as a saveable state, and the time-parallel video path on the VHS build.

crtx_get_rand / crtx_set_rand expose each monitor's generator (glibc TYPE_3: the last 31 raw values, oldest first), and
crtx_skip_fields advances it by whole fields without running them (k_vhs_skip, crt_vhs.cuh).  A field's draw count
depends on its own draws only, so skipping k fields must leave exactly the state k real fields leave, whatever their
images, pixel formats, noise and knobs.  VideoConverter("vhs") builds on that: every segment's generator is made exact
from the seed, so the sequence must come out bit-identical to srand(seed) followed by video_convert.c's loop.

The check_* functions take their sizes as arguments: tests/test_vhs_video_logic.py runs the same checks, smaller, on the
SIMT interpreter's build of the library.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import support as S
import test_gpu_vhs as V
from ntsc_crt_b200 import capi, layout

pytestmark = pytest.mark.gpu

SKIPS = (0, 1, 2, 3, 8, 17)


def oracle_words(ora):
    """an OracleEngine's generator in the public order: chronological, oldest first (its ring starts at index f)"""
    r = ora.rand
    return np.array([r.r[(r.f + j) % 31] for j in range(31)], dtype=np.uint32)


def set_oracle_words(ora, words):
    for j in range(31):
        ora.rand.r[j] = int(words[j])
    ora.rand.f, ora.rand.b = 0, 28


def seeded_words(seed):
    o = S.oracle_lib()
    g = S._ORand()
    o.ocrt_rand_seed(C.byref(g), seed)
    return np.array([g.r[(g.f + j) % 31] for j in range(31)], dtype=np.uint32)


def device(img):
    import torch
    return torch.from_numpy(img).cuda()


def check_seed_words(seeds):
    """1. after crtx_seed, get_rand equals the oracle's ocrt_rand_seed state, oldest word first"""
    b = capi.Batch("vhs", len(seeds))
    for i, s in enumerate(seeds):
        b.seed(s, first=i, count=1)
    got = b.get_rand()
    b.close()
    for i, s in enumerate(seeds):
        assert np.array_equal(got[i], seeded_words(s)), "seed %d" % s


def check_set_get_roundtrip(n=7, first=2, count=3):
    """2. set_rand then get_rand on a subrange; the monitors outside it keep their words"""
    rng = np.random.default_rng(5)
    b = capi.Batch("vhs", n)
    for i in range(n):
        b.seed(1000 + i, first=i, count=1)
    before = b.get_rand()
    words = rng.integers(0, 1 << 32, size=(count, 31), dtype=np.uint64).astype(np.uint32)
    b.set_rand(words, first=first)
    after = b.get_rand()
    b.close()
    assert np.array_equal(after[first:first + count], words)
    keep = [i for i in range(n) if not first <= i < first + count]
    assert np.array_equal(after[keep], before[keep])


def random_field(rng, case):
    """one field's source and settings the way test_gpu_vhs draws them, with a known pixel format"""
    kw, _ = V.draw_call(rng, case)
    kw["format"] = case["pack"]
    kw["do_aberration"] = case["ab"]
    return kw


def check_skip_equals_real_fields(seeds, skips, aberrations=(0, 1)):
    """3. monitor 0 runs k real fields (random images, pixel formats, noise and knobs), monitor 1 skips k: same generator,
    equal to the oracle's after the same k fields; then one more real field on both gives the same images and states"""
    rng = np.random.default_rng(11)
    for seed in seeds:
        for ab in aberrations:
            for k in skips:
                case = V.draw_case(rng)
                case["ab"] = ab
                noise = V.draw_noise(rng, loud=True)
                knobs = dict(case["knobs"], blend=0 if (ab or abs(noise) > 255) else case["knobs"]["blend"])
                mon = dict(outw=case["outw"], outh=case["outh"], fmt=case["fmt"] if layout.bpp4fmt(case["fmt"]) else layout.PIX_BGRA,
                           noise=noise, knobs=knobs, seed=seed)
                what = "seed %d aberration %d k %d noise %d %r" % (seed, ab, k, noise, mon)
                rig = S.BatchRig("vhs", [dict(mon), dict(mon)])
                img = device(case["img"])
                for f in range(k):
                    kw = random_field(rng, case)
                    rig.b.set_source(0, img, **kw)
                    rig.b.modulate(first=0, count=1)
                    rig.b.demodulate(first=0, count=1)
                    rig.oras[0].modulate(case["img"], **kw)
                    rig.oras[0].demodulate(noise)
                rig.b.skip_fields([k], ab, first=1)
                words = rig.b.get_rand()
                assert np.array_equal(words[0], oracle_words(rig.oras[0])), "real fields vs oracle: " + what
                assert np.array_equal(words[1], words[0]), "skipped vs real fields: " + what
                # the same starting point for one more real field: monitor 1 takes monitor 0's image, sync state and
                # analog[] (a modulate leaves the samples around a smaller or shifted picture as earlier fields wrote them)
                rig.outs[1].copy_(rig.outs[0])
                rig.b.set_state(rig.b.get_state(first=0, count=1), first=1)
                rig.b.write_signal(1, rig.b.signal(0, "analog"), "analog")
                kw = random_field(rng, case)
                for i in (0, 1):
                    rig.b.set_source(i, img, **kw)
                rig.b.modulate()
                rig.b.demodulate()
                S.assert_same_state(S.monitor_state(rig.b, 0, rig.outs[0]), S.monitor_state(rig.b, 1, rig.outs[1]),
                                    "the field after: " + what)
                words = rig.b.get_rand()
                assert np.array_equal(words[0], words[1]), "the field after: " + what
                rig.close()


def check_field_from_set_state(n_states):
    """4. after set_rand to an arbitrary state, one field equals the oracle's run from that state (pins the word order)"""
    rng = np.random.default_rng(12)
    for it in range(n_states):
        words = rng.integers(0, 1 << 32, size=31, dtype=np.uint64).astype(np.uint32)
        mon = dict(outw=320, outh=240, fmt=layout.PIX_BGRA, noise=24, knobs=dict(blend=0, scanlines=1))
        rig = S.BatchRig("vhs", [mon])
        rig.b.set_rand(words[None, :], first=0)
        set_oracle_words(rig.oras[0], words)
        img = S.rand_image(320, 240, seed=it)
        rig.source(0, img, format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=0, do_aberration=it & 1)
        rig.modulate()
        rig.demodulate()
        rig.check("state %d" % it)
        assert np.array_equal(rig.b.get_rand()[0], oracle_words(rig.oras[0])), "state %d" % it
        rig.close()


def test_seed_words():
    check_seed_words(V.SEEDS)


def test_set_get_roundtrip():
    check_set_get_roundtrip()


def test_skip_equals_real_fields():
    check_skip_equals_real_fields(V.SEEDS[:3] + (123456789,), SKIPS)


def test_field_from_set_state():
    check_field_from_set_state(4)


def test_skip_rejects_negative_counts_and_leaves_the_context():
    b = capi.Batch("vhs", 3)
    b.seed(7)
    before = b.get_rand()
    with pytest.raises(capi.CrtxError, match="negative field count"):
        b.skip_fields([2, -1, 0])
    assert np.array_equal(b.get_rand(), before)
    b.close()


def test_other_builds_have_no_generator():
    b = capi.Batch("ntsc", 2)
    for call in (lambda: b.get_rand(), lambda: b.set_rand(np.zeros((1, 31), np.uint32)), lambda: b.skip_fields([1])):
        with pytest.raises(capi.CrtxError, match="draws no rand"):
            call()
    b.close()


# ---------------------------------------------------------------------------------------------------------------
# VideoConverter("vhs")
# ---------------------------------------------------------------------------------------------------------------

def sequential_vhs(frames, outw, outh, noise, seed, aberration, as_color=1, progressive=False):
    """srand(seed), then video_convert.c:246-277 with ntsc.do_aberration set, on the oracle; and its final generator"""
    from ntsc_crt_b200 import video
    ora = S.OracleEngine("vhs", outw, outh, seed=seed)
    ora.set(blend=0, scanlines=1, saturation=10)
    want = []
    for f in range(len(frames)):
        field, frame = video.frame_parity(f, progressive)
        ora.modulate(frames[f], format=layout.PIX_BGRA, as_color=as_color, field=field, frame=frame, do_aberration=aberration)
        ora.demodulate(noise)
        want.append(ora.out.copy())
    return np.stack(want), oracle_words(ora)


class WrongHaloSync(capi.Batch):
    """capi.Batch whose first get_state of a multi-monitor batch -- the sync state after the halo -- reports every
    segment's vsync off by one, so that verification repairs every segment that has a predecessor"""
    def __init__(self, variant, n):
        super().__init__(variant, n)
        self._lied = n == 1

    def get_state(self, first=0, count=None, stream=0):
        st = super().get_state(first, count, stream)
        if not self._lied:
            self._lied = True
            for x in st:
                x.vsync += 1
        return st


VIDEO_CASES = [  # noise, aberration, segments, as_color, progressive
    (0, 0, 1, 1, False), (24, 1, 4, 1, False), (24, 0, 23, 0, False), (0, 1, 4, 0, True), (24, 1, 23, 1, True),
    (0, 1, 23, 1, False), (24, 0, 4, 1, True), (0, 0, 4, 0, False), (24, 1, 1, 0, False),
]


@pytest.mark.parametrize("noise,aberration,segments,as_color,progressive", VIDEO_CASES)
def test_video_converter_matches_sequential_loop(noise, aberration, segments, as_color, progressive):
    check_video(noise, aberration, segments, as_color, progressive)


def test_video_converter_repairs_a_wrong_speculation():
    vc = check_video(24, 1, 4, 1, False, factory=WrongHaloSync)
    assert vc.recomputed == 3


def check_video(noise, aberration, segments, as_color, progressive, factory=None, seed=4242):
    import torch
    from ntsc_crt_b200 import video
    n, w, h = 23, 320, 240
    frames = S.moving_bars(n, w, h)
    want, want_words = sequential_vhs(frames, 640, 480, noise, seed, aberration, as_color, progressive)
    vc = video.VideoConverter("vhs", 640, 480, noise=noise, scanlines=1, as_color=as_color, progressive=progressive,
                              segments=segments, seed=seed, do_aberration=aberration, batch_factory=factory)
    got = vc.convert(torch.from_numpy(frames).cuda()).cpu().numpy()
    for f in range(n):
        assert np.array_equal(got[f], want[f]), "frame %d (recomputed segments: %d)" % (f, vc.recomputed)
    S_ = max(1, min(segments, n))
    b = vc._batch(S_)
    last = S_ - 1  # the last segment ends the sequence: its generator is the sequential loop's final one
    assert np.array_equal(b.get_rand(last, 1)[0], want_words), "final generator state"
    print("noise %d aberration %d segments %d: recomputed %d" % (noise, aberration, segments, vc.recomputed))
    vc.close()
    return vc


# ---------------------------------------------------------------------------------------------------------------
# tools/crtx_video.c linked against the VHS library (bin/crtx_video_vhs)
# ---------------------------------------------------------------------------------------------------------------

DRIVER_VHS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ntsc-crt_b200", "bin", "crtx_video_vhs")


@pytest.mark.skipif(not os.path.exists(DRIVER_VHS), reason="tools/crtx_video_vhs not built")
@pytest.mark.parametrize("flags,noise,segments", [(["-a"], 24, 5), (["-s"], 0, 4), (["-m", "-a", "-s"], 24, 23), (["-p"], 0, 1),
                                                  (["-p", "-a"], 24, 6)])
def test_vhs_video_driver_writes_the_sequential_loops_images(tmp_path, flags, noise, segments):
    n, w, h, seed = 23, 320, 240, 31337
    frames = S.moving_bars(n, w, h)
    os.mkdir(tmp_path / "frames")
    os.mkdir(tmp_path / "output")
    for k in range(n):
        S.write_bmp(str(tmp_path / "frames" / ("%06d.bmp" % (k + 1))), frames[k], 24)
    res = subprocess.run([DRIVER_VHS] + flags + ["-R", str(seed), "-S", str(segments), str(n + 1), "640", "480", str(noise)],
                         cwd=str(tmp_path), stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=300)
    assert res.returncode == 0, res.stderr.decode()
    assert ("rand() seed %d" % seed).encode() in res.stdout
    ora = S.OracleEngine("vhs", 640, 480, seed=seed)
    ora.set(blend=0, scanlines=0 if "-s" in flags else 1, saturation=10)
    progressive = "-p" in flags
    for k in range(n):
        field, frame = (0, 0) if progressive else (k & 1, (k >> 1) & 1)
        ora.modulate(frames[k], format=layout.PIX_BGRA, as_color=0 if "-m" in flags else 1, field=field, frame=frame,
                     do_aberration=int("-a" in flags))
        ora.demodulate(noise)
        got = S.read_bmp32(str(tmp_path / "output" / ("%06d.bmp" % (k + 1))))
        assert np.array_equal(got, ora.out), "image %d: %s\n%s" % (k + 1, S.diff_report("image", got, ora.out),
                                                                   res.stdout.decode()[-300:])
    print(res.stdout.decode().splitlines()[-1])
