"""The VHS build across its input space: the drop-in interface against the oracle on random cases, and the batch
interface's device replica of glibc's rand() over many generator states, subranges, re-seeding and unknown formats.

VHS is the one build whose output depends on a random stream.  The drop-in draws it on the host from libc rand(); the
batch interface keeps one replica of glibc's generator per monitor (crtx_seed) and runs it on the device in k_noise_vhs
(crt_vhs.cuh): jump-ahead matrices for the bulk of the field and a walk for the last lines, where a sample takes 2 or
3 draws depending on the data.  A wrong draw count can heal within the field (a stream shifted by one draw re-merges in
that walk), so every test here compares the whole state after every call, not only at the end.  The random cases are
drawn by draw_case / draw_call, which tests/test_oracle_vhs.py shares to pin the oracle to the reference on them.
"""
import ctypes as C

import numpy as np
import pytest

import support as S
from ntsc_crt_b200 import layout

pytestmark = pytest.mark.gpu

SPEC = layout.system_spec("vhs")
MAXH = (SPEC.lines * 64500) >> 16  # the picture height of a scaled source (crt_ntscvhs.c:163-172)
NOISES = (0, 3, 12, 24, 40, 255)
LOUD_NOISES = (1000, 70000, 1 << 20, 1 << 23)  # |noise| <= 2^23: the reference's (rand term) * noise stays within int
SEEDS = (0, 1, 42, (1 << 31) - 1, 1 << 31, 0xFFFFFFFF)
UNKNOWN_FORMATS = (-1, 6, 9)

# sizes of the runs below (the interpreter suite, tests/test_simt_kernels.py, runs smaller ones)
SWEEP_CASES = 4
SWEEP_CALLS = 3
BATCH = 32
FIELDS = 8


def source_row_max(h, raw, field):
    """the last source row the encoder reads for a source of height h, before its clamp to h (crt_ntscvhs.c:265-270)"""
    desth = min(h, MAXH) if raw else MAXH
    return (desth - 1) * h // desth + (field * h + desth) // desth // 2


def draw_noise(rng, loud=False):
    mag = int(rng.choice(LOUD_NOISES)) if loud and rng.random() < 0.5 else int(rng.choice(NOISES))
    return -mag if rng.random() < 0.3 else mag


def draw_case(rng):
    """output geometry and format, monitor knobs (15% of them far out), whether the fields draw an aberration or loud
    noise (both with blend 0: see tests/test_oracle_vhs.py), the generator's seed and the source image"""
    fmt = int(rng.integers(0, 6))
    outw = int(rng.choice([64, 97, 256, 320, 333, 400, 512, 640, 641, 832, 1024, 1280, 1921]))
    outh = int(rng.choice([31, 80, 224, 240, 241, 300, 448, 480, 624, 720, 1081]))
    knobs = dict(blend=int(rng.integers(0, 2)), scanlines=int(rng.integers(0, 2)),
                 hue=int(rng.integers(-400, 400)), brightness=int(rng.integers(-60, 60)),
                 contrast=int(rng.integers(60, 320)), saturation=int(rng.integers(0, 40)),
                 black_point=int(rng.integers(-10, 20)), white_point=int(rng.integers(50, 130)))
    if rng.random() < 0.15:  # far outside the packed path's exact range
        knobs.update(saturation=int(rng.integers(300, 5000)), brightness=int(rng.integers(-6000, 6000)),
                     contrast=int(rng.integers(300, 1200)))
    aberration = bool(rng.random() < 0.4)
    loud = bool(rng.random() < 0.3)
    if aberration or loud:
        knobs["blend"] = 0
    seed = int(rng.choice(SEEDS)) if rng.random() < 0.5 else int(rng.integers(0, 1 << 32, dtype=np.uint64))
    w, h = int(rng.integers(40, 900)), int(rng.integers(40, 700))
    pack = int(rng.integers(0, 6))
    img = S.pack_rgb(S.rand_image(w, h, bpp=3, seed=int(rng.integers(0, 1 << 30))), pack)
    return dict(fmt=fmt, outw=outw, outh=outh, knobs=knobs, aberration=aberration, loud=loud, seed=seed, img=img, pack=pack)


def draw_call(rng, case):
    """(modulate settings, demodulate noise) of one field of a case"""
    h = case["img"].shape[0]
    raw, field = int(rng.integers(0, 2)), int(rng.integers(0, 2))
    if source_row_max(h, raw, field) >= h:
        field = 0  # field 1 would read row h, one past the image (crt_ntscvhs.c:270); field 0 never does
    assert source_row_max(h, raw, field) < h
    src_fmt = case["pack"] if rng.random() >= 0.1 else int(rng.choice(UNKNOWN_FORMATS))
    kw = dict(format=src_fmt, as_color=int(rng.integers(0, 2)), field=field, frame=int(rng.integers(0, 2)), raw=raw,
              hue=int(rng.integers(0, 360)), xoffset=int(rng.integers(0, 16)), yoffset=int(rng.integers(0, 3)),
              do_aberration=int(case["aberration"] and rng.random() < 0.7))
    return kw, draw_noise(rng, case["loud"])


def libc_srand(seed):
    libc = C.CDLL(None)
    libc.srand.argtypes = [C.c_uint]
    libc.srand(seed)


@pytest.mark.parametrize("seed", [1, 2, 3, 4, 5, 6])
def test_dropin_random_cases(seed):
    """the drop-in (host libc rand()) against the oracle (its own replica, same seed) after every call"""
    rng = np.random.default_rng(3000 + seed)
    for case in range(SWEEP_CASES):
        c = draw_case(rng)
        gpu = S.ProductEngine("vhs", c["outw"], c["outh"], c["fmt"])
        ora = S.OracleEngine("vhs", c["outw"], c["outh"], c["fmt"], seed=c["seed"])
        libc_srand(c["seed"])
        for e in (gpu, ora):
            e.set(**c["knobs"])
        for call in range(SWEEP_CALLS):
            kw, noise = draw_call(rng, c)
            what = "seed %d case %d call %d: %dx%d fmt %d knobs %r src %r %r noise %d rand seed %d" % (
                seed, case, call, c["outw"], c["outh"], c["fmt"], c["knobs"], c["img"].shape, kw, noise, c["seed"])
            for e in (gpu, ora):
                e.modulate(c["img"], **kw)
            S.assert_same_state(gpu.state(), ora.state(), "modulate " + what)
            for e in (gpu, ora):
                e.demodulate(noise)
            S.assert_same_state(gpu.state(), ora.state(), "demodulate " + what)


# ----------------------------------------------------------------------------------
# the batch interface
# ----------------------------------------------------------------------------------

def seed_oracle(ora, seed):
    ora.lib.ocrt_rand_seed(C.byref(ora.rand), seed)


class Rig:
    """a VHS batch and one oracle per monitor, driven through the same calls; mons[i] = dict(seed, noise, fmt, outw,
    outh, knobs)"""

    def __init__(self, mons):
        import torch
        from ntsc_crt_b200 import capi
        self.mons = mons
        self.b = capi.Batch("vhs", len(mons))
        self.outs, self.oras, self._dev = [], [], {}
        for i, m in enumerate(mons):
            out = torch.zeros(m["outh"], m["outw"], max(1, layout.bpp4fmt(m["fmt"])), dtype=torch.uint8, device="cuda")
            self.b.set_monitor(i, out, fmt=m["fmt"], noise=m["noise"], **m["knobs"])
            self.b.seed(m["seed"], first=i, count=1)
            o = S.OracleEngine("vhs", m["outw"], m["outh"], m["fmt"], seed=m["seed"])
            o.set(**m["knobs"])
            self.outs.append(out)
            self.oras.append(o)
        self.b.commit_monitors()

    def device(self, img):
        import torch
        if id(img) not in self._dev:
            self._dev[id(img)] = (img, torch.from_numpy(img).cuda())
        return self._dev[id(img)][1]

    def seed(self, seed, first, count):
        self.b.seed(seed, first=first, count=count)
        for i in range(first, first + count):
            seed_oracle(self.oras[i], seed)
            self.mons[i]["seed"] = seed

    def modulate(self, calls, first=0, count=None):
        """calls[i] = (image, settings) for the monitors i of [first, first + count)"""
        count = len(self.mons) - first if count is None else count
        for i in range(first, first + count):
            img, kw = calls[i]
            self.b.set_source(i, self.device(img), **kw)
            self.oras[i].modulate(img, **kw)
        self.b.modulate(first=first, count=count)

    def demodulate(self, first=0, count=None):
        count = len(self.mons) - first if count is None else count
        self.b.demodulate(first=first, count=count)
        for i in range(first, first + count):
            self.oras[i].demodulate(self.mons[i]["noise"])

    def frames_host(self, calls, host):
        """crtx_frames_host: modulate from host images, demodulate, copy the images to host[i]"""
        for i, (img, kw) in enumerate(calls):
            s = self.b.sources[i]
            s.data, s.h, s.w, s.pitch = img.ctypes.data, img.shape[0], img.shape[1], 0
            for k, v in kw.items():
                setattr(s, k, v)
            self.oras[i].modulate(img, **kw)
            self.oras[i].demodulate(self.mons[i]["noise"])
        self.b.frames_host([h.ctypes.data for h in host])

    def check(self, what):
        import torch
        torch.cuda.synchronize()
        st = self.b.get_state()
        for i, o in enumerate(self.oras):
            got = dict(analog=self.b.signal(i, "analog"), inp=self.b.signal(i, "inp"), out=self.outs[i].cpu().numpy(),
                       ccf=np.array([[st[i].ccf[r][x] for x in range(SPEC.cc_samples)] for r in range(SPEC.vper)]),
                       hsync=st[i].hsync, vsync=st[i].vsync, rn=st[i].rn)
            m = self.mons[i]
            S.assert_same_state(got, o.state(), "%s, monitor %d (seed %d, noise %d, out fmt %d)" % (what, i, m["seed"], m["noise"], m["fmt"]))

    def close(self):
        self.b.close()


def field_settings(rng, it, src_fmt=layout.PIX_BGRA, aberration=0):
    return dict(format=src_fmt, as_color=int(rng.integers(0, 2)), field=it & 1, frame=(it >> 1) & 1, raw=0,
                hue=int(rng.integers(0, 360)), xoffset=int(rng.integers(0, 16)), yoffset=int(rng.integers(0, 3)),
                do_aberration=aberration)


def sources(rng, k=3):
    """k source images of different sizes and pixel formats (heights the encoder never reads past: row_max < h)"""
    out = []
    for j in range(k):
        w, h = int(rng.integers(100, 700)), int(rng.integers(240, 500))
        fmt = int(rng.integers(0, 6))
        assert source_row_max(h, 0, 1) < h
        out.append((S.pack_rgb(S.rand_image(w, h, bpp=3, seed=int(rng.integers(0, 1 << 30))), fmt), fmt))
    return out


def test_batch_many_generator_states():
    """BATCH monitors, each with its own seed and noise, FIELDS consecutive fields: every generator state passes through
    k_noise_vhs and k_vhs_commit FIELDS times.  A quarter of the monitors draw an aberration every field (blend 0)."""
    rng = np.random.default_rng(71)
    seeds = list(SEEDS) + [int(s) for s in rng.integers(0, 1 << 32, size=max(0, BATCH - len(SEEDS)), dtype=np.uint64)]
    geometries = [(320, 240, layout.PIX_BGRA), (400, 300, layout.PIX_RGB), (641, 480, layout.PIX_ABGR)]
    mons = []
    for i in range(BATCH):
        aberr = i % 4 == 1
        noise = draw_noise(rng, loud=i % 3 == 2)
        outw, outh, fmt = geometries[i % len(geometries)]
        knobs = dict(blend=0 if aberr else i & 1, scanlines=(i >> 1) & 1, hue=int(rng.integers(-60, 60)),
                     saturation=int(rng.integers(5, 30)))
        mons.append(dict(seed=seeds[i], noise=noise, fmt=fmt, outw=outw, outh=outh, knobs=knobs, aberr=aberr))
    rig = Rig(mons)
    imgs = sources(rng)
    for it in range(FIELDS):
        calls = {}
        for i, m in enumerate(mons):
            img, fmt = imgs[(i + it) % len(imgs)]
            calls[i] = (img, field_settings(rng, it, fmt, int(m["aberr"])))
        rig.modulate(calls)
        rig.check("field %d modulate" % it)
        rig.demodulate()
        rig.check("field %d demodulate" % it)
    rig.close()


def test_batch_subranges_and_reseeding():
    """modulate / demodulate [first, first + count) at several offsets: the monitors outside keep their bytes and their
    generator (their oracles skip the call, and their next field must still match); crtx_seed on a subset mid-run"""
    rng = np.random.default_rng(72)
    n = 6
    mons = [dict(seed=SEEDS[i], noise=(24, 3, 255, 12, 40, 1 << 20)[i], fmt=layout.PIX_BGRA, outw=320, outh=240,
                 knobs=dict(blend=0, scanlines=i & 1)) for i in range(n)]
    rig = Rig(mons)
    imgs = sources(rng, 2)
    # (first, count) of each step; None: re-seed monitors 2 and 3 with a fresh seed before the step
    steps = [(0, n), (1, 3), (0, 1), (n - 2, 2), None, (2, 3), (0, n), (5, 1), (0, n)]
    it = 0
    for step in steps:
        if step is None:
            rig.seed(0xDEADBEEF, first=2, count=2)
            continue
        first, count = step
        calls = {i: (imgs[(i + it) % 2][0], field_settings(rng, it, imgs[(i + it) % 2][1], int(i == 3))) for i in range(first, first + count)}
        rig.modulate(calls, first, count)
        rig.check("step %d [%d, %d) modulate" % (it, first, first + count))
        rig.demodulate(first, count)
        rig.check("step %d [%d, %d) demodulate" % (it, first, first + count))
        it += 1
    rig.close()


def test_batch_unknown_formats():
    """monitors whose source has an unknown format draw no aberration (the encoder returns first: crt_ntscvhs.c:191-193),
    with do_aberration set or not; a monitor whose output format is unknown makes no draws when it demodulates
    (crt_core.c:312-315).  Known and unknown formats alternate, so a stray draw shifts every later field's stream."""
    rng = np.random.default_rng(73)
    n = 6
    # 0, 1: unknown source formats on odd fields, with and without aberration; 2: unknown output format;
    # 3: aberration every field; 4: unknown source format with aberration every third field; 5: plain
    fmts = [layout.PIX_BGRA, layout.PIX_RGB, 9, layout.PIX_BGRA, layout.PIX_ARGB, layout.PIX_BGRA]
    mons = [dict(seed=SEEDS[(i + 1) % len(SEEDS)], noise=(24, 12, 24, 40, 3, 255)[i], fmt=fmts[i], outw=320, outh=240,
                 knobs=dict(blend=0, scanlines=1)) for i in range(n)]
    rig = Rig(mons)
    imgs = sources(rng, 2)
    for it in range(6):
        calls = {}
        for i in range(n):
            img, fmt = imgs[(i + it) % 2]
            unknown, aberr = {0: (it & 1, 1), 1: (it & 1, 0), 2: (0, 1), 3: (0, 1), 4: (it % 3 == 1, 1), 5: (0, 0)}[i]
            calls[i] = (img, field_settings(rng, it, int(rng.choice(UNKNOWN_FORMATS)) if unknown else fmt, aberr))
        rig.modulate(calls)
        rig.check("field %d modulate" % it)
        rig.demodulate()
        rig.check("field %d demodulate" % it)
    rig.close()


def test_frames_host_with_aberration():
    """crtx_frames_host on the VHS build: host images in and out, an aberration on two monitors, one of them with a
    source of unknown format (which must not draw)"""
    rng = np.random.default_rng(74)
    n = 3
    mons = [dict(seed=SEEDS[i + 2], noise=(24, 12, 40)[i], fmt=layout.PIX_BGRA, outw=400, outh=300,
                 knobs=dict(blend=0, scanlines=1)) for i in range(n)]
    rig = Rig(mons)
    imgs = sources(rng, n)
    host = [np.full((300, 400, 4), 0xA5, dtype=np.uint8) for _ in range(n)]
    for it in range(4):
        calls = []
        for i in range(n):
            img, fmt = imgs[i]
            calls.append((img, field_settings(rng, it, 9 if (i == 1 and it % 2 == 0) else fmt, int(i != 2))))
        rig.frames_host(calls, host)
        rig.check("frames_host field %d" % it)
        for i in range(n):
            assert np.array_equal(host[i], rig.oras[i].out), "field %d monitor %d: %s" % (it, i, S.diff_report("host image", host[i], rig.oras[i].out))
    rig.close()


def test_dropin_and_batch_draw_the_same_stream():
    """one call sequence per seed through the drop-in (host libc rand()) and a batch monitor seeded alike (the device
    replica): the same bytes after every call, aberrations and an unknown source format included"""
    rng = np.random.default_rng(75)
    seeds = [1, 0xFFFFFFFF, 123456789]
    noises = [24, -40, 1 << 23]
    mons = [dict(seed=s, noise=noises[i], fmt=layout.PIX_BGRA, outw=400, outh=300, knobs=dict(blend=0, scanlines=1))
            for i, s in enumerate(seeds)]
    rig = Rig(mons)
    imgs = sources(rng, 2)
    fields = []
    for it in range(5):
        fields.append({i: (imgs[(i + it) % 2][0], field_settings(rng, it, 9 if it == 1 else imgs[(i + it) % 2][1], int(it in (1, 2, 4))))
                       for i in range(len(seeds))})
    states = {}
    for it, calls in enumerate(fields):
        rig.modulate(calls)
        rig.demodulate()
        rig.check("field %d" % it)
        st = rig.b.get_state()
        for i in range(len(seeds)):
            states[(i, it)] = dict(analog=rig.b.signal(i, "analog"), inp=rig.b.signal(i, "inp"), out=rig.outs[i].cpu().numpy().copy(),
                                   ccf=np.array([[st[i].ccf[r][x] for x in range(SPEC.cc_samples)] for r in range(SPEC.vper)]),
                                   hsync=st[i].hsync, vsync=st[i].vsync, rn=st[i].rn)
    rig.close()
    for i, s in enumerate(seeds):
        gpu = S.ProductEngine("vhs", 400, 300)
        gpu.set(blend=0, scanlines=1)
        libc_srand(s)
        for it, calls in enumerate(fields):
            img, kw = calls[i]
            gpu.modulate(img, **kw)
            gpu.demodulate(noises[i])
            S.assert_same_state(states[(i, it)], gpu.state(), "seed %d field %d: batch vs drop-in" % (s, it))
