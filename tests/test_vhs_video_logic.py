"""VideoConverter's VHS scheduling on the CPU, and the rand() replica calls on the SIMT interpreter's VHS build.

The first part stands the batch interface in with the oracle (tests/mock_batch.OracleBatch, extended below with the
generator calls): seeding every segment, skipping it to its first decoded frame, saving the generator after the halo
and restoring it on repair, single process and over gloo with 2 and 3 ranks.  Its skip_fields runs real oracle fields
on a blank image, so these runs also check that what a field draws does not depend on the signal.  The result has to
be srand(seed) followed by video_convert.c's loop, image for image.

The second part runs tests/test_gpu_vhs_video.py's checks 1-4 on tests/simt/_build/libcrt_simt_vhs.so, so k_vhs_skip is
exercised here before it runs on a GPU (tests/test_simt_kernels.py does the same for the other GPU tests).
"""
import ctypes as C
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import support as S
from mock_batch import OracleBatch
from ntsc_crt_b200 import capi, layout, sharding, video

HERE = os.path.dirname(os.path.abspath(__file__))
SEED = 977


class VhsOracleBatch(OracleBatch):
    """OracleBatch with the VHS generator calls of capi.Batch"""

    def seed(self, seed, first=0, count=None):
        count = self.n - first if count is None else count
        for i in range(first, first + count):
            self._eng[i].lib.ocrt_rand_seed(C.byref(self._eng[i].rand), seed)

    def get_rand(self, first=0, count=None, stream=0):
        count = self.n - first if count is None else count
        out = np.zeros((count, 31), dtype=np.uint32)
        for k in range(count):
            r = self._eng[first + k].rand
            out[k] = [r.r[(r.f + j) % 31] for j in range(31)]
        return out

    def set_rand(self, words, first=0, stream=0):
        for k, w in enumerate(np.asarray(words, dtype=np.uint32).reshape(-1, 31)):
            r = self._eng[first + k].rand
            for j in range(31):
                r.r[j] = int(w[j])
            r.f, r.b = 0, 28

    def skip_fields(self, fields, do_aberration=0, first=0, stream=0):
        """real oracle fields on a blank image, drawing from the monitor's generator"""
        blank = np.zeros((48, 64, 4), dtype=np.uint8)
        for k, n in enumerate(fields):
            assert n >= 0
            eng = self._eng[first + k]
            scratch = S.OracleEngine(self.variant, 64, 48)
            C.memmove(C.byref(scratch.rand), C.byref(eng.rand), C.sizeof(eng.rand))
            for f in range(n):
                scratch.modulate(blank, format=layout.PIX_BGRA, as_color=1, field=f & 1, frame=0, do_aberration=do_aberration)
                scratch.demodulate(7)
            C.memmove(C.byref(eng.rand), C.byref(scratch.rand), C.sizeof(eng.rand))


class WrongHaloSync(VhsOracleBatch):
    """the first get_state of a multi-monitor batch (the sync state after the halo) reports every vsync off by one"""
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


def make_frames(n, w=160, h=240):
    rng = np.random.default_rng(19)
    base = S.bars_image(w, h)
    out = []
    for k in range(n):
        f = np.roll(base, 7 * k, axis=1).copy()
        if k % 5 == 3:
            f[..., :3] = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        out.append(f)
    return np.stack(out)


def sequential(frames, outw, outh, noise, aberration):
    ora = S.OracleEngine("vhs", outw, outh, seed=SEED)
    ora.set(blend=0, scanlines=1, saturation=10)
    want = []
    for f in range(len(frames)):
        field, frame = video.frame_parity(f)
        ora.modulate(frames[f], format=layout.PIX_BGRA, as_color=1, field=field, frame=frame, do_aberration=aberration)
        ora.demodulate(noise)
        want.append(ora.out.copy())
    return np.stack(want)


def converter(noise, aberration, segments, factory):
    return video.VideoConverter("vhs", 320, 240, noise=noise, scanlines=1, segments=segments, batch_factory=factory,
                                seed=SEED, do_aberration=aberration)


@pytest.mark.parametrize("noise,aberration,segments,n,wrong", [(0, 0, 4, 11, False), (24, 1, 5, 13, False),
                                                               (24, 1, 3, 10, True), (0, 1, 10, 10, True)])
def test_single_process(noise, aberration, segments, n, wrong):
    frames = make_frames(n)
    vc = converter(noise, aberration, segments, WrongHaloSync if wrong else VhsOracleBatch)
    got = vc.convert(torch.from_numpy(frames)).numpy()
    want = sequential(frames, 320, 240, noise, aberration)
    for f in range(n):
        assert np.array_equal(got[f], want[f]), "image %d (redone %d)" % (f, vc.recomputed)
    if wrong:
        assert vc.recomputed == segments - 1


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q, noise, aberration, segments, n, wrong):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    sys.path.insert(0, HERE)
    import pkgload
    pkgload.load()
    import test_vhs_video_logic as T
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        frames = T.make_frames(n)
        lo, hi = sharding.shard_range(n, rank, world)
        vc = T.converter(noise, aberration, segments, T.WrongHaloSync if wrong else T.VhsOracleBatch)
        mine = vc.convert(torch.from_numpy(frames[lo:hi]), first_frame=lo)
        q.put((rank, lo, hi, mine.numpy().copy(), vc.recomputed))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,noise,aberration,segments,n,wrong", [(2, 24, 1, 2, 10, False), (3, 0, 1, 2, 12, True),
                                                                     (2, 24, 0, 3, 12, True)])
def test_over_ranks(world, noise, aberration, segments, n, wrong):
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q, noise, aberration, segments, n, wrong)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=900) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want = sequential(make_frames(n), 320, 240, noise, aberration)
    redone = 0
    for rank, lo, hi, got, rec in results:
        redone += rec
        for f in range(lo, hi):
            assert np.array_equal(got[f - lo], want[f]), "rank %d image %d (redone %d)" % (rank, f, rec)
    if wrong:
        assert redone > 0


def test_skip_does_not_depend_on_the_signal():
    """the stand-in's skip (blank fields) against real fields on an image at a loud noise, from one seed"""
    b = VhsOracleBatch("vhs", 1)
    b.set_monitor(0, torch.zeros(240, 320, 4, dtype=torch.uint8), noise=200)
    b.commit_monitors()
    b.seed(SEED)
    b.skip_fields([3], 1)
    ora = S.OracleEngine("vhs", 320, 240, seed=SEED)
    img = S.rand_image(300, 200, seed=3)
    for f in range(3):
        ora.modulate(img, format=layout.PIX_BGRA, as_color=1, field=f & 1, frame=1, do_aberration=1)
        ora.demodulate(200)
    r = ora.rand
    assert np.array_equal(b.get_rand()[0], [r.r[(r.f + j) % 31] for j in range(31)])


# ---------------------------------------------------------------------------------------------------------------
# checks 1-4 of tests/test_gpu_vhs_video.py on the SIMT interpreter's VHS build
# ---------------------------------------------------------------------------------------------------------------

@pytest.fixture
def simt_vhs(monkeypatch):
    sys.path.insert(0, os.path.join(HERE, "simt"))
    import build as simt_build
    simt_build.build(["vhs"])
    monkeypatch.setattr(capi, "lib_path", lambda v: simt_build.lib_path(v))
    monkeypatch.setattr(capi, "_libs", {})
    real_zeros = torch.zeros

    def host_zeros(*a, **kw):
        kw.pop("device", None)
        return real_zeros(*a, **kw)
    monkeypatch.setattr(torch, "zeros", host_zeros)
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **kw: self)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **kw: None)
    import test_gpu_vhs_video as G
    return G


def test_simt_seed_words(simt_vhs):
    simt_vhs.check_seed_words((0, 1, 42, 0xFFFFFFFF))


def test_simt_set_get_roundtrip(simt_vhs):
    simt_vhs.check_set_get_roundtrip()


def test_simt_skip_equals_real_fields(simt_vhs):
    simt_vhs.check_skip_equals_real_fields((1, 0xDEADBEEF), (0, 1, 2))


def test_simt_field_from_set_state(simt_vhs):
    simt_vhs.check_field_from_set_state(2)
