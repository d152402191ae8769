"""N > 1 host logic on CPU: world_size 2 over gloo (frames shard, timings reduce with max,
the optional all_gather of decoded frames reassembles the batch in rank order)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import pkgload

pkgload.load()
from ntsc_crt_b200 import sharding


def test_shard_range_partitions_exactly():
    for n in (0, 1, 7, 8, 296, 4999):
        for world in (1, 2, 3, 4, 8):
            spans = [sharding.shard_range(n, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            for (a, b), (c, d) in zip(spans, spans[1:]):
                assert b == c and b - a >= d - c >= b - a - 1


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import pkgload as pl
    pl.load()
    from ntsc_crt_b200 import sharding as sh
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        assert sh.rank_info() == (rank, rank, world)
        lo, hi = sh.shard_range(10, rank, world)
        # every rank "decodes" its slice of 10 frames: frame k is filled with k
        local = torch.stack([torch.full((4, 6, 4), k, dtype=torch.uint8) for k in range(lo, hi)])
        allf = sh.allgather_frames(local)
        ms = sh.max_over_ranks([10.0 + rank, 5.0 - rank])
        q.put((rank, allf.numpy().copy(), ms))
    finally:
        dist.destroy_process_group()


def test_world_size_2_gloo():
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want = np.stack([np.full((4, 6, 4), k, dtype=np.uint8) for k in range(10)])
    for rank, allf, ms in results:
        assert np.array_equal(allf, want)
        assert ms == [11.0, 5.0]


# ---------------------------------------------------------------------------------------------
# scanline-block partition of ONE image (SURVEY 8e): the host logic, with the oracle's staged decode
# standing in for the kernels (noise + sync replicated, line pass restricted to the rank's block)
# ---------------------------------------------------------------------------------------------
def test_line_blocks_and_row_ownership():
    for world in (1, 2, 3, 8):
        for outh in (624, 480, 240, 100, 1080):
            blocks = [sharding.block_rows(*sharding.line_block(r, world, 240), outh, 240) for r in range(world)]
            assert blocks[0][0] == 0 and blocks[-1][1] == outh
            for (a, b), (c, d) in zip(blocks, blocks[1:]):
                assert b == c and a <= b
    assert sharding.block_rows(0, 30, 624, 240) == (0, 78)  # SURVEY 8e: 30 lines <-> 78 rows at 832x624


def test_row_span_wraps_like_the_reference():
    """outh + v_fac is 32-bit unsigned in the reference (crt_core.c:428): a "negative" v_fac shrinks the span, and a
    span whose products wrap has no partition into blocks of consecutive lines"""
    edge = (2**32 - 1) // 240
    assert sharding.row_span(200, 2**32 - 60, 240) == 140
    assert sharding.row_span(200, 100, 240) == 300
    assert sharding.row_span(200, edge - 200, 240) == edge
    assert sharding.block_rows(0, 120, 200, 240, v_fac=100) == (0, 150)
    assert sharding.block_rows(120, 240, 200, 240, v_fac=100) == (150, 200)
    for v_fac in (edge + 1 - 200, 2**31, 2**32 - 201):  # spans edge + 1, 2^31 + 200, 2^32 - 1
        with pytest.raises(ValueError, match="wraps"):
            sharding.block_rows(0, 120, 200, 240, v_fac=v_fac)
        with pytest.raises(ValueError, match="wraps"):
            sharding.ImageSharder(torch.zeros(200, 64, 4, dtype=torch.uint8), 240, rank=0, world=2, v_fac=v_fac)
    with pytest.raises(ValueError, match="at least one output row"):  # shrunk below one row per line by the wrap
        sharding.ImageSharder(torch.zeros(200, 64, 4, dtype=torch.uint8), 240, rank=0, world=2, v_fac=2**32 - 60)
    part = sharding.ImageSharder(torch.zeros(200, 64, 4, dtype=torch.uint8), 240, rank=1, world=2, v_fac=100)
    assert (part.r0, part.r1) == (150, 200)


def _image_worker(rank, world, port, q, cfg):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import pkgload as pl
    pl.load()
    import support as S
    from ntsc_crt_b200 import layout, sharding as sh
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        outw, outh, scanlines, blend, progressive, noise = cfg
        img = S.rand_image(200, 150, seed=5)
        eng = S.OracleEngine("ntsc", outw, outh)
        eng.set(blend=blend, scanlines=scanlines)
        image = torch.from_numpy(eng.out)  # shares memory with the monitor's output buffer
        part = sh.ImageSharder(image, eng.spec.lines)
        for it in range(6):
            field = 0 if progressive else it & 1
            eng.modulate(img, format=layout.PIX_BGRA, as_color=1, field=field, frame=(it >> 1) & 1)
            part.fetch_halo_rows()
            eng.noise_pass(noise)
            _, table = eng.sync_pass()
            eng.line_pass(table, part.lo, part.hi - part.lo)
            last = table[part.hi - 1]
            part.exchange_spill_rows(0 if last.skip else max(last.beg + 1, last.end - scanlines))
        q.put((rank, part.gather().numpy().copy()))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,cfg", [
    (2, (832, 624, 1, 1, False, 0)),   # config 2's knobs: blocks are independent
    (2, (640, 480, 0, 1, False, 7)),   # scanlines 0 + blend + interlaced: the spill row must travel
    (3, (333, 250, 0, 1, False, 0)),   # uneven blocks
    (2, (256, 240, 0, 0, True, 3)),
    (2, (400, 1080, 0, 1, False, 0)),  # ratio 4.5: two spill rows per odd field
    (16, (320, 360, 0, 1, False, 0)),  # 1.5 rows per line: blocks whose last line is ONE row tall put their computed,
    (16, (320, 360, 1, 1, False, 5)),  # blended row into the next block in odd fields (round-1 advisor finding)
    (7, (320, 300, 0, 1, False, 0)),
    (5, (200, 241, 0, 1, False, 2)),   # barely one row per line
])
def test_one_image_over_ranks_matches_the_sequential_decode(world, cfg):
    import support as S
    from ntsc_crt_b200 import layout
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_image_worker, args=(r, world, port, q, cfg)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    outw, outh, scanlines, blend, progressive, noise = cfg
    img = S.rand_image(200, 150, seed=5)
    ref = S.OracleEngine("ntsc", outw, outh)
    ref.set(blend=blend, scanlines=scanlines)
    for it in range(6):
        field = 0 if progressive else it & 1
        ref.modulate(img, format=layout.PIX_BGRA, as_color=1, field=field, frame=(it >> 1) & 1)
        ref.demodulate(noise)
    for rank, full in results:
        assert np.array_equal(full, ref.out), "rank %d: %s" % (rank, S.diff_report("image", full, ref.out))


def test_geometries_the_partition_cannot_serve_are_refused():
    """fewer output rows than decoded lines: lines of two ranks would share a row and must be applied in order
    (crt_core.c:409-664), which blocks cannot do -- a clear error instead of a wrong image; likewise blocks thinner than
    the odd-field shift"""
    img = torch.zeros(120, 64, 4, dtype=torch.uint8)
    with pytest.raises(ValueError, match="one output row per decoded line"):
        sharding.ImageSharder(img, 240, rank=0, world=7)
    sharding.ImageSharder(img, 240, rank=0, world=1)  # a single rank is always fine
    tall = torch.zeros(2400, 8, 4, dtype=torch.uint8)  # ratio 10: shift 5 rows; 240 ranks x 10 rows is fine, 5-row blocks are not possible
    sharding.ImageSharder(tall, 240, rank=3, world=240)
