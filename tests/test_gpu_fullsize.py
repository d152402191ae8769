"""BASELINE configs[1] at the bench's full size -- a batch of 264 monitors (two per SM of an H100), 832x624 BGRA in and out,
interlaced, blend 1, scanlines 1 -- checked through a size-independent property instead of 264 oracle runs: monitors
that are fed the same image, settings and noise must stay bit-identical to each other through every field (a checksum
of checksums: one representative per group against all its members, on the device), and the representatives are
compared with the oracle, whole state.  Also: the context's whole state after the run equals the oracle's for every monitor."""
import pytest

import support as S
from ntsc_crt_b200 import layout

pytestmark = pytest.mark.gpu

BATCH = 264   # bench.py's batch per GPU; tests/test_simt_kernels.py shrinks it for the CPU interpreter
GROUPS = 4
FIELDS = 4


def test_full_size_batch_is_consistent_and_matches_the_oracle():
    import torch
    from ntsc_crt_b200 import capi
    n = BATCH
    b = capi.Batch("ntsc", n)
    imgs = [S.rand_image(832, 624, seed=70 + g) if g else S.bars_image(832, 624) for g in range(GROUPS)]
    noises = [0, 24, 0, 255][:GROUPS]
    dimgs = [torch.from_numpy(im).cuda() for im in imgs]
    outs = torch.zeros(n, 624, 832, 4, dtype=torch.uint8, device="cuda")
    for i in range(n):
        b.set_monitor(i, outs[i], fmt=layout.PIX_BGRA, noise=noises[i % GROUPS], blend=1, scanlines=1)
    b.commit_monitors()
    oras = []
    for g in range(GROUPS):
        o = S.OracleEngine("ntsc", 832, 624)
        o.set(blend=1, scanlines=1)
        oras.append(o)
    for it in range(FIELDS):
        kw = dict(format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=(it >> 1) & 1)
        for i in range(n):
            b.set_source(i, dimgs[i % GROUPS], **kw)
        b.modulate()
        b.demodulate()
        torch.cuda.synchronize()
        for g in range(GROUPS):
            oras[g].modulate(imgs[g], **kw)
            oras[g].demodulate(noises[g])
            members = outs[g::GROUPS]
            same = (members == members[0:1]).reshape(members.shape[0], -1).all(dim=1)
            assert bool(same.all()), "field %d group %d: monitors %r differ from monitor %d" % (
                it, g, [g + GROUPS * int(k) for k in torch.nonzero(~same).flatten()[:8]], g)
            S.assert_same_state(S.monitor_state(b, g, outs[g]), oras[g].state(), "field %d group %d" % (it, g))
    want = [o.state() for o in oras]
    for i in range(n):
        S.assert_same_state(S.monitor_state(b, i, outs[i]), want[i % GROUPS], "monitor %d after the run" % i)
    b.close()
