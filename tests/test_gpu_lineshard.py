"""Scanline-block partition of one image (SURVEY 8e) on the GPU: two crtx contexts stand in for two ranks,
each decoding its own block of lines of every field (crtx_set_option line_lo/line_hi) into its own image;
rows are handed over / merged by the rules of ntsc_crt_b200.sharding.ImageSharder.  The merged image must equal
the sequential decode (oracle).  The collective plumbing itself is covered on CPU by
tests/test_sharding_gloo.py."""
import numpy as np
import pytest

import support as S
from ntsc_crt_b200 import layout, sharding

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("variant", ["ntsc", "ntsc_conv"])
@pytest.mark.parametrize("outw,outh,scanlines,blend,world", [
    (832, 624, 1, 1, 2),
    (640, 480, 0, 1, 2),   # spill row travels after odd fields
    (400, 1080, 0, 1, 3),  # two spill rows, uneven blocks
    (320, 360, 0, 1, 16),  # 1.5 rows per line: a block's last line can be ONE row tall, its computed (blended) row then
    (320, 360, 1, 1, 16),  # lands in the next block in odd fields -- needs that block's rows first (the halo)
])
def test_two_contexts_decode_one_image(variant, outw, outh, scanlines, blend, world):
    decode_one_image_in_blocks(variant, outw, outh, scanlines, blend, world)


@pytest.mark.parametrize("variant,outw,outh,scanlines,blend,world", [("pv1k", 640, 480, 0, 1, 2), ("template", 832, 624, 1, 1, 2),
                                                                    ("ntsc_bloom", 640, 480, 0, 1, 2), ("ntsc_bloom", 400, 1080, 0, 1, 3)])
def test_blocks_of_the_newer_variants(variant, outw, outh, scanlines, blend, world):
    """the line window (line_lo / line_hi) through the PV-1000 line kernel and through k_lines_bloom, whose energy
    chain still runs over every line of the field on every rank"""
    decode_one_image_in_blocks(variant, outw, outh, scanlines, blend, world)


def decode_one_image_in_blocks(variant, outw, outh, scanlines, blend, world, v_fac=0):
    import torch
    from ntsc_crt_b200 import capi
    img = S.rand_image(320, 240, seed=11)
    dimg = torch.from_numpy(img).cuda()
    ora = S.OracleEngine(variant, outw, outh)
    ora.set(blend=blend, scanlines=scanlines, v_fac=v_fac)
    ranks = []
    for r in range(world):
        b = capi.Batch(variant, 1)
        out = torch.zeros(outh, outw, 4, dtype=torch.uint8, device="cuda")
        b.set_monitor(0, out, fmt=layout.PIX_BGRA, noise=4, blend=blend, scanlines=scanlines, v_fac=v_fac)
        b.commit_monitors()
        part = sharding.ImageSharder(out, b.spec.lines, rank=r, world=world, v_fac=v_fac)
        part.apply(b)
        ranks.append((b, out, part))
    for it in range(6):
        ora.modulate(img, format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=(it >> 1) & 1)
        ora.demodulate(4)
        ends = []
        for r in range(world - 1):  # what ImageSharder.fetch_halo_rows does over the process group, before the field
            (_, dst, ps), (_, src, pn) = ranks[r], ranks[r + 1]
            cnt = ps._halo_count(r)
            if cnt:
                dst[ps.r1:ps.r1 + cnt].copy_(src[pn.r0:pn.r0 + cnt])
        for b, out, part in ranks:
            b.set_source(0, dimg, format=layout.PIX_BGRA, as_color=1, field=it & 1, frame=(it >> 1) & 1)
            b.modulate()
            b.demodulate()
            last = b.get_lines(0)[part.hi - 1]
            ends.append(0 if last.beg < 0 else max(last.beg + 1, last.end - scanlines))
        torch.cuda.synchronize()
        for r in range(world - 1):  # what ImageSharder.exchange_spill_rows does over the process group
            (_, src, ps), (_, dst, pd) = ranks[r], ranks[r + 1]
            cnt = max(0, min(ends[r], outh, ps.r1 + ps.max_spill()) - ps.r1)
            if cnt and pd.r0 == ps.r1:
                dst[pd.r0:pd.r0 + cnt].copy_(src[ps.r1:ps.r1 + cnt])
    full = np.zeros((outh, outw, 4), dtype=np.uint8)
    for b, out, part in ranks:
        full[part.r0:part.r1] = out[part.r0:part.r1].cpu().numpy()
        b.close()
    assert np.array_equal(full, ora.out), S.diff_report("merged image", full, ora.out)
