"""config 4 (video_convert.c flow): the time-parallel VideoConverter against the sequential loop run on the
oracle -- one CRT, blend 0, field toggling every frame (extra/video_convert.c:226-277)."""
import numpy as np
import pytest

import support as S
from ntsc_crt_b200 import layout

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("noise,segments", [(0, 5), (12, 4)])
def test_video_sequence_matches_sequential_reference_loop(noise, segments):
    import torch
    from ntsc_crt_b200 import video
    n, w, h = 23, 320, 240
    frames = S.moving_bars(n, w, h)
    ora = S.OracleEngine("ntsc", 640, 480)
    ora.set(blend=0, scanlines=1, saturation=10)
    want = []
    for f in range(n):
        field, frame = video.frame_parity(f)
        ora.modulate(frames[f], format=layout.PIX_BGRA, as_color=1, field=field, frame=frame)
        ora.demodulate(noise)
        want.append(ora.out.copy())
    vc = video.VideoConverter("ntsc", 640, 480, noise=noise, scanlines=1, segments=segments)
    got = vc.convert(torch.from_numpy(frames).cuda()).cpu().numpy()
    for f in range(n):
        assert np.array_equal(got[f], want[f]), "frame %d (recomputed segments: %d)" % (f, vc.recomputed)
    if noise == 0:
        assert vc.recomputed == 0, "steady-state speculation should hold without noise"
