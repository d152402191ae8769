"""CPU half of tests/test_gpu_video_convert_unmodified.py: pins the stack-clearing harness (oracle/zero_stack_main.c) in
front of the reference's UNMODIFIED extra/video_convert.c against the oracle's sequential loop.  Where oracle/_ref is not
built, the digests of the driver's images are replayed from tests/golden/ref_states.json."""
import pytest

import support as S
from ntsc_crt_b200 import layout
from test_gpu_video_driver import moving_bars, read_bmp32
from test_gpu_video_convert_unmodified import REF_VIDEO, run_driver


@pytest.mark.parametrize("flags,noise", [("-o", 0), ("-om", 7)])
def test_reference_video_driver_with_a_cleared_stack_is_the_sequential_loop(tmp_path, flags, noise):
    """CPU only: pins the harness -- with the stack cleared the unmodified driver equals the oracle's loop with
    xoffset = yoffset = 0 (video_convert.c:226-277: blend 0, scanlines 1, field toggles every image, frame every other)"""
    frames = moving_bars(6, 320, 240, seed=2)

    def reference(exe):
        run_driver(exe, str(tmp_path), frames, flags, 640, 480, noise)
        return [S.digest(read_bmp32(str(tmp_path / "output" / ("%06d.bmp" % (k + 1))))) for k in range(len(frames))]
    want = S.from_reference(REF_VIDEO, reference)
    assert len(want) == 6
    ora = S.OracleEngine("ntsc", 640, 480)
    ora.set(blend=0, scanlines=1, saturation=10)
    field = frame = 0
    for k in range(len(frames)):
        ora.modulate(frames[k], format=layout.PIX_BGRA, as_color=0 if "m" in flags else 1, field=field, frame=frame, raw=0, hue=0)
        ora.demodulate(noise)
        field ^= 1
        if ((k + 1) & 1) == 0:
            frame ^= 1
        assert S.digest(ora.out) == want[k], "image %d differs from the reference driver's" % (k + 1)


