"""oracle/wire_oracle.py's restatement of the live driver's phosphor decay against the reference's own function: the lines
of fade_phosphors() are cut out of /root/reference/crt_main.c (437-452; that branch of the file needs an external windowing
library and cannot be compiled whole) into a scratch translation unit by oracle/Makefile (libref_fade.so); where that is not built, the reference's results
are replayed from tests/golden/ref_states.json.  This is what
pins `crtx_fade_phosphors` (tests/test_gpu_wire.py) to the reference rather than to our own reading of it."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import support as S

sys.path.insert(0, S.ORACLE_DIR)
import wire_oracle as W  # noqa: E402

REF = os.path.join(S.REF_DIR, "libref_fade.so")


@pytest.mark.parametrize("w,h,seed", [(832, 624, 1), (53, 37, 2), (1, 1, 3), (640, 480, 4)])
def test_fade_phosphors_restatement_is_the_reference_function(w, h, seed):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 1 << 32, size=w * h, dtype=np.uint32)
    img[:4] = (0, 0xFFFFFFFF, 0x00FFFFFF, 0xFF000000)[: min(4, img.size)]

    def reference(path):  # digest of the image after each of six applications (the live loop: frame after frame)
        R = C.CDLL(path)
        theirs = img.astype(np.int32).copy()
        out = []
        for _ in range(6):
            R.ref_fade_phosphors(theirs.ctypes.data_as(C.c_void_p), w, h)
            out.append(S.digest(theirs.view(np.uint32)))
        return out
    want = S.from_reference(REF, reference)
    ours = img.copy()
    for k in range(6):
        ours = W.fade_phosphors(ours).astype(np.uint32)
        assert S.digest(ours) == want[k], "application %d" % (k + 1)
