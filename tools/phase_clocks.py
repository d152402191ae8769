#!/usr/bin/env python
"""Where the time of one step goes INSIDE the kernels: a debug build of the NTSC library (-DCRTX_PHASE_CLOCKS=1, built by
`make -C ntsc-crt_b200/csrc custom NAME=ntsc DEFS="-DCRT_SYSTEM=0 -DCRTX_PHASE_CLOCKS=1" LIB=../lib_dbg`) stamps the SM
cycle counter at the phase boundaries of k_sync and at the start / end of the encoder and of k_lines2, per CTA; this
script runs bench.py's step on the headline workload with that library and prints the averages.  Not a bench: the
stamps cost a little, and nothing printed here is a throughput figure."""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ.setdefault("CRT_B200_LIB_DIR", os.path.join(ROOT, "ntsc-crt_b200", "lib_dbg"))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import pkgload  # noqa: E402
pkgload.load()
from ntsc_crt_b200 import capi, layout  # noqa: E402

B, W, H = 264, 832, 624
dev = torch.device("cuda", 0)
gen = torch.Generator(device="cpu").manual_seed(1234)
src = torch.randint(0, 256, (B, H, W, 4), dtype=torch.uint8, generator=gen).to(dev)
out = torch.zeros(B, H, W, 4, dtype=torch.uint8, device=dev)
batch = capi.Batch("ntsc", B)
for kv in sys.argv[1:]:
    name, val = kv.split("=")
    batch.set_option(name, int(val))
for i in range(B):
    batch.set_monitor(i, out[i], fmt=layout.PIX_BGRA, noise=0, blend=1, scanlines=1)
batch.commit_monitors()
for f in range(6):
    for i in range(B):
        batch.set_source(i, src[i], format=layout.PIX_BGRA, as_color=1, field=f & 1, frame=0)
    batch.modulate()
    batch.demodulate()
torch.cuda.synchronize()
fn = batch.lib.crtx_debug_clocks
fn.argtypes = [C.c_void_p]
fn.restype = C.c_int
tab = np.zeros((4, 512, 16), dtype=np.uint64)
assert fn(tab.ctypes.data) == 0
names = {0: "k_sync", 1: "k_lines2", 2: "k_mod_picture"}
mhz = 1965.0
for k, name in names.items():
    t = tab[k]
    n = int((t[:, 0] != 0).sum())
    if n == 0:
        continue
    t = t[:n].astype(np.int64)
    start_ns, end_ns = t[:, 0], t[:, 14]
    print("== %s: %d CTAs; start skew %.1f us, end skew %.1f us, first start -> last end %.1f us" % (
        name, n, (start_ns.max() - start_ns.min()) / 1e3, (end_ns.max() - end_ns.min()) / 1e3, (end_ns.max() - start_ns.min()) / 1e3))
    c0 = t[:, 15]
    prev = c0
    for ph in list(range(1, 13)) + [13]:
        if (t[:, ph] == 0).all():
            continue
        d_start = (t[:, ph] - c0) / mhz
        print("   phase %2d reached at %7.2f us after the CTA's start (min %7.2f, max %7.2f)" % (ph, d_start.mean(), d_start.min(), d_start.max()))
