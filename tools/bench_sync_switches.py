"""What switching the decoder's sync searches off costs or saves: the stock NTSC library (libcrt_b200_ntsc.so) against
the CRT_DO_VSYNC 0 / CRT_DO_HSYNC 0 build (libcrt_b200_ntsc_nosync.so), 264 monitors per step at 832x624 (the
crt_main.c geometry: blend 1, scanlines 1), at noise 0 and 60, the two libraries alternated in one run.  Each kernel is
timed with the library's per-kernel CUDA events (option "timing": sync is k_sync with the fused noise pass, lines the
line passes), the whole step with a pair of CUDA events around it.  Prints one JSON line per round and a summary line
per noise level, with the card's name and power limit beside the numbers.  Writes nothing.

    python tools/bench_sync_switches.py [--monitors 264] [--steps 50] [--warmup 10] [--rounds 4]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tools"))

import pkgload  # noqa: E402

pkgload.load()
import numpy as np  # noqa: E402
import torch  # noqa: E402
from bench_nes_border import power_limit  # noqa: E402
from ntsc_crt_b200 import capi, layout  # noqa: E402

VARIANTS = ("ntsc", "ntsc_nosync")
NOISES = (0, 60)


def make_batch(variant, n, noise, imgs):
    b = capi.Batch(variant, n)
    outs = []
    for i in range(n):
        t = torch.zeros(624, 832, 4, dtype=torch.uint8, device="cuda")
        outs.append(t)
        b.set_monitor(i, t, fmt=layout.PIX_BGRA, noise=noise, blend=1, scanlines=1)
    b.commit_monitors()
    for i in range(n):
        b.set_source(i, imgs[i % len(imgs)], format=layout.PIX_BGRA, as_color=1, hue=0)
    b._outs = outs
    return b


def run(b, steps, warmup):
    """({kernel: ms per step}, step ms) over `steps` steps after `warmup` untimed ones"""
    def step(it):
        for i in range(b.n):
            b.sources[i].field = it & 1
            b.sources[i].frame = (it >> 1) & 1
        b.modulate()
        b.demodulate()
    for it in range(warmup):
        step(it)
    torch.cuda.synchronize()
    b.set_option("timing", 1)
    b.timing()  # (drops anything recorded so far)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for it in range(steps):
        step(it)
    e1.record()
    torch.cuda.synchronize()
    t = b.timing()
    b.set_option("timing", 0)
    return {k: v[0] / steps for k, v in t.items() if v[1]}, e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--monitors", type=int, default=264)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=4)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    card = dict(gpu=torch.cuda.get_device_name(0), power_limit=power_limit())
    imgs = [torch.from_numpy(np.random.default_rng(s).integers(0, 256, size=(240, 320, 4), dtype=np.uint8)).cuda()
            for s in range(8)]
    for noise in NOISES:
        batches = {v: make_batch(v, a.monitors, noise, imgs) for v in VARIANTS}
        res = {v: ([], []) for v in VARIANTS}
        for r in range(a.rounds):
            for v in (VARIANTS if r % 2 == 0 else VARIANTS[::-1]):  # alternated, each first in every other round
                kern, step = run(batches[v], a.steps, a.warmup)
                res[v][0].append(kern)
                res[v][1].append(step)
                print(json.dumps(dict(round=r, variant=v, noise=noise, monitors=a.monitors,
                                      kernel_ms={k: round(x, 4) for k, x in kern.items()}, step_ms=round(step, 4), **card)))
        med = {v: ({k: statistics.median(d[k] for d in res[v][0]) for k in res[v][0][0]}, statistics.median(res[v][1]))
               for v in VARIANTS}
        print(json.dumps(dict(summary=True, noise=noise, monitors=a.monitors, steps=a.steps, rounds=a.rounds,
                              kernel_ms={v: {k: round(x, 4) for k, x in med[v][0].items()} for v in VARIANTS},
                              step_ms={v: round(med[v][1], 4) for v in VARIANTS},
                              sync_ratio=round(med["ntsc_nosync"][0]["sync"] / med["ntsc"][0]["sync"], 4),
                              step_ratio=round(med["ntsc_nosync"][1] / med["ntsc"][1], 4), **card)))
        for b in batches.values():
            b.close()


if __name__ == "__main__":
    main()
