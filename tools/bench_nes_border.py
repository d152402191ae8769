"""What the NES border colour costs: 264 monitors per step (one NES field each: modulate + demodulate), the stock NES
library (libcrt_b200_nes.so) against the NES_BORDER 1 build (libcrt_b200_nes_border.so), alternated in one run.  The
encoder is timed with the library's per-kernel CUDA events (option "timing": kernel 0 is k_nes_table + k_mod_nes), the
whole step with a pair of CUDA events around it.  Prints one JSON line per round and a summary line, with the card's
name and power limit beside the numbers.  Writes nothing.

    python tools/bench_nes_border.py [--monitors 264] [--steps 50] [--warmup 10] [--rounds 4]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import pkgload  # noqa: E402

pkgload.load()
import numpy as np  # noqa: E402
import torch  # noqa: E402
from ntsc_crt_b200 import capi, layout  # noqa: E402

VARIANTS = ("nes", "nes_border")


def power_limit():
    """the card's enforced power limit as nvidia-smi reports it (a read-only query), or 'unknown'"""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                           text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def make_batch(variant, n, imgs):
    b = capi.Batch(variant, n)
    outs = []
    for i in range(n):
        t = torch.zeros(480, 640, 4, dtype=torch.uint8, device="cuda")
        outs.append(t)
        b.set_monitor(i, t, fmt=layout.PIX_BGRA, noise=4, blend=1, scanlines=1)
    b.commit_monitors()
    for i in range(n):
        b.set_source(i, imgs[i % len(imgs)], dot_crawl_offset=i % 3, xoffset=(4 * i) % 31, yoffset=i % 8,
                     border_color=(0x22 + 7 * i) & 0x1ff)
    b._outs = outs
    return b


def run(b, steps, warmup):
    """(encoder ms per step, step ms) over `steps` steps after `warmup` untimed ones"""
    for it in range(warmup):
        for i in range(b.n):
            b.sources[i].reinit = int(it == 0)
            b.sources[i].dot_crawl_offset = (i + it) % 3
        b.modulate()
        b.demodulate()
    torch.cuda.synchronize()
    b.set_option("timing", 1)
    b.timing()  # (drops anything recorded so far)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for it in range(steps):
        for i in range(b.n):
            b.sources[i].dot_crawl_offset = (i + it) % 3
        b.modulate()
        b.demodulate()
    e1.record()
    torch.cuda.synchronize()
    t = b.timing()
    b.set_option("timing", 0)
    return t["mod_skeleton"][0] / steps, e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--monitors", type=int, default=264)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=4)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    card = dict(gpu=torch.cuda.get_device_name(0), power_limit=power_limit())
    imgs = [torch.from_numpy(np.random.default_rng(s).integers(0, 512, size=(240, 256)).astype(np.int16)).cuda()
            for s in range(8)]
    batches = {v: make_batch(v, a.monitors, imgs) for v in VARIANTS}
    res = {v: ([], []) for v in VARIANTS}
    for r in range(a.rounds):
        for v in (VARIANTS if r % 2 == 0 else VARIANTS[::-1]):  # alternated, each first in every other round
            enc, step = run(batches[v], a.steps, a.warmup)
            res[v][0].append(enc)
            res[v][1].append(step)
            print(json.dumps(dict(round=r, variant=v, monitors=a.monitors, encoder_ms=round(enc, 4), step_ms=round(step, 4),
                                  **card)))
    med = {v: (statistics.median(res[v][0]), statistics.median(res[v][1])) for v in VARIANTS}
    print(json.dumps(dict(summary=True, monitors=a.monitors, steps=a.steps, rounds=a.rounds,
                          encoder_ms={v: round(med[v][0], 4) for v in VARIANTS},
                          step_ms={v: round(med[v][1], 4) for v in VARIANTS},
                          encoder_ratio=round(med["nes_border"][0] / med["nes"][0], 4),
                          step_ratio=round(med["nes_border"][1] / med["nes"][1], 4), **card)))
    for b in batches.values():
        b.close()


if __name__ == "__main__":
    main()
