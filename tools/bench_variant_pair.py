"""What one library variant costs or saves against another: 264 monitors per step (one field each: modulate +
demodulate), the two libraries alternated in one run, at each noise level given.  The sources follow the system: NES
pixels (dot crawl, picture offsets and border colour varying over the monitors) or RGB pictures (interlaced fields).
Each kernel is timed with the library's per-kernel CUDA events (option "timing": mod_skeleton is the encoder's first
kernel -- k_nes_table + k_mod_nes on the NES --, sync is k_sync with the fused noise pass, lines the line passes), the
whole step with a pair of CUDA events around it.  Prints one JSON line per round and a summary line per noise level
(medians, and B / A ratios), with the card's name and power limit beside the numbers.  Writes nothing.

    python tools/bench_variant_pair.py A B [--noise N ...] [--size WxH] [--monitors 264] [--steps 50] [--warmup 10]
                                           [--rounds 4]
e.g.
    python tools/bench_variant_pair.py nes nes_border --size 640x480 --noise 4
    python tools/bench_variant_pair.py ntsc ntsc_nosync --noise 0 60
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


def power_limit():
    """the card's enforced power limit as nvidia-smi reports it (a read-only query), or 'unknown'"""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                           text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def is_nes(variant):
    return layout.system_spec(variant).system == layout.SYS_NES


def sources(nes):
    """eight device source images: NES pixels or BGRA pictures"""
    if nes:
        return [torch.from_numpy(np.random.default_rng(s).integers(0, 512, size=(240, 256)).astype(np.int16)).cuda()
                for s in range(8)]
    return [torch.from_numpy(np.random.default_rng(s).integers(0, 256, size=(240, 320, 4), dtype=np.uint8)).cuda()
            for s in range(8)]


def make_batch(variant, n, size, noise):
    nes = is_nes(variant)
    imgs = sources(nes)
    b = capi.Batch(variant, n)
    outs = []
    for i in range(n):
        t = torch.zeros(size[1], size[0], 4, dtype=torch.uint8, device="cuda")
        outs.append(t)
        b.set_monitor(i, t, fmt=layout.PIX_BGRA, noise=noise, blend=1, scanlines=1)
    b.commit_monitors()
    for i in range(n):
        if nes:
            b.set_source(i, imgs[i % len(imgs)], dot_crawl_offset=i % 3, xoffset=(4 * i) % 31, yoffset=i % 8,
                         border_color=(0x22 + 7 * i) & 0x1ff)
        else:
            b.set_source(i, imgs[i % len(imgs)], format=layout.PIX_BGRA, as_color=1, hue=0)
    b._outs = outs
    return b


def run(b, steps, warmup):
    """({kernel: ms per step}, step ms) over `steps` steps after `warmup` untimed ones, the first of which re-initialises"""
    nes = b.spec.system == layout.SYS_NES

    def step(it, reinit=0):
        for i in range(b.n):
            s = b.sources[i]
            s.reinit = reinit
            if nes:
                s.dot_crawl_offset = (i + it) % 3
            else:
                s.field, s.frame = it & 1, (it >> 1) & 1
        b.modulate()
        b.demodulate()
    for it in range(warmup):
        step(it, int(it == 0))
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
    ap.add_argument("a", help="the variant measured against (e.g. nes, ntsc)")
    ap.add_argument("b", help="the variant measured (e.g. nes_border, ntsc_nosync)")
    ap.add_argument("--noise", type=int, nargs="+", default=[0])
    ap.add_argument("--size", default="832x624", help="output image WxH (the crt_main.c geometry by default)")
    ap.add_argument("--monitors", type=int, default=264)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=4)
    a = ap.parse_args()
    size = tuple(int(x) for x in a.size.split("x"))
    pair = (a.a, a.b)
    torch.cuda.set_device(0)
    card = dict(gpu=torch.cuda.get_device_name(0), power_limit=power_limit())
    for noise in a.noise:
        batches = {v: make_batch(v, a.monitors, size, noise) for v in pair}
        res = {v: ([], []) for v in pair}
        for r in range(a.rounds):
            for v in (pair if r % 2 == 0 else pair[::-1]):  # alternated, each first in every other round
                kern, step = run(batches[v], a.steps, a.warmup)
                res[v][0].append(kern)
                res[v][1].append(step)
                print(json.dumps(dict(round=r, variant=v, noise=noise, monitors=a.monitors, size=a.size,
                                      kernel_ms={k: round(x, 4) for k, x in kern.items()}, step_ms=round(step, 4), **card)))
        med = {v: ({k: statistics.median(d[k] for d in res[v][0]) for k in res[v][0][0]}, statistics.median(res[v][1]))
               for v in pair}
        ka, kb = med[a.a][0], med[a.b][0]
        print(json.dumps(dict(summary=True, noise=noise, monitors=a.monitors, size=a.size, steps=a.steps, rounds=a.rounds,
                              kernel_ms={v: {k: round(x, 4) for k, x in med[v][0].items()} for v in pair},
                              step_ms={v: round(med[v][1], 4) for v in pair},
                              kernel_ratio={k: round(kb[k] / ka[k], 4) for k in ka if k in kb and ka[k] > 0},
                              step_ratio=round(med[a.b][1] / med[a.a][1], 4), **card)))
        for b in batches.values():
            b.close()


if __name__ == "__main__":
    main()
