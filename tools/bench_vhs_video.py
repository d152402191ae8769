"""Timing of the VHS video path on one GPU (prints one JSON line).

  skip_field_us     device time of k_vhs_skip per skipped field (CUDA events around one crtx_skip_fields of many fields)
  skip_5000_s       wall time of crtx_skip_fields over a 5 000-field sequence, one monitor, ending in a synchronise
  sequential_s      a one-monitor capi.Batch looping over the frames: set_source, modulate, demodulate, one field per step
  converter_s       VideoConverter("vhs") over the same frames (after a warm-up call that builds its contexts)
  recomputed        segments the converter had to redo; identical is its output against the sequential loop's

    python tools/bench_vhs_video.py [--frames 1000] [--size 640x480] [--noise 24] [--aberration 1] [--segments 64]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_name_and_power():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                             stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def frames_of(n, w, h, torch):
    """n moving-bar frames (BGRA), made on the device"""
    x = torch.arange(w, device="cuda").view(1, 1, w)
    t = torch.arange(n, device="cuda").view(n, 1, 1)
    y = torch.arange(h, device="cuda").view(1, h, 1)
    f = torch.empty(n, h, w, 4, dtype=torch.uint8, device="cuda")
    f[..., 0] = ((x * 3 + t * 5) % 256).to(torch.uint8).expand(n, h, w)
    f[..., 1] = ((x + y + t * 7) % 256).to(torch.uint8)
    f[..., 2] = (((x // 40 + t) % 8) * 32).to(torch.uint8).expand(n, h, w)
    f[..., 3] = 255
    return f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--size", default="640x480")
    ap.add_argument("--noise", type=int, default=24)
    ap.add_argument("--aberration", type=int, default=1)
    ap.add_argument("--segments", type=int, default=64)
    ap.add_argument("--skip-fields", type=int, default=2000)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    import pkgload
    pkgload.load()
    import torch
    from ntsc_crt_b200 import capi, layout, video
    if not torch.cuda.is_available():
        raise SystemExit("bench_vhs_video: no CUDA device")
    w, h = (int(v) for v in args.size.split("x"))
    res = dict(gpu=gpu_name_and_power(), frames=args.frames, size=args.size, noise=args.noise, aberration=args.aberration,
               segments=args.segments)

    # ---- k_vhs_skip: device time per field, and a 5 000-field skip end to end
    b = capi.Batch("vhs", 1)
    b.seed(args.seed)
    b.skip_fields([4], args.aberration)  # (warm-up: module load)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    b.skip_fields([args.skip_fields], args.aberration)
    e1.record()
    torch.cuda.synchronize()
    res["skip_field_us"] = round(e0.elapsed_time(e1) * 1000.0 / args.skip_fields, 2)
    t0 = time.perf_counter()
    b.skip_fields([5000], args.aberration)
    b.get_rand()  # (synchronises)
    res["skip_5000_s"] = round(time.perf_counter() - t0, 4)
    b.close()

    # ---- the sequential one-monitor loop against VideoConverter("vhs")
    frames = frames_of(args.frames, w, h, torch)
    seq = torch.empty(args.frames, h, w, 4, dtype=torch.uint8, device="cuda")
    b = capi.Batch("vhs", 1)
    out = torch.zeros(h, w, 4, dtype=torch.uint8, device="cuda")
    b.set_monitor(0, out, fmt=layout.PIX_BGRA, noise=args.noise, blend=0, scanlines=1, saturation=10)
    b.commit_monitors()
    b.seed(args.seed)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for f in range(args.frames):
        field, frame = video.frame_parity(f)
        b.set_source(0, frames[f], format=layout.PIX_BGRA, as_color=1, field=field, frame=frame, do_aberration=args.aberration)
        b.modulate()
        b.demodulate()
        seq[f].copy_(out)
    torch.cuda.synchronize()
    res["sequential_s"] = round(time.perf_counter() - t0, 4)
    b.close()

    vc = video.VideoConverter("vhs", w, h, noise=args.noise, scanlines=1, segments=args.segments, seed=args.seed,
                              do_aberration=args.aberration)
    vc.convert(frames[:max(2, args.segments)])  # (warm-up: builds the pooled contexts the timed call uses)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    got = vc.convert(frames)
    torch.cuda.synchronize()
    res["converter_s"] = round(time.perf_counter() - t0, 4)
    res["recomputed"] = vc.recomputed
    res["identical"] = bool(torch.equal(got, seq))
    res["speedup"] = round(res["sequential_s"] / res["converter_s"], 2)
    vc.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
