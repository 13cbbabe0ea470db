"""Timing of the interlaced-video kernels (interlace_kernels.cu) on device-resident frames.

  deinterlace_ex  UYVY, v210, RG48, R12L at 1080p, 4K, 8K, in place and out of place
  deinterlace     (the legacy recursive filter, in place) UYVY and RGB at 1080p, 4K, 8K
  il_upper_to_merged / il_merged_to_upper  in place, UYVY line size, 1080p, 4K, 8K

Each case: --warmup launches, then CUDA events around --iters (>= 32) back-to-back launches on one stream; the time per
frame is the mean.  GB/s counts compulsory bytes only: one read and one write of the frame (linesize * lines each).
Prints the card name and power limit read in the same run, then one line per case (and JSON with --json).

    python tools/interlace_bench.py [--iters N] [--warmup N] [--json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = ((1920, 1080), (3840, 2160), (7680, 4320))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def timed(fn, iters, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters  # µs per frame


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--json", action="store_true")
    args = ap.parse_args()
    assert args.iters >= 32
    import torch
    from ultragrid_b200 import Codec, api, vc_get_linesize
    assert torch.cuda.is_available(), "interlace_bench.py needs a GPU"
    print("card:", card())
    cases = []
    for w, h in SIZES:
        for codec in (Codec.UYVY, Codec.v210, Codec.RG48, Codec.R12L):
            ls = vc_get_linesize(w, codec)
            src = torch.randint(0, 256, (ls * h,), dtype=torch.uint8, device="cuda")
            dst = torch.empty_like(src)
            cases.append((f"deinterlace_ex {codec.name} {w}x{h} out of place", ls * h,
                          lambda c=codec, s=src, d=dst, ls=ls, h=h: api.deinterlace_ex(c, s, ls, h, dst=d)))
            cases.append((f"deinterlace_ex {codec.name} {w}x{h} in place", ls * h,
                          lambda c=codec, s=src, ls=ls, h=h: api.deinterlace_ex(c, s, ls, h, dst=s)))
        for codec in (Codec.UYVY, Codec.RGB):
            ls = vc_get_linesize(w, codec)
            buf = torch.randint(0, 256, (ls * h,), dtype=torch.uint8, device="cuda")
            cases.append((f"deinterlace (legacy) {codec.name} {w}x{h} in place", ls * h, lambda b=buf, ls=ls, h=h: api.deinterlace(b, ls, h)))
        ls = vc_get_linesize(w, Codec.UYVY)
        buf = torch.randint(0, 256, (ls * h,), dtype=torch.uint8, device="cuda")
        cases.append((f"il_upper_to_merged UYVY {w}x{h} in place", ls * h, lambda b=buf, ls=ls, h=h: api.il_upper_to_merged(b, ls, h)))
        cases.append((f"il_merged_to_upper UYVY {w}x{h} in place", ls * h, lambda b=buf, ls=ls, h=h: api.il_merged_to_upper(b, ls, h)))
    for name, nbytes, fn in cases:
        us = timed(fn, args.iters, args.warmup)
        gbs = 2 * nbytes / (us * 1e-6) / 1e9
        print(f"{name:52s} {us:9.1f} us  {gbs:7.0f} GB/s")
        if args.json:
            print(json.dumps({"case": name, "us_per_frame": round(us, 2), "compulsory_GBps": round(gbs, 1)}))


if __name__ == "__main__":
    main()
