"""Timing of the colour capture filters (ugb200_cf_*, colour_filter_kernels.cu) on device-resident frames, with
ugb200_pixfmt_convert UYVY -> RGB as the same-run streaming baseline.

  gamma      RGB and RG48 in, 8- and 16-bit out (the four tables)
  matrix     UYVY -> RGB, RGB, RG48, with and without bounds checking
  matrix2    UYVY, v210, Y416
  grayscale  UYVY

at 4K and 8K, on random frames (so the gamma gathers hit random table entries).  Each case: --warmup launches, then
CUDA events around --iters (>= 64) back-to-back launches on one stream; the time per frame is the mean.  TB/s counts
compulsory bytes only: the input frame read once plus the output frame written once.  Prints the card name and
power limit read in the same run.

    python tools/colour_filter_bench.py [--iters N] [--warmup N] [--json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = ((3840, 2160), (7680, 4320))


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
    assert args.iters >= 64
    import torch
    from ultragrid_b200 import Codec, api, vc_get_linesize
    assert torch.cuda.is_available(), "colour_filter_bench.py needs a GPU"
    print("card:", card())
    m = (0.9, 0.05, 0.1, -0.2, 1.1, 0.05, 0.3, -0.1, 0.95)
    g = api.gamma(1 / 2.2)
    cases = []
    for w, h in SIZES:
        frames = {c: torch.randint(0, 256, (vc_get_linesize(w, c) * h,), dtype=torch.uint8, device="cuda")
                  for c in (Codec.UYVY, Codec.RGB, Codec.RG48, Codec.v210, Codec.Y416)}
        out = torch.empty(w * h * 8, dtype=torch.uint8, device="cuda")
        F = {c: t.numel() for c, t in frames.items()}
        n = f"{w}x{h}"
        s = frames[Codec.UYVY]
        cases.append((f"pixfmt_convert UYVY->RGB (baseline) {n}", F[Codec.UYVY] + F[Codec.RGB],
                      lambda s=s, w=w, h=h: api.pixfmt_convert(Codec.UYVY, Codec.RGB, s, w, h, dst=out)))
        cases.append((f"grayscale UYVY {n}", 2 * F[Codec.UYVY], lambda s=s, w=w, h=h: api.grayscale(s, w, h, dst=out)))
        for c in (Codec.RGB, Codec.RG48):
            for d in (8, 16):
                ob = F[Codec.RGB] if d == 8 else F[Codec.RG48]
                cases.append((f"gamma {c.name}->{d}-bit {n}", F[c] + ob, lambda c=c, d=d, w=w, h=h: g(c, frames[c], w, h, d, dst=out)))
        for c in (Codec.UYVY, Codec.RGB, Codec.RG48):
            ob = F[Codec.RGB] if c == Codec.UYVY else F[c]
            for b in (True, False):
                cases.append((f"matrix {c.name}{'' if b else ' no-bound-check'} {n}", F[c] + ob,
                              lambda c=c, b=b, w=w, h=h: api.matrix(c, frames[c], w, h, m, b, dst=out)))
        for c in (Codec.UYVY, Codec.v210, Codec.Y416):
            cases.append((f"matrix2 {c.name} {n}", 2 * F[c], lambda c=c, w=w, h=h: api.matrix2(c, frames[c], w, h, m, dst=out)))
    for name, nbytes, fn in cases:
        us = timed(fn, args.iters, args.warmup)
        tbs = nbytes / (us * 1e-6) / 1e12
        print(f"{name:48s} {us:9.1f} us  {nbytes / 1e6:8.1f} MB  {tbs:5.2f} TB/s")
        if args.json:
            print(json.dumps({"case": name, "us_per_frame": round(us, 2), "compulsory_MB": round(nbytes / 1e6, 2), "TBps": round(tbs, 3)}))


if __name__ == "__main__":
    main()
