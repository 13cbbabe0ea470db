"""Timing of the field-rate postprocessors (ugb200_pp_*, interlace_kernels.cu) on device-resident frames, with
ugb200_vc_deinterlace_ex as the same-run baseline.

  bob, linear      every linear layout (UYVY, RG48, v210, R10k, R12L), calls 0 and 1
  double_framerate calls 0 and 1; `:d` fused (one pass) against composed (weave, then vc_deinterlace_ex in place)
  interlace        UYVY
  deinterlace_ex   UYVY, v210, RG48, R12L out of place

at 4K and 8K.  Each case: --warmup launches, then CUDA events around --iters (>= 32) back-to-back launches on one
stream; the time per frame is the mean.  TB/s counts compulsory bytes only, computed from the shapes (F = one frame,
linesize * height): bob and linear 1.5 F (read the field, write the frame), weave, interlace and fused `:d` 2 F,
composed `:d` 4 F, deinterlace_ex 2 F.  Prints the card name and power limit read in the same run.

    python tools/field_rate_bench.py [--iters N] [--warmup N] [--json]
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
    assert args.iters >= 32
    import torch
    from ultragrid_b200 import Codec, api, vc_get_linesize
    assert torch.cuda.is_available(), "field_rate_bench.py needs a GPU"
    print("card:", card())
    cases = []
    for w, h in SIZES:
        bufs = {}
        for codec in (Codec.UYVY, Codec.RG48, Codec.v210, Codec.R10k, Codec.R12L):
            L = vc_get_linesize(w, codec)
            prev = torch.randint(0, 256, (L * h,), dtype=torch.uint8, device="cuda")
            cur = torch.randint(0, 256, (L * h,), dtype=torch.uint8, device="cuda")
            dst = torch.empty_like(cur)
            bufs[codec] = (L, prev, cur, dst)
            F = L * h
            n = f"{codec.name} {w}x{h}"
            for call in (0, 1):
                cases.append((f"bob call {call} {n}", 1.5 * F, lambda q=cur, d=dst, L=L, c=call, h=h: api.deinterlace_bob(q, L, h, c, dst=d)))
                cases.append((f"linear call {call} {n}", 1.5 * F,
                              lambda k=codec, q=cur, d=dst, L=L, c=call, h=h: api.deinterlace_linear(k, q, L, h, c, dst=d)))
        for codec in (Codec.UYVY, Codec.v210, Codec.RG48, Codec.R12L):
            L, prev, cur, dst = bufs[codec]
            F = L * h
            n = f"{codec.name} {w}x{h}"
            for call in (0, 1):
                cases.append((f"double_framerate call {call} {n}", 2 * F,
                              lambda k=codec, p=prev, q=cur, d=dst, L=L, c=call, h=h: api.double_framerate(k, p, q, L, h, c, dst=d)))
            cases.append((f"double_framerate:d call 0 fused {n}", 2 * F,
                          lambda k=codec, p=prev, q=cur, d=dst, L=L, h=h: api.double_framerate(k, p, q, L, h, 0, True, dst=d)))

            def composed(k=codec, p=prev, q=cur, d=dst, L=L, h=h):
                api.double_framerate(k, p, q, L, h, 0, dst=d)
                api.deinterlace_ex(k, d, L, h, dst=d)
            cases.append((f"double_framerate:d call 0 composed {n}", 4 * F, composed))
            cases.append((f"deinterlace_ex (baseline) {n}", 2 * F,
                          lambda k=codec, q=cur, d=dst, L=L, h=h: api.deinterlace_ex(k, q, L, h, dst=d)))
        L, prev, cur, dst = bufs[Codec.UYVY]
        cases.append((f"interlace UYVY {w}x{h}", 2 * L * h, lambda p=prev, q=cur, d=dst, L=L, h=h: api.interlace(q, p, L, h, dst=d)))
    for name, nbytes, fn in cases:
        us = timed(fn, args.iters, args.warmup)
        tbs = nbytes / (us * 1e-6) / 1e12
        print(f"{name:48s} {us:9.1f} us  {nbytes / 1e6:8.1f} MB  {tbs:5.2f} TB/s")
        if args.json:
            print(json.dumps({"case": name, "us_per_frame": round(us, 2), "compulsory_MB": round(nbytes / 1e6, 2), "TBps": round(tbs, 3)}))


if __name__ == "__main__":
    main()
