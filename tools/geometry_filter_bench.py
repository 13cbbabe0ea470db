"""Timing of the geometry filters (ugb200_cf_flip / _mirror / _crop / _split, ugb200_pp_border / _interlaced_3d,
geometry_kernels.cu) on device-resident 7680x4320 frames, each against a device-to-device cudaMemcpy2DAsync of the
same compulsory bytes in the same run.

  flip, interlaced_3d   UYVY, RGB, v210
  mirror                UYVY
  crop                  a 3840x2160 window at xoff 1001 (odd and off every pixel block), yoff 17; UYVY, RGB, v210
  split                 2x2 and 4x4 tiles; UYVY, RGB, v210
  border                UYVY, RGB (the default 10-pixel border)

Each case: --warmup launches, then CUDA events around --iters (>= 64) back-to-back launches on one stream; the filter
and its copy baseline alternate for --rounds rounds and the best round of each is kept.  Compulsory bytes: the output
frame written once plus the bytes it is computed from read once (interlaced_3d reads both eye tiles).  Prints the card
name and power limit read in the same run.

    python tools/geometry_filter_bench.py [--iters N] [--warmup N] [--rounds N] [--json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def cudart():
    for name in ("libcudart.so.12", "libcudart.so"):
        try:
            return ctypes.CDLL(name)
        except OSError:
            pass
    import glob
    import torch
    for p in glob.glob(os.path.join(os.path.dirname(torch.__file__), "..", "nvidia", "cuda_runtime", "lib", "libcudart.so*")):
        return ctypes.CDLL(p)
    raise RuntimeError("libcudart not found")


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
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", action="store_true")
    args = ap.parse_args()
    assert args.iters >= 64
    import torch
    import geometry_filter_ref as R
    from ultragrid_b200 import api
    assert torch.cuda.is_available(), "geometry_filter_bench.py needs a GPU"
    print("card:", card())
    rt = cudart()
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    rt.cudaMemcpy2DAsync.argtypes = [vp, sz, vp, sz, sz, sz, ctypes.c_int, vp]
    w, h = 7680, 4320
    frames = {c: torch.randint(0, 256, (R.linesize(w, c) * h,), dtype=torch.uint8, device="cuda") for c in (R.UYVY, R.RGB, R.v210)}
    right = {c: torch.randint(0, 256, (t.numel(),), dtype=torch.uint8, device="cuda") for c, t in frames.items()}
    out = torch.empty(max(t.numel() for t in frames.values()) + 4096, dtype=torch.uint8, device="cuda")
    base_dst = torch.empty_like(out)

    def copy2d(src, spitch, width, rows):
        st = vp(torch.cuda.current_stream().cuda_stream)
        return lambda: rt.cudaMemcpy2DAsync(vp(base_dst.data_ptr()), width, vp(src.data_ptr()), spitch, width, rows, 3, st)

    cases = []  # (name, compulsory bytes, filter, baseline)
    for c in (R.UYVY, R.RGB, R.v210):
        s, L, nm = frames[c], R.linesize(w, c), R.NAMES[c]
        cases.append((f"flip {nm}", 2 * L * h, lambda c=c, s=s: api.flip(c, s, w, h, dst=out), copy2d(s, L, L, h)))
        if c == R.UYVY:
            cases.append((f"mirror {nm}", 2 * L * h, lambda c=c, s=s: api.mirror(c, s, w, h, dst=out), copy2d(s, L, L, h)))
        ow, oh, _, _ = R.crop_geometry(c, w, h, 3840, 2160, 1001, 17)
        p = R.linesize(ow, c)
        cases.append((f"crop {nm} 3840x2160+1001+17", 2 * p * oh, lambda c=c, s=s: api.crop(c, s, w, h, 3840, 2160, 1001, 17, dst=out),
                      copy2d(s, L, p, oh)))
        for x in (2, 4):
            tiles = api.split(c, s, w, h, x, x)
            n = int((w // x) * R.bpp(c))
            cases.append((f"split {nm} {x}x{x}", 2 * n * x * h, lambda c=c, s=s, x=x, t=tiles: api.split(c, s, w, h, x, x, tiles=t),
                          copy2d(s, L, n * x, h)))
        if c != R.v210:
            cases.append((f"border {nm}", 2 * L * h, lambda c=c, s=s: api.border(c, s, w, h, dst=out), copy2d(s, L, L, h)))
        cases.append((f"interlaced_3d {nm}", 3 * L * h, lambda c=c, s=s: api.interlaced_3d(c, s, right[c], w, h, dst=out),
                      copy2d(s, L, L, h)))
    for name, nbytes, fn, base in cases:
        tf, tb = float("inf"), float("inf")
        for _ in range(args.rounds):
            tf = min(tf, timed(fn, args.iters, args.warmup))
            tb = min(tb, timed(base, args.iters, args.warmup))
        tbs = nbytes / (tf * 1e-6) / 1e12
        print(f"{name:34s} {tf:8.1f} us  {tbs:5.2f} TB/s   copy2D {tb:8.1f} us  {nbytes / (tb * 1e-6) / 1e12:5.2f} TB/s   ratio {tf / tb:5.2f}")
        if args.json:
            print(json.dumps({"case": name, "us": round(tf, 2), "copy2d_us": round(tb, 2), "compulsory_MB": round(nbytes / 1e6, 2),
                              "TBps": round(tbs, 3)}))


if __name__ == "__main__":
    main()
