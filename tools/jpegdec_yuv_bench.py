"""JPEG decode to YCbCr video: what the routes of ugb200_jpeg_decode_to cost, on the GPU (fails without one).

For 4K and 8K natural frames at q 90, decoded into device buffers, CUDA events around the whole decode call (upload, marker scan, Huffman, IDCT
and packing kernels) over enough calls to fill about --seconds, after a warm-up, the routes of a comparison alternating call by call:
  (a) 4:2:0 -> I420: the fused kernel's planar epilogue against decode to UYVY + ugb200_uyvy_to_i420 (the route it replaced);
  (b) 4:2:2 JFIF -> UYVY: with the Y601FULL -> Y709 matrix against the plain UYVY epilogue (the cost of the conversion);
  (c) grayscale -> UYVY (the two-warp form of the fused kernel), alone.
Also torch.profiler kernel times of the fused IDCT kernel per route, in a run of its own.  The outputs of (a) are compared byte for byte.  Bytes
moved by the IDCT / packing stage are computed from the shapes: coefficients read (2 B per sample of the padded planes) plus the frame written, plus,
for the two-pass route, the UYVY frame written and read again.  Prints the card's name, power limit and max SM clock, then one JSON line per comparison.

    python tools/jpegdec_yuv_bench.py [--seconds S] [--quick] [--out DIR]
"""
import argparse
import io
import json
import os
import subprocess
import sys
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def pil(img, mode=None, **kw):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(img, mode).save(b, "JPEG", quality=90, **kw)
    return b.getvalue()


def timed(torch, routes, seconds):
    """alternates the routes; returns median ms per call of each (CUDA events, each call synchronised before the next route starts)"""
    for f in routes.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    t = defaultdict(list)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    spent = 0.0
    while spent < seconds * 1e3 * len(routes):
        for name, f in routes.items():
            a, b = ev(), ev()
            a.record()
            f()
            b.record()
            b.synchronize()
            t[name].append(a.elapsed_time(b))
            spent += t[name][-1]
    return {k: (round(float(np.median(v)), 4), len(v)) for k, v in t.items()}


def idct_kernel_us(torch, f, reps=5):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            f()
        torch.cuda.synchronize()
    per = defaultdict(float)
    for e in prof.events():
        if e.device_type.name == "CUDA" and ("jpeg_idct" in e.name or "planar" in e.name.lower() or "i420" in e.name.lower()):
            per[e.name.split("(")[0][:60]] += e.device_time / reps
    return {k: round(v, 1) for k, v in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--quick", action="store_true", help="4K only")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("jpegdec_yuv_bench: needs a GPU")
    from test_jpeg import natural_rgb
    from ultragrid_b200 import Codec, api
    dev_card = card()
    print(json.dumps({"card (name, power limit, max SM clock)": dev_card}), flush=True)
    dec = api.JpegDecoder()
    rows = []
    for w, h in [(3840, 2160)] + ([] if a.quick else [(7680, 4320)]):
        rgb = natural_rgb(w, h, 5)
        s420, s422, sgray = pil(rgb, subsampling=2), pil(rgb, subsampling=1), pil(rgb[:, :, 1].copy(), "L")
        px = w * h
        uy = torch.empty((w + 1) // 2 * 4 * h, dtype=torch.uint8, device="cuda")
        i420 = torch.empty(px + 2 * ((w + 1) // 2) * ((h + 1) // 2), dtype=torch.uint8, device="cuda")
        i420b = torch.empty_like(i420)
        cw, ch = (w + 1) // 2, (h + 1) // 2
        planes = [i420b[:px], i420b[px:px + cw * ch], i420b[px + cw * ch:]]

        def direct():
            dec.decode(s420, Codec.I420, device=True, out=i420, sync=False)

        def two_pass():
            dec.decode(s420, Codec.UYVY, device=True, out=uy, sync=False)
            api.to_planar("uyvy_to_i420", uy, w, h, planes, [w, cw, cw])

        direct(), two_pass()
        torch.cuda.synchronize()
        assert torch.equal(i420, i420b), "planar epilogue differs from UYVY + uyvy_to_i420"
        ta = timed(torch, {"direct": direct, "two_pass": two_pass}, a.seconds)
        rows.append({"case": f"(a) {w}x{h} 4:2:0 -> I420", "stream_bytes": len(s420), "ms_per_call (median, calls)": ta,
                     "bytes_idct_stage": {"direct": int(px * 1.5 * 2 + px * 1.5), "two_pass": int(px * 1.5 * 2 + px * 2 + px * 2 + px * 1.5)},
                     "us_kernels": {"direct": idct_kernel_us(torch, direct), "two_pass": idct_kernel_us(torch, two_pass)}})
        print(json.dumps(rows[-1]), flush=True)

        def plain():
            dec.decode(s422, Codec.UYVY, device=True, out=uy, sync=False)

        def matrix():
            dec.decode_to(s422, Codec.UYVY, "Y601full", "Y709", device=True, out=uy, sync=False)

        tb = timed(torch, {"plain": plain, "matrix": matrix}, a.seconds)
        rows.append({"case": f"(b) {w}x{h} 4:2:2 JFIF -> UYVY", "stream_bytes": len(s422), "ms_per_call (median, calls)": tb,
                     "bytes_idct_stage": {"plain": px * 2 * 2 + px * 2, "matrix": px * 2 * 2 + px * 2},
                     "us_kernels": {"plain": idct_kernel_us(torch, plain), "matrix": idct_kernel_us(torch, matrix)}})
        print(json.dumps(rows[-1]), flush=True)

        def gray():
            dec.decode_to(sgray, Codec.UYVY, "native", "native", device=True, out=uy, sync=False)

        tc = timed(torch, {"gray": gray}, a.seconds)
        rows.append({"case": f"(c) {w}x{h} grayscale -> UYVY", "stream_bytes": len(sgray), "ms_per_call (median, calls)": tc,
                     "bytes_idct_stage": {"gray": px * 2 + px * 2}, "us_kernels": {"gray": idct_kernel_us(torch, gray)}})
        print(json.dumps(rows[-1]), flush=True)
    dec.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "jpegdec_yuv_bench.json"), "w") as f:
            json.dump({"card": dev_card, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
