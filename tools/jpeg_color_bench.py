"""JPEG decode to RGB: the fused kernel of ugb200_jpeg_decode (IDCT, chroma replication and the UYVY -> RGB line converter in one pass) against
decode(UYVY) followed by ugb200_pixfmt_convert(UYVY -> RGB), the two-pass form the fused kernel replaces.

Workloads: natural frames at 1080p, 4K and 8K, q 90, as 4:2:0 (PIL / libjpeg, no DRI) and 4:2:2 (this project's encoder, restart interval 4) streams,
decoded to a device RGB buffer.  In one process, for each workload:
  * wall clock (profiler off): the two routes alternating, each call synchronised, median of --reps;
  * kernel times: torch.profiler with CUDA activities in a run of its own, summed per kernel name over --prof-reps calls of each route;
  * the outputs of both routes are compared byte for byte.
Also decode_cs(Y601full) to RGB (the colour-space epilogue) as a third timed route.  Prints one JSON line per workload and the card name and power
limit read in the same run.

    python tools/jpeg_color_bench.py [--reps N] [--prof-reps N] [--out DIR] [--quick]
"""
import argparse
import io
import json
import os
import subprocess
import sys
import time
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def workloads(quick):
    import torch
    from PIL import Image
    from test_jpeg import natural_rgb
    from ultragrid_b200 import Codec, api
    enc = api.JpegEncoder()
    sizes = [(1920, 1080), (3840, 2160)] + ([] if quick else [(7680, 4320)])
    out = []
    for w, h in sizes:
        rgb = natural_rgb(w, h, 5)
        b = io.BytesIO()
        Image.fromarray(rgb).save(b, "JPEG", quality=90, subsampling=2)
        out.append((f"{w}x{h} 420 q90 (PIL)", b.getvalue(), w, h))
        uyvy = api.pixfmt_convert(Codec.RGB, Codec.UYVY, torch.from_numpy(rgb.reshape(-1)).cuda(), w, h)
        enc.encode_device(uyvy, w, h, Codec.UYVY, quality=90)
        out.append((f"{w}x{h} 422 q90 (this encoder)", bytes(enc.result()), w, h))
    enc.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--prof-reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true")
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from ultragrid_b200 import Codec, api
    assert torch.cuda.is_available(), "needs a GPU"
    dev_card = card()
    print(json.dumps({"card": dev_card}), flush=True)
    dec = api.JpegDecoder()
    rows = []
    for name, s, w, h in workloads(a.quick):
        rgb = torch.empty(w * 3 * h, dtype=torch.uint8, device="cuda")
        rgb2 = torch.empty_like(rgb)
        uy = torch.empty((w + 1) // 2 * 4 * h, dtype=torch.uint8, device="cuda")

        def fused():
            dec.decode(s, Codec.RGB, device=True, out=rgb, sync=False)

        def two_pass():
            dec.decode(s, Codec.UYVY, device=True, out=uy, sync=False)
            api.pixfmt_convert(Codec.UYVY, Codec.RGB, uy, w, h, dst=rgb2)

        def cs601():
            dec.decode(s, Codec.RGB, device=True, out=rgb, sync=False, color_space="Y601full")

        routes = {"fused": fused, "two_pass": two_pass, "cs_y601full": cs601}
        for f in routes.values():  # warm-up, every shape of the timed window
            f()
            f()
        torch.cuda.synchronize()
        fused()
        two_pass()
        torch.cuda.synchronize()
        assert torch.equal(rgb, rgb2), name
        t = defaultdict(list)
        for _ in range(a.reps):
            for r, f in routes.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                f()
                torch.cuda.synchronize()
                t[r].append((time.perf_counter() - t0) * 1e3)
        kern = {}
        for r in ("fused", "two_pass"):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.prof_reps):
                    routes[r]()
                torch.cuda.synchronize()
            per = defaultdict(float)
            for e in prof.events():
                if e.device_type.name == "CUDA" and ("jpeg_idct" in e.name or "line_conv" in e.name):
                    per[e.name.split("(")[0].split("<")[0]] += e.device_time / a.prof_reps
            kern[r] = {k: round(v, 1) for k, v in per.items()}
        row = {"workload": name, "bytes": len(s), "ms_fused": round(float(np.median(t["fused"])), 3),
               "ms_two_pass": round(float(np.median(t["two_pass"])), 3), "ms_cs_y601full": round(float(np.median(t["cs_y601full"])), 3),
               "us_kernels_fused": kern["fused"], "us_kernels_two_pass": kern["two_pass"]}
        rows.append(row)
        print(json.dumps(row), flush=True)
    dec.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "jpeg_color_bench.json"), "w") as f:
            json.dump({"card": dev_card, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
