"""JPEG decode to RGB with interpolated chroma (ugb200_jpeg_decoder_set_upsampling FANCY) against replicated chroma (REPLICATE), same stream, same
colour space (Y601full), decoded into a device RGB buffer.

Workloads: natural frames at 1080p, 4K and 8K, q 90: 4:2:2 from this project's encoder (restart interval 4), 4:2:0 from PIL / libjpeg without DRI
and with a restart marker every MCU row.  In one process, for each workload:
  * wall clock (profiler off): the two modes alternating, each call synchronised, median of --reps;
  * kernel time of the fused IDCT kernel (jpeg_idct_packed_kernel): torch.profiler with CUDA activities in a run of its own per mode, mean over
    --prof-reps calls.
Prints the card name and power limit read in the same run, then one JSON line per workload.

    python tools/jpeg_fancy_bench.py [--reps N] [--prof-reps N] [--out DIR] [--quick]
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
        for name, kw in (("420 no DRI (PIL)", {}), ("420 DRI per MCU row (PIL)", {"restart_marker_rows": 1})):
            b = io.BytesIO()
            Image.fromarray(rgb).save(b, "JPEG", quality=90, subsampling=2, **kw)
            out.append((f"{w}x{h} {name}", b.getvalue(), w, h))
        uyvy = api.pixfmt_convert(Codec.RGB, Codec.UYVY, torch.from_numpy(rgb.reshape(-1)).cuda(), w, h)
        enc.encode_device(uyvy, w, h, Codec.UYVY, quality=90)
        out.append((f"{w}x{h} 422 DRI 4 (this encoder)", bytes(enc.result()), w, h))
    enc.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--prof-reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true")
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from ultragrid_b200 import Codec, api
    assert torch.cuda.is_available(), "needs a GPU"
    dev_card = card()
    print(json.dumps({"card": dev_card}), flush=True)
    decs = {"replicate": api.JpegDecoder(), "fancy": api.JpegDecoder()}
    decs["fancy"].set_upsampling("fancy")
    rows = []
    for name, s, w, h in workloads(a.quick):
        outs = {m: torch.empty(w * 3 * h, dtype=torch.uint8, device="cuda") for m in decs}
        routes = {m: (lambda m=m: decs[m].decode(s, Codec.RGB, device=True, out=outs[m], sync=False, color_space="Y601full")) for m in decs}
        for f in routes.values():  # warm-up, every shape of the timed window
            f()
            f()
        torch.cuda.synchronize()
        t = defaultdict(list)
        for _ in range(a.reps):
            for m, f in routes.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                f()
                torch.cuda.synchronize()
                t[m].append((time.perf_counter() - t0) * 1e3)
        kern = {}
        for m, f in routes.items():
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.prof_reps):
                    f()
                torch.cuda.synchronize()
            kern[m] = sum(e.device_time for e in prof.events() if e.device_type.name == "CUDA" and "jpeg_idct_packed_kernel" in e.name) / a.prof_reps
        row = {"workload": name, "bytes": len(s), "ms_replicate": round(float(np.median(t["replicate"])), 3), "ms_fancy": round(float(np.median(t["fancy"])), 3),
               "us_kernel_replicate": round(kern["replicate"], 1), "us_kernel_fancy": round(kern["fancy"], 1)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    for d in decs.values():
        d.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "jpeg_fancy_bench.json"), "w") as f:
            json.dump({"card": dev_card, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
