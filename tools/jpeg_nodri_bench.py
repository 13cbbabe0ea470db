"""JPEG decode of streams with long or no restart intervals: the self-synchronising Huffman route against one thread per restart segment.

For every workload (PIL / libjpeg streams of the natural test frames at 1080p, 4K and 8K, 4:2:0 and 4:2:2, q 75 and 90, without DRI, with one MCU
row per interval and with 4 MCUs per interval, and an 8K noise frame) the wall clock of ugb200_jpeg_decode to a device buffer (synchronised) is
taken with the route forced on (UGB200_JPEG_SYNC=on), forced off (=off, what the parent decoder did) and as selected, the three alternating in one
process; also the subsequences and rounds, and PIL's CPU decode of the same stream.  Prints one JSON line per workload and the card name and
power limit read in the same run.

    python tools/jpeg_nodri_bench.py [--reps N] [--out DIR] [--quick]
"""
import argparse
import io
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def workloads(quick):
    from PIL import Image
    from test_jpeg import natural_rgb
    sizes = [(1920, 1080), (3840, 2160)] + ([] if quick else [(7680, 4320)])
    out = []
    for w, h in sizes:
        rgb = natural_rgb(w, h, 5)
        for ss, ssn in ((2, "420"), (1, "422")):
            for q in (75, 90):
                for dri, kw in (("none", {}), ("row", {"restart_marker_rows": 1}), ("4mcu", {"restart_marker_blocks": 4})):
                    if dri != "none" and q != 90:
                        continue
                    b = io.BytesIO()
                    Image.fromarray(rgb).save(b, "JPEG", quality=q, subsampling=ss, **kw)
                    out.append((f"{w}x{h} {ssn} q{q} dri={dri}", b.getvalue()))
    if not quick:
        noise = np.random.default_rng(3).integers(0, 256, (4320, 7680, 3), dtype=np.uint8)
        b = io.BytesIO()
        Image.fromarray(noise).save(b, "JPEG", quality=90, subsampling=2)
        out.append(("7680x4320 420 q90 noise dri=none", b.getvalue()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true")
    a = ap.parse_args()
    import torch
    from PIL import Image
    from ultragrid_b200 import api, Codec
    assert torch.cuda.is_available(), "needs a GPU"
    print(json.dumps({"card": card()}), flush=True)
    decs = {}
    for mode in ("on", "off", "auto"):
        if mode == "auto":
            os.environ.pop("UGB200_JPEG_SYNC", None)
        else:
            os.environ["UGB200_JPEG_SYNC"] = mode
        decs[mode] = api.JpegDecoder()
    os.environ.pop("UGB200_JPEG_SYNC", None)
    rows = []
    for name, s in workloads(a.quick):
        info = api.jpeg_image_info(s)
        out = torch.empty(((info.width + 1) // 2 * 4) * info.height, dtype=torch.uint8, device="cuda")
        ref = None
        t = {m: [] for m in decs}
        stats = {}
        serial_big = len(s) > (4 << 20)
        for rep in range(a.reps + 1):
            for m, d in decs.items():
                if m == "off" and serial_big and rep > 2:
                    continue  # one thread for the whole scan: seconds per frame
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                d.decode(s, Codec.UYVY, device=True, out=out)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                if rep:
                    t[m].append(dt * 1e3)
                if ref is None:
                    ref = out.clone()
                elif rep == 0:
                    assert torch.equal(out, ref), (name, m)
                stats[m] = d.last_sync()
        t0 = time.perf_counter()
        for _ in range(3):
            Image.open(io.BytesIO(s)).load()
        pil_ms = (time.perf_counter() - t0) / 3 * 1e3
        row = {"workload": name, "bytes": len(s), "ri": info.restart_interval,
               "ms_sync": round(float(np.median(t["on"])), 3), "ms_serial": round(float(np.median(t["off"])), 3),
               "ms_selected": round(float(np.median(t["auto"])), 3), "selected_sync": stats["auto"]["scans"] > 0,
               "subsequences": stats["on"]["subsequences"], "rounds": stats["on"]["rounds"], "ms_pil_cpu": round(pil_ms, 2)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "jpeg_nodri_bench.json"), "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
