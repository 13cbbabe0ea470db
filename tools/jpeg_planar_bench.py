"""Times the planar JPEG layouts (ugb200_jpeg_encode_device_ex) at 8K, q = 90, on the natural test frame:
I420 -> 4:2:0, UYVY -> 4:2:0, RGB -> Y709 4:2:0 per component and interleaved, RGB -> Y601full 4:2:0.

Every variant is warmed up, then the variants alternate over interleaved rounds (CUDA events around a window of encodes on the
encoder's stream) and the medians are reported.  A second, separate run records a torch.profiler trace and sums the device time by
kernel name: pre-processing, DCT, Huffman, offset scan, compaction.  RGB-interleaved against I420 (the same planes read in place)
isolates the cost of the pre-processing pass.  Prints one JSON object; with --out DIR also writes it to DIR/jpeg_planar_bench.json."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

UYVY, RGB, I420 = 2, 12, 29
VARIANTS = {  # name: (input codec, subsampling, colour space, interleaved)
    "i420_420": (I420, 0, 0, 1),
    "uyvy_420": (UYVY, 420, 0, 1),
    "rgb_y709_420": (RGB, 420, 3, 0),
    "rgb_y709_420_interleaved": (RGB, 420, 3, 1),
    "rgb_y601full_420": (RGB, 420, 2, 0),
}
KERNELS = {"prep": "jpeg_prep_kernel", "dct": "jpeg_dct_kernel", "huffman": "jpeg_huffman_kernel", "scan": "jpeg_scan_kernel", "compact": "jpeg_compact_kernel"}


def frames(w, h):
    import util
    from test_jpeg import natural_rgb
    orc = util.oracle()
    rgb = np.ascontiguousarray(natural_rgb(w, h, 1)).reshape(-1)
    uyvy = util.convert_cpu(orc, "orc_convert", RGB, UYVY, rgb, w, h)
    from test_jpeg_planar import orc_uyvy_to_i420
    cw, ch = (w + 1) // 2, (h + 1) // 2
    planes = [np.zeros(w * h, np.uint8), np.zeros(cw * ch, np.uint8), np.zeros(cw * ch, np.uint8)]
    orc_uyvy_to_i420(orc, uyvy, w, h, planes)
    return {RGB: rgb, UYVY: uyvy, I420: np.concatenate(planes)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=7680)
    ap.add_argument("--height", type=int, default=4320)
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--window", type=int, default=20, help="encodes per timed window")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from ultragrid_b200 import api
    w, h = args.width, args.height
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    enc = api.JpegEncoder(stream)
    src = {k: torch.from_numpy(v).cuda() for k, v in frames(w, h).items()}

    def run(name, n):
        codec, sub, cs, il = VARIANTS[name]
        for _ in range(n):
            enc.encode_device(src[codec], w, h, codec, quality=90, interleaved=bool(il), subsampling=sub, color_space=cs)
        return enc.result_size()

    sizes = {name: run(name, 3) for name in VARIANTS}  # warm-up of every shape
    times = {name: [] for name in VARIANTS}
    for r in range(args.rounds):
        order = list(VARIANTS) if r % 2 == 0 else list(reversed(VARIANTS))
        for name in order:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record(stream)
            run(name, args.window)
            b.record(stream)
            b.synchronize()
            times[name].append(a.elapsed_time(b) * 1000.0 / args.window)
    result = {"frame": [w, h], "quality": 90,
              "us_per_frame_median": {k: round(statistics.median(v), 1) for k, v in times.items()},
              "us_spread": {k: [round(min(v), 1), round(max(v), 1)] for k, v in times.items()},
              "stream_bytes": sizes}
    # per-kernel device time in a profiled run of its own
    from torch.profiler import ProfilerActivity, profile
    per = {}
    for name in VARIANTS:
        run(name, 2)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(name, 5)
            torch.cuda.synchronize()
        acc = {k: 0.0 for k in KERNELS}
        for ev in prof.key_averages():
            for k, kn in KERNELS.items():
                if kn in ev.key:
                    acc[k] += ev.device_time_total / 5.0
        per[name] = {k: round(v, 1) for k, v in acc.items()}
    result["profiler_us_per_frame"] = per
    try:
        result["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        result["gpu"] = "unknown"
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "jpeg_planar_bench.json"), "w") as f:
            f.write(line + "\n")
    enc.close()


if __name__ == "__main__":
    main()
