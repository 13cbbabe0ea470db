"""Times the RGBA layouts of the JPEG stage (ugb200_jpeg_encode_device_ex with UGB_RGBA, subsampling 4444: the GPUJPEG module's `alpha`
stream) at 8K, q = 90, on the natural test frame with a natural alpha plane (a soft-edged key shape, tests/test_jpeg_alpha.py:rgba_frame):
  rgb          RGB, three scans (the existing layout, for comparison)
  rgba         RGBA 4444, four scans, fused kernel (the default)
  rgba_il      RGBA 4444, one interleaved scan, split path
  decode_rgba  the four-scan stream decoded to RGBA on the host stream (wall clock around a synchronous decode, as bench.py's decode records)

Every variant is warmed up, then the variants alternate over interleaved rounds and the medians are reported (encodes: CUDA events around a
window of encodes on the encoder's stream).  A second, separate run records a torch.profiler trace and sums the device time per kernel.
The card's name and power limit are read in the same run.  Prints one JSON object; with --out DIR also writes it to DIR/jpeg_alpha_bench.json."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

RGB, RGBA = 12, 1
ENCODES = {"rgb": (RGB, 0, 0), "rgba": (RGBA, 4444, 0), "rgba_il": (RGBA, 4444, 1)}  # name: (codec, subsampling, interleaved)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=7680)
    ap.add_argument("--height", type=int, default=4320)
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--window", type=int, default=20, help="encodes per timed window")
    ap.add_argument("--decodes", type=int, default=5, help="decodes per timed window")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from test_jpeg_alpha import rgba_frame
    from ultragrid_b200 import api
    w, h = args.width, args.height
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    enc = api.JpegEncoder(stream)
    f = rgba_frame(w, h, 1)
    src = {RGB: torch.from_numpy(np.ascontiguousarray(f[..., :3]).reshape(-1)).cuda(), RGBA: torch.from_numpy(f.reshape(-1)).cuda()}

    def run(name, n):
        codec, sub, il = ENCODES[name]
        for _ in range(n):
            enc.encode_device(src[codec], w, h, codec, quality=90, interleaved=bool(il), subsampling=sub)
        return enc.result_size()

    sizes = {name: run(name, 3) for name in ENCODES}  # warm-up of every shape
    run("rgba", 1)
    stream4 = enc.result()  # the four-scan stream for the decode
    dec = api.JpegDecoder()
    for _ in range(3):
        dec.decode(stream4, RGBA)
    times = {name: [] for name in list(ENCODES) + ["decode_rgba"]}
    for r in range(args.rounds):
        order = list(times) if r % 2 == 0 else list(reversed(list(times)))
        for name in order:
            if name == "decode_rgba":
                t0 = time.perf_counter()
                for _ in range(args.decodes):
                    dec.decode(stream4, RGBA)  # host destination: synchronous
                times[name].append((time.perf_counter() - t0) * 1e6 / args.decodes)
                continue
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
    for name in list(ENCODES) + ["decode_rgba"]:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                if name == "decode_rgba":
                    dec.decode(stream4, RGBA)
                else:
                    run(name, 1)
            torch.cuda.synchronize()
        acc = {}
        for ev in prof.key_averages():
            if ev.device_time_total > 0:
                k = ev.key.split("<")[0].split("(")[0].replace("void ", "").replace("ugb::", "")
                acc[k] = acc.get(k, 0.0) + ev.device_time_total / 5.0
        per[name] = {k: round(v, 1) for k, v in sorted(acc.items(), key=lambda kv: -kv[1])}
    result["profiler_us_per_frame"] = per
    try:
        result["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        result["gpu"] = "unknown"
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "jpeg_alpha_bench.json"), "w") as fh:
            fh.write(line + "\n")
    enc.close(), dec.close()


if __name__ == "__main__":
    main()
