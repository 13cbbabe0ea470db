"""BT.709 against BT.601 on the colour converters at 8K: ugb200_pixfmt_convert_cs / ugb200_to_lavc_convert_cs with UGB_CS_709 and UGB_CS_601,
alternating in one process, timed with CUDA events.  The two instantiations differ in immediates only, so the expectation is equal times.

    python tools/color601_bench.py [--rounds 7] [--iters 200]

Prints one JSON line: the card, its power limit, and per conversion the median microseconds per frame of each colour space over the rounds."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from ultragrid_b200 import api, vc_get_linesize  # noqa: E402
from ultragrid_b200.codec import Codec  # noqa: E402

W, H = 7680, 4320
CASES = [("UYVY->RGB", Codec.UYVY, Codec.RGB), ("RGB->UYVY", Codec.RGB, Codec.UYVY), ("v210->RGB", Codec.v210, Codec.RGB),
         ("RG48->v210", Codec.RG48, Codec.v210), ("RGB->YUV444P", Codec.RGB, "YUV444P")]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    name, limit = q.stdout.strip().splitlines()[0].rsplit(",", 1)
    return name.strip(), limit.strip()


def runner(inc, out):
    src = torch.randint(0, 256, (vc_get_linesize(W, inc) * H,), dtype=torch.uint8, device="cuda")
    if out == "YUV444P":
        planes = [torch.empty(ls * rows, dtype=torch.uint8, device="cuda") for ls, rows in api.av_plane_shapes(out, W, H)]
        return lambda cs: api.to_lavc(inc, out, src, W, H, planes=planes, cs=cs)
    dst = torch.empty(vc_get_linesize(W, out) * H, dtype=torch.uint8, device="cuda")
    return lambda cs: api.pixfmt_convert(inc, out, src, W, H, dst=dst, cs=cs)


def time_us(fn, cs, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn(cs)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1000.0 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    name, limit = card()
    result = {"gpu": name, "power_limit": limit, "size": f"{W}x{H}", "iters": args.iters, "rounds": args.rounds, "us_per_frame": {}}
    for label, inc, out in CASES:
        fn = runner(inc, out)
        for cs in (api.CS_709, api.CS_601):  # warm-up: module load, first launch of each instantiation
            time_us(fn, cs, 10)
        t = {api.CS_709: [], api.CS_601: []}
        for r in range(args.rounds):
            for cs in ((api.CS_709, api.CS_601) if r % 2 == 0 else (api.CS_601, api.CS_709)):
                t[cs].append(time_us(fn, cs, args.iters))
        result["us_per_frame"][label] = {"bt709": round(statistics.median(t[api.CS_709]), 2), "bt601": round(statistics.median(t[api.CS_601]), 2),
                                         "bt709_spread": round(max(t[api.CS_709]) - min(t[api.CS_709]), 2),
                                         "bt601_spread": round(max(t[api.CS_601]) - min(t[api.CS_601]), 2)}
        del fn
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
