"""Timing of the resize filter (ugb200_cf_resize, resize_kernels.cu) on device-resident frames.

Workloads: 8K UYVY -> 1/2 linear, 8K UYVY -> 1/4 area, 4K RGB -> 1280x720 linear, 1080p UYVY -> 3840x2160 linear and
8K v210 -> 1/2 linear (the staged route: v210 -> RG48 into the handle's staging frame, then the fused kernel); then,
on ugb200_cf_resize_create2 handles, 8K UYVY -> 1/2 cubic and lanczos4, 8K UYVY -> 1/3 cubic (dense staging) and
-> 1/6 cubic (sparse: scale_x above K = 4), 4K RGB -> 1920x1080 lanczos4, 1080p UYVY -> 1280x720 area (generic, scale
1.5) and 1080p UYVY -> 3840x2160 area (upscale), each also timed as the linear call at the same geometry.  The
algorithmic bytes of a call are the source read once plus the output written once; for the staged route they also
count the staging frame written and read.  Each workload is timed against a device-to-device cudaMemcpyAsync of the
same byte count (half read, half written: n / 2 bytes copied) in the same run.

Each case: --warmup calls, then CUDA events around --iters (>= 64) back-to-back calls on one stream; a workload and its
copy alternate for --rounds rounds and the best round of each is kept.  Prints the card name and power limit read in
the same run.

    python tools/resize_bench.py [--iters N] [--warmup N] [--rounds N] [--json]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from geometry_filter_bench import card, cudart, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", action="store_true")
    args = ap.parse_args()
    assert args.iters >= 64
    import torch
    from ultragrid_b200 import api, Codec, vc_get_linesize
    assert torch.cuda.is_available(), "resize_bench.py needs a GPU"
    print("card:", card())
    rt = cudart()
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    rt.cudaMemcpyAsync.argtypes = [vp, vp, sz, ctypes.c_int, vp]

    work = [("8K UYVY -> 1/2 linear", Codec.UYVY, 7680, 4320, dict(factor=0.5, algo="linear")),
            ("8K UYVY -> 1/4 area", Codec.UYVY, 7680, 4320, dict(factor=0.25, algo="area")),
            ("4K RGB -> 1280x720 linear", Codec.RGB, 3840, 2160, dict(size=(1280, 720), algo="linear")),
            ("1080p UYVY -> 3840x2160 linear", Codec.UYVY, 1920, 1080, dict(size=(3840, 2160), algo="linear")),
            ("8K v210 -> 1/2 linear (staged)", Codec.v210, 7680, 4320, dict(factor=0.5, algo="linear")),
            ("8K UYVY -> 1/2 cubic", Codec.UYVY, 7680, 4320, dict(factor=0.5, algo="cubic")),
            ("8K UYVY -> 1/2 lanczos4", Codec.UYVY, 7680, 4320, dict(factor=0.5, algo="lanczos4")),
            ("8K UYVY -> 1/3 cubic (dense)", Codec.UYVY, 7680, 4320, dict(factor=1 / 3, algo="cubic")),
            ("8K UYVY -> 1/6 cubic (sparse)", Codec.UYVY, 7680, 4320, dict(factor=1 / 6, algo="cubic")),
            ("4K RGB -> 1920x1080 lanczos4", Codec.RGB, 3840, 2160, dict(size=(1920, 1080), algo="lanczos4")),
            ("1080p UYVY -> 1280x720 area", Codec.UYVY, 1920, 1080, dict(size=(1280, 720), algo="area")),
            ("1080p UYVY -> 3840x2160 area (up)", Codec.UYVY, 1920, 1080, dict(size=(3840, 2160), algo="area"))]
    res = []
    for name, c, w, h, kw in work:
        r = api.Resize(all_algos=True, **kw)
        lin = api.Resize(**dict(kw, algo="linear")) if kw["algo"] != "linear" else None
        route, oc, ow, oh, _ = r.geometry(c, w, h)
        n_in = vc_get_linesize(w, c) * h
        n_out = vc_get_linesize(ow, oc) * oh
        n_stage = 0 if route == c else 2 * vc_get_linesize(w, route) * h
        nbytes = n_in + n_out + n_stage
        src = torch.randint(0, 256, (n_in,), dtype=torch.uint8, device="cuda")
        dst = torch.empty(n_out, dtype=torch.uint8, device="cuda")
        half = nbytes // 2
        cs, cd = torch.empty(half, dtype=torch.uint8, device="cuda"), torch.empty(half, dtype=torch.uint8, device="cuda")

        def run():
            r(src, c, w, h, dst=dst)

        def linear():
            lin(src, c, w, h, dst=dst)

        def copy():
            rt.cudaMemcpyAsync(vp(cd.data_ptr()), vp(cs.data_ptr()), half, 3, vp(torch.cuda.current_stream().cuda_stream))

        tr, tc, tl = [], [], []
        for _ in range(args.rounds):
            tr.append(timed(run, args.iters, args.warmup))
            tc.append(timed(copy, args.iters, args.warmup))
            if lin is not None:
                tl.append(timed(linear, args.iters, args.warmup))
        t, t0 = min(tr), min(tc)
        row = dict(workload=name, us=round(t, 1), bytes=nbytes, GBps=round(nbytes / t / 1e3, 1), copy_us=round(t0, 1),
                   copy_GBps=round(nbytes / t0 / 1e3, 1), of_copy=round(t0 / t, 2), linear_us=round(min(tl), 1) if tl else None)
        res.append(row)
        print(f"{name:34s} {t:9.1f} us  {nbytes / 1e6:7.1f} MB  {row['GBps']:7.1f} GB/s   copy {t0:8.1f} us  {row['copy_GBps']:7.1f} GB/s  "
              f"({row['of_copy']:.2f} of copy rate)" + (f"   linear {min(tl):8.1f} us" if tl else ""))
        r.close()
        if lin is not None:
            lin.close()
    if args.json:
        print(json.dumps(dict(card=card(), results=res)))


if __name__ == "__main__":
    main()
