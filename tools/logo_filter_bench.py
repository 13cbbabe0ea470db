"""Timing of the logo filter and the R12L <-> Y416 pass-through filters (ugb200_cf_logo, ugb200_cf_r12l_to_y416_fake,
ugb200_pp_y416_to_r12l_fake, logo_kernels.cu) on device-resident 7680x4320 frames.

  r12l_to_y416_fake, y416_to_r12l_fake   both ranges; each against a device-to-device cudaMemcpyAsync of the same
                                         compulsory bytes (36 B of R12L and 64 B of Y416 per 8 pixels: 12.5 B/px,
                                         414.7 MB per frame) in the same run
  logo                                   UYVY and R12L frames, 256x128 and 1920x1080 logos at the default position;
                                         also the unmodified reference filter on the host (oracle/_ref/
                                         liblogo_filters_ref.so), when it was built, on a host copy of the frame

Each device case: --warmup launches, then CUDA events around --iters (>= 64) back-to-back launches on one stream; a
filter and its copy baseline alternate for --rounds rounds and the best round of each is kept.  The 256x128 logo
touches about 100 KB, so its time is launch overhead, not bandwidth.  Prints the card name and power limit read in
the same run.

    python tools/logo_filter_bench.py [--iters N] [--warmup N] [--rounds N] [--json]
"""
import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
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
    import numpy as np
    import torch
    import logo_filter_ref as R
    from ultragrid_b200 import api
    assert torch.cuda.is_available(), "logo_filter_bench.py needs a GPU"
    print("card:", card())
    rt = cudart()
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    rt.cudaMemcpyAsync.argtypes = [vp, vp, sz, ctypes.c_int, vp]
    w, h = 7680, 4320
    r12 = torch.randint(0, 256, (R.linesize(w, R.R12L) * h,), dtype=torch.uint8, device="cuda")
    y416 = torch.randint(0, 256, (8 * w * h,), dtype=torch.uint8, device="cuda")
    r12_out = torch.empty_like(r12)
    y416_out = torch.empty_like(y416)
    nbytes = r12.numel() + y416.numel()
    base_dst = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    base_src = torch.empty(nbytes, dtype=torch.uint8, device="cuda")

    def copy():
        st = vp(torch.cuda.current_stream().cuda_stream)
        rt.cudaMemcpyAsync(vp(base_dst.data_ptr()), vp(base_src.data_ptr()), nbytes // 2, 3, st)

    rows = []
    for full in (False, True):
        rng = "full" if full else "limited"
        for name, fn in ((f"r12l_to_y416_fake {rng}", lambda f=full: api.r12l_to_y416_fake(r12, w, h, f, dst=y416_out)),
                         (f"y416_to_r12l_fake {rng}", lambda f=full: api.y416_to_r12l_fake(y416, w, h, f, dst=r12_out))):
            tf, tb = float("inf"), float("inf")
            for _ in range(args.rounds):
                tf = min(tf, timed(fn, args.iters, args.warmup))
                tb = min(tb, timed(copy, args.iters, args.warmup))
            # the copy moves nbytes / 2 bytes once: it reads and writes nbytes in all, as the filter does
            rows.append({"case": name, "us": round(tf, 2), "copy_us": round(tb, 2), "compulsory_MB": round(nbytes / 1e6, 1),
                         "TBps": round(nbytes / (tf * 1e-6) / 1e12, 3), "copy_TBps": round(nbytes / (tb * 1e-6) / 1e12, 3)})
    ref = None
    try:
        import test_logo_filters as T
        ref = T.ref_lib()
    except OSError:
        pass
    for c in (R.UYVY, R.R12L):
        f = torch.randint(0, 256, (R.linesize(w, c) * h,), dtype=torch.uint8, device="cuda")
        for lw, lh in ((256, 128), (1920, 1080)):
            rgba = np.random.default_rng(lw).integers(0, 256, (lh, lw, 4), dtype=np.uint8)
            lg = api.logo(rgba.reshape(-1), lw, lh)
            t = min(timed(lambda: lg(c, f, w, h), args.iters, args.warmup) for _ in range(args.rounds))
            row = {"case": f"logo {R.NAMES[c]} {lw}x{lh}", "us": round(t, 2)}
            if ref is not None:
                # a logo width whose segment the reference allocates too short would make it write past its malloc:
                # time it at the next width it handles, padded with transparent columns (R12L: 256 -> 287, 1920 -> 1943)
                pw = R.logo_padded_width(c, lw)
                padded = np.zeros((lh, pw, 4), np.uint8)
                padded[:, :lw] = rgba
                host = np.concatenate([f.cpu().numpy(), np.zeros(4096, np.uint8)])
                st = ref.ref_logo_make(padded.ctypes.data, pw, lh, -1, -1)
                best = float("inf")
                for _ in range(5):
                    t0 = time.perf_counter()
                    ref.ref_logo_filter(st, c, w, h, host.ctypes.data)
                    best = min(best, time.perf_counter() - t0)
                ref.ref_logo_done(st)
                row["reference_host_us"] = round(best * 1e6, 1)
                row["reference_logo_width"] = pw
            lg.close()
            rows.append(row)
    for r in rows:
        if "copy_us" in r:
            print(f"{r['case']:30s} {r['us']:8.1f} us  {r['TBps']:5.2f} TB/s   copy {r['copy_us']:8.1f} us  {r['copy_TBps']:5.2f} TB/s"
                  f"   ratio {r['us'] / r['copy_us']:5.2f}")
        else:
            print(f"{r['case']:30s} {r['us']:8.1f} us" + (f"   reference on the host {r['reference_host_us']:10.1f} us" if "reference_host_us" in r else ""))
        if args.json:
            print(json.dumps(r))


if __name__ == "__main__":
    main()
