"""A/B timing of the JPEG encoder's lean and general fused kernels at 8K (single stream, two streams, per-stage device times).  The kernel is
chosen by an environment variable read once per process (UGB200_JPEG_LEAN), so each variant runs in a child process.
usage: python tools/jpeg_ab.py            (parent: runs every variant)"""
import os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
# the instantiation without fall-back paths (default where the frame geometry allows) against the general kernel
VARIANTS = [("lean kernel (default)", {}), ("general kernel", {"UGB200_JPEG_LEAN": "0"}), ("lean kernel again", {})]


def child():
    import torch
    from ultragrid_b200 import api
    W, H = 7680, 4320
    dev = torch.device("cuda:0")
    xx = torch.arange(W, device=dev, dtype=torch.int32).view(1, W)
    yy = torch.arange(H, device=dev, dtype=torch.int32).view(H, 1)
    base = torch.stack([(xx * 255 // (W - 1)).expand(H, W), (yy * 255 // (H - 1)).expand(H, W), (xx + yy) % 256], dim=2)
    g = torch.Generator(device=dev)
    rgbs = []
    for k in range(6):
        g.manual_seed(k)
        rgbs.append((base + torch.randint(-6, 7, base.shape, dtype=torch.int32, device=dev, generator=g)).clamp_(0, 255).to(torch.uint8).reshape(-1))
    for codec, frames in ((2, [api.pixfmt_convert(12, 2, r, W, H) for r in rgbs]), (12, rgbs)):
        enc = api.JpegEncoder()
        for f in frames:
            for _ in range(2):
                enc.encode_device(f, W, H, codec, quality=90)
                n = enc.result_size()
        nf = len(frames)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        N = 600
        for i in range(8):
            enc.encode_device(frames[i % nf], W, H, codec, quality=90)
        torch.cuda.synchronize()
        e0.record()
        for i in range(N):
            enc.encode_device(frames[i % nf], W, H, codec, quality=90)
        e1.record()
        torch.cuda.synchronize()
        single = e0.elapsed_time(e1) / N * 1e3
        enc.result_size()
        enc.stage_timing(True)
        st = [0.0] * 4
        for i in range(nf):
            enc.encode_device(frames[i], W, H, codec, quality=90)
            st = [a + b / nf for a, b in zip(st, enc.stage_times())]
            enc.result_size()
        enc.stage_timing(False)
        enc.close()
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        encs = [api.JpegEncoder(stream=s) for s in streams]
        for e in encs:
            for f in frames:
                e.encode_device(f, W, H, codec, quality=90)
                e.result_size()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(N):
            encs[i & 1].encode_device(frames[i % nf], W, H, codec, quality=90)
        torch.cuda.synchronize()
        two = (time.perf_counter() - t0) / N * 1e6
        for e in encs:
            e.result_size()
            e.close()
        print("%-5s bytes %8d  single %.1f us  two-stream %.1f us  stages %s" % ("UYVY" if codec == 2 else "RGB", n, single, two, ["%.1f" % x for x in st]), flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "child":
        child()
    else:
        for name, env in VARIANTS:
            print("==", name, flush=True)
            subprocess.run([sys.executable, os.path.abspath(__file__), "child"], env={**os.environ, **env}, timeout=400)
