"""Times the LDGM FEC coder (include/ugb200_ldgm.h) on frames of the sizes it codes in practice, at the default (k, m, c) = (512, 384, 5)
of src/rtp/ldgm.cpp and at the extremes of its range:
  jpeg1080   300 KB (a 1080p JPEG)         (512, 384, 5), (64, 64, 2), (8191, 8191, 63)
  jpeg4k     1.2 MB (a 4K JPEG)            (512, 384, 5), (8191, 8191, 63)
  uyvy8k     66 MB (an 8K UYVY frame)      (8191, 8191, 5), (8191, 8191, 63) - at k = 512 its packets would pass 65535 bytes
For each it reports, as medians over alternating rounds:
  enc_device_us   ugb200_ldgm_encode_device from a device frame (copy into the buffer, header and padding, parity), CUDA events
  enc_host_us     ugb200_ldgm_encode_frame from host memory into a pinned buffer, wall clock around the synchronous call
  dec_host_us     ugb200_ldgm_decode of the host buffer with 10 % of the packets lost at random, wall clock
  ref_cpu_enc_us / ref_cpu_dec_us   the reference's LDGM_session_cpu on the same inputs (oracle/_ref/libldgm_ref.so), when built
and, from a torch.profiler run of its own, the device time of each kernel per call.  The card's name, power limit and clocks are read in the
same run.  Prints one JSON object; with --out DIR also writes DIR/ldgm_bench.json."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CASES = [("jpeg1080", 300_000, (512, 384, 5)), ("jpeg1080", 300_000, (64, 64, 2)), ("jpeg1080", 300_000, (8191, 8191, 63)),
         ("jpeg4k", 1_200_000, (512, 384, 5)), ("jpeg4k", 1_200_000, (8191, 8191, 63)),
         ("uyvy8k", 7680 * 4320 * 2, (8191, 8191, 5)), ("uyvy8k", 7680 * 4320 * 2, (8191, 8191, 63))]
HDR = b"\0" * 24  # the size of the video header ldgm.cpp puts in front of a frame


def wall(fn, n):
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    return (time.perf_counter() - t0) * 1e6 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--window", type=int, default=20, help="device encodes per timed window")
    ap.add_argument("--ref-rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import ldgm_cases as lc
    import util
    from ultragrid_b200 import api
    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    ref = lc.ref_lib()
    tmpdir = tempfile.TemporaryDirectory()
    tmp = tmpdir.name
    results = []
    for name, size, (k, m, c) in CASES:
        pcm = lc.matrix(k, m, c, 1)
        coder = api.LdgmCoder(pcm, k, m, stream=stream)
        frame = util.rng_bytes(size, size)
        dev = torch.from_numpy(frame).cuda()
        total, ps = coder.buffer_size(len(HDR) + size)
        out_dev = torch.empty(total, dtype=torch.uint8, device="cuda")
        out_pin = torch.empty(total, dtype=torch.uint8, pin_memory=True).numpy()
        enc = coder.encode(frame, HDR, out=out_pin).copy()
        rng = np.random.default_rng(1)
        ranges = lc.packets_received(k + m, ps, rng.random(k + m) >= 0.10)
        lost_buf = np.zeros_like(enc)  # lost packets arrive as zeros
        for o, n in ranges:
            lost_buf[o:o + n] = enc[o:o + n]
        pin_dec = torch.empty(total, dtype=torch.uint8, pin_memory=True).numpy()

        def enc_dev(n):
            for _ in range(n):
                coder.encode(dev, HDR, out=out_dev)

        def dec_host():
            pin_dec[:] = lost_buf
            return coder.decode(pin_dec, ranges)

        torch.cuda.synchronize()
        enc_dev(3), dec_host(), dec_host()
        recovered = dec_host() == len(HDR) + size
        t = {"enc_device_us": [], "enc_host_us": [], "dec_host_us": [], "copy_only_us": []}
        for r in range(args.rounds):
            for key in (list(t) if r % 2 == 0 else list(reversed(list(t)))):
                if key == "enc_device_us":
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    a.record(stream)
                    enc_dev(args.window)
                    b.record(stream)
                    b.synchronize()
                    t[key].append(a.elapsed_time(b) * 1000.0 / args.window)
                elif key == "enc_host_us":
                    t[key].append(wall(lambda: coder.encode(frame, HDR, out=out_pin), 3))
                elif key == "dec_host_us":
                    t[key].append(wall(dec_host, 3))
                else:  # the buffer refill dec_host does before each decode, to subtract
                    t[key].append(wall(lambda: pin_dec.__setitem__(slice(None), lost_buf), 3))
        res = {"case": name, "frame_bytes": size, "k": k, "m": m, "c": c, "w_f": int(pcm.shape[1]), "packet_size": ps,
               "buffer_bytes": total, "decode_recovered": recovered}
        for key, v in t.items():
            res[key] = round(statistics.median(v), 1)
            res[key.replace("_us", "_spread_us")] = [round(min(v), 1), round(max(v), 1)]
        res["dec_host_us"] = round(res["dec_host_us"] - res["copy_only_us"], 1)
        if ref is not None:
            path = os.path.join(tmp, f"{k}-{m}-{c}.bin")
            lc.write_matrix_file(path, pcm, k, m)
            s = lc.RefSession(ref, path, k, m, c)
            want = s.encode(HDR, frame)
            assert np.array_equal(want, enc), "GPU and reference encodes differ"
            res["ref_cpu_enc_us"] = round(min(wall(lambda: s.encode(HDR, frame), 1) for _ in range(args.ref_rounds)), 1)
            buf = lost_buf.copy()

            def ref_dec():
                buf[:] = lost_buf
                return s.decode(buf, ranges)
            res["ref_cpu_dec_us"] = round(min(wall(ref_dec, 1) for _ in range(args.ref_rounds)) - res["copy_only_us"], 1)
            s.close()
        else:
            res["ref_cpu_enc_us"] = res["ref_cpu_dec_us"] = "not built"
        # device time per kernel, in a profiled run of its own
        from torch.profiler import ProfilerActivity, profile
        for key, fn in (("enc_device_kernels_us", lambda: enc_dev(1)), ("dec_kernels_us", dec_host)):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    fn()
                torch.cuda.synchronize()
            acc = {}
            for ev in prof.key_averages():
                if ev.device_time_total > 0:
                    kname = ev.key.replace("(anonymous namespace)::", "").split("<")[0].split("(")[0].replace("void ", "")
                    acc[kname] = acc.get(kname, 0.0) + ev.device_time_total / 5.0
            res[key] = {kk: round(v, 1) for kk, v in sorted(acc.items(), key=lambda kv: -kv[1])}
        coder.close()
        results.append(res)
        print(json.dumps(res), file=sys.stderr)
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        gpu = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        gpu = "unknown"
    line = json.dumps({"gpu": gpu, "gpu_fields": q, "results": results})
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ldgm_bench.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
