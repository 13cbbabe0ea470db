"""exercises every C-ABI entry point once or twice at small, odd sizes - meant to run under `compute-sanitizer --tool memcheck`"""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch
import util
import planar_cases as pc
from test_oracle_pinning import PAIRS
from ultragrid_b200 import api, _lib, vc_get_linesize
lib = _lib.load()
n = 0
ONLY = sys.argv[1] if len(sys.argv) > 1 else ""
for inc, outc in ([] if ONLY in ("jpeg", "staged") else PAIRS):  # line converters: tight buffers, ragged widths
    for w, h in ((50, 3), (17, 2), (256, 2)):
        ls_i, ls_o = vc_get_linesize(w, inc), vc_get_linesize(w, outc)
        src = torch.randint(0, 256, (ls_i * h + 64,), dtype=torch.uint8, device="cuda")  # MAX_PADDING of over-read slack, video_codec.h:61
        dst = torch.zeros(ls_o * h + 64, dtype=torch.uint8, device="cuda")
        api.pixfmt_convert(inc, outc, src, w, h, dst=dst)
        n += 1
for name, depth in ([] if ONLY in ("jpeg", "staged") else pc.all_cases()):  # planar converters
    for w, h in ((50, 5), (17, 3), (64, 4)):
        if name == "yuv420_to_i420" and (w % 2 or h % 2):
            continue
        for mode in (0, 2):
            c = pc.Case(name, w, h, seed=3, mode=mode, depth=depth)
            c.run_gpu(lib, torch, 0)
            n += 1
for w, h in ([] if ONLY == "staged" else ((8, 4), (260, 36))):  # DXT encode / decode
    uy = torch.randint(0, 256, (w * h * 2,), dtype=torch.uint8, device="cuda")
    rgb = torch.randint(0, 256, (w * h * 3,), dtype=torch.uint8, device="cuda")
    for t in (1, 6):
        blocks = api.uyvy_to_dxt(uy, w, h, dxt_type=t)
        api.dxt_to_rgb(blocks, w, h, t)
        api.compat_to_dxt("cuda_rgb_to_dxt1" if t == 1 else "cuda_rgb_to_dxt6", rgb, w, -h)
        n += 3
enc, dec = api.JpegEncoder(), api.JpegDecoder()
for codec, w, h, q, ri in ([] if ONLY == "staged" else ((2, 100, 52, 90, 0), (2, 98, 50, 100, 1), (12, 77, 33, 85, 8), (12, 64, 64, 100, 5))):  # JPEG encode (fused, serial route, split) / decode
    bpp = 2 if codec == 2 else 3
    src = torch.randint(0, 256, (((w + 1) // 2 * 2) * bpp * h,), dtype=torch.uint8, device="cuda")
    for _ in range(2):
        enc.encode_device(src, w, h, codec, quality=q, restart_interval=ri)
        try:
            s = enc.result()
        except RuntimeError:
            s = None
    if s:
        for out_c in (2, 12, 1, 29):
            dec.decode(s, out_c)
        n += 6
# JPEG planar layouts (ugb200_jpeg_encode_device_ex) at ragged sizes, one per new row of the supported matrix: I420 read in place,
# UYVY -> 4:2:0, RGB -> Y709 / Y601 / Y601full at 4:4:4 / 4:2:2 / 4:2:0, per-component and interleaved; the 4:2:0 streams decode to I420
for codec, sub, cs, il in ([] if ONLY == "staged" else ((29, 0, 0, 1), (2, 420, 3, 1), (12, 0, 3, 0), (12, 422, 1, 1), (12, 420, 2, 0), (12, 420, 3, 1))):
    for w, h, ri in ((17, 9, 3), (130, 37, 0)):
        nbytes = w * h + 2 * ((w + 1) // 2) * ((h + 1) // 2) if codec == 29 else ((w + 1) // 2 * 4 if codec == 2 else w * 3) * h
        src = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda")
        enc.encode_device(src, w, h, codec, quality=90, restart_interval=ri, pitch=(w + 1) // 2 * 4 if codec == 2 else 0, interleaved=bool(il),
                          subsampling=sub, color_space=cs)
        s = enc.result()
        if sub == 420 or codec == 29:
            dec.decode(s, 29)
        n += 2
# round 2, state i: the staged launch forms of the line converters (16-byte aligned pitches, tight buffers), every form of every converter
for inc, outc in ([] if ONLY == "jpeg" else PAIRS):
    for w, h in ((64, 2), (192, 3), (2048 + 64, 2)):
        ls_i, ls_o = vc_get_linesize(w, inc), vc_get_linesize(w, outc)
        sp, dp = (ls_i + 15) // 16 * 16, (ls_o + 15) // 16 * 16
        src = torch.randint(0, 256, (sp * h + 64,), dtype=torch.uint8, device="cuda")
        dst = torch.zeros(dp * h, dtype=torch.uint8, device="cuda")
        for mode in (1, 2, 3):
            api.pixfmt_staged_mode(mode)
            api.pixfmt_convert(inc, outc, src, w, h, dst=dst, src_pitch=sp, dst_pitch=dp)
            n += 1
api.pixfmt_staged_mode(-1)
# src/cuda_wrapper/kernels.cu entry points (tight buffers, widths with and without a partial last group)
import ctypes
VP, SZ, I = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
post = getattr(lib, "_Z24postprocess_rg48_to_r12lPvS_miiP25cmpto_j2k_dec_comp_formatiS_mS_mS_mS_")
pre = getattr(lib, "_Z23preprocess_r12l_to_rg48PvS_miiP25cmpto_j2k_enc_comp_formatiS_mS_mS_")
post.argtypes, post.restype = [VP, VP, SZ, I, I, VP, I, VP, SZ, VP, SZ, VP, SZ, VP], I
pre.argtypes, pre.restype = [VP, VP, SZ, I, I, VP, I, VP, SZ, VP, SZ, VP], I
for w, h in ((64, 3), (30, 2), (1921, 2)):
    nb = (w + 7) // 8
    rg48 = torch.randint(0, 256, (w * 6 * h,), dtype=torch.uint8, device="cuda")
    r12l = torch.zeros(nb * 36 * h, dtype=torch.uint8, device="cuda")
    assert post(None, None, 0, w, h, None, 3, rg48.data_ptr(), rg48.numel(), None, 0, r12l.data_ptr(), r12l.numel(), None) == 0
    back = torch.zeros(w * 6 * h, dtype=torch.uint8, device="cuda")
    assert pre(None, None, 0, w, h, None, 3, r12l.data_ptr(), r12l.numel(), back.data_ptr(), back.numel(), None) == 0
    n += 2
# JPEG decoder with the marker scan forced onto the device: one interleaved scan (UYVY) and one scan per component (RGB), intact and truncated
os.environ["UGB200_JPEG_MARKER_SCAN"] = "device"
dec2 = api.JpegDecoder()
for codec, w, h in ([] if ONLY == "staged" else ((2, 320, 200), (12, 200, 120), (12, 1920, 1080))):
    bpp = 2 if codec == 2 else 3
    src = torch.randint(96, 160, (w * bpp * h,), dtype=torch.uint8, device="cuda")
    enc.encode_device(src, w, h, codec, quality=90)
    s = enc.result()
    for data in (s, s[:len(s) * 2 // 3]):
        for out_c in (codec, 1):
            try:
                dec2.decode(data, out_c)
            except RuntimeError:
                pass
            n += 1
torch.cuda.synchronize()
print("exercised", n, "calls")
