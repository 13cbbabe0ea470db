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
# JPEG with alpha: RGBA 4444 on tight buffers, four scans (fused kernel; restart interval 5: split path) and one interleaved scan (split path);
# the four-component streams decode to RGBA, RGB and UYVY
for w, h, ri, il in ([] if ONLY == "staged" else ((17, 9, 0, 0), (130, 37, 5, 0), (130, 37, 0, 1))):
    src = torch.randint(0, 256, (w * h * 4,), dtype=torch.uint8, device="cuda")
    enc.encode_device(src, w, h, 1, quality=90, restart_interval=ri, interleaved=bool(il), subsampling=4444)
    s = enc.result()
    for out_c in (1, 12, 2):
        dec.decode(s, out_c)
    n += 4
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
# JPEG decoder, self-synchronising Huffman route: a no-DRI 4:2:0 stream (default subsequences and 8-byte ones), truncated, and the adversarial stream
# of tests/test_jpeg_decode_sync.py (many rounds)
if ONLY != "staged":
    import io
    from PIL import Image
    from test_jpeg import natural_rgb
    from test_jpeg_decode_sync import adversarial_stream
    b = io.BytesIO()
    Image.fromarray(natural_rgb(333, 211, 4)).save(b, "JPEG", quality=90, subsampling=2)
    s420 = b.getvalue()
    os.environ.pop("UGB200_JPEG_MARKER_SCAN", None)
    for sync in ("on", "on:8"):
        os.environ["UGB200_JPEG_SYNC"] = sync
        dec3 = api.JpegDecoder()
        for data in (s420, s420[:len(s420) // 2], adversarial_stream()):
            for out_c in (2, 29):
                try:
                    dec3.decode(data, out_c)
                except RuntimeError:
                    pass
                n += 1
        dec3.close()
    os.environ.pop("UGB200_JPEG_SYNC", None)
# JPEG decoder, fused IDCT + chroma replication + packing kernel (4:2:2 and 4:2:0) and the 4:4:4 colour-space kernel: odd and even sizes, tight
# device buffers and a pitch wider than the row, UYVY / RGB / RGBA with shifts (8, 16, 0), every colour space
if ONLY != "staged":
    dec4 = api.JpegDecoder()
    for ss, w, h in ((1, 333, 211), (2, 333, 211), (2, 64, 32), (0, 37, 19)):
        b = io.BytesIO()
        Image.fromarray(natural_rgb(w, h, 6)).save(b, "JPEG", quality=90, subsampling=ss)
        s = b.getvalue()
        for out_c, bpp in ((2, 2), (12, 3), (1, 4)):
            ls = vc_get_linesize(w, out_c)
            for pitch in (ls, ls + 40):
                for cs in ((None,) if out_c == 2 else (None, "native", "Y709", "Y601", "Y601full", "auto")):
                    out = torch.empty(pitch * h, dtype=torch.uint8, device="cuda")
                    try:
                        dec4.decode(s, out_c, shifts=(8, 16, 0) if out_c == 1 else (0, 8, 16), device=True, pitch=pitch, out=out, color_space=cs)
                    except RuntimeError:  # 4:4:4 YCbCr to RGBA without a colour space: no VUYA -> RGBA line converter (-4)
                        assert ss == 0 and out_c == 1 and cs in (None, "native")
                    n += 1
    dec4.close()
# JPEG decode to a YCbCr colour space (ugb200_jpeg_decode_to) and grayscale streams: the matrix phase of the fused kernel to UYVY for 4:2:2 / 4:2:0 at
# odd and even sizes, its planar (I420) epilogue into tight buffers, the 4:4:4 plane kernel, and the two-warp grayscale form (odd block counts) to
# UYVY, I420, RGB and RGBA, tight and pitched device destinations
if ONLY != "staged":
    dec5 = api.JpegDecoder()
    streams = []
    for ss, w, h in ((1, 333, 211), (2, 333, 211), (1, 64, 32), (2, 64, 32), (0, 37, 19)):
        b = io.BytesIO()
        Image.fromarray(natural_rgb(w, h, 6)).save(b, "JPEG", quality=90, subsampling=ss)
        streams.append((b.getvalue(), w, h, ss == 0))
    for w, h in ((333, 211), (72, 40), (9, 1), (1, 1)):
        b = io.BytesIO()
        Image.fromarray(natural_rgb(w, h, 6)[:, :, 1].copy(), "L").save(b, "JPEG", quality=90)
        streams.append((b.getvalue(), w, h, False))
    for s, w, h, is444 in streams:
        for out_c in (2, 29, 12, 1) + ((4,) if is444 else ()):  # UYVY, I420, RGB, RGBA, VUYA
            ls = vc_get_linesize(w, out_c)
            size = w * h + 2 * ((w + 1) // 2) * ((h + 1) // 2) if out_c == 29 else None
            for pitch in ((ls,) if out_c == 29 else (ls, ls + 40)):
                for cs_in, cs_out in (("native", "native"), ("auto", "Y709"), ("Y709", "Y601full")):
                    out = torch.empty(size or pitch * h, dtype=torch.uint8, device="cuda")
                    try:
                        dec5.decode_to(s, out_c, cs_in, cs_out, device=True, pitch=pitch, out=out)
                    except RuntimeError:  # as above
                        assert is444 and out_c == 1 and cs_in == "native"
                    n += 1
    dec5.close()
# JPEG decode with interpolated chroma (ugb200_jpeg_decoder_set_upsampling FANCY): the halo IDCT and the filter phase of the fused kernel, 4:2:2 and
# 4:2:0 at odd and even sizes down to 1 x 1 and widths across CTA boundaries (512 pixels), to RGB and RGBA, tight and pitched device destinations
if ONLY != "staged":
    dec6 = api.JpegDecoder()
    dec6.set_upsampling("fancy")
    for ss in (1, 2):
        for w, h in ((1, 1), (2, 2), (3, 3), (5, 17), (64, 32), (333, 211), (513, 9), (1041, 40), (1553, 17)):
            b = io.BytesIO()
            Image.fromarray(natural_rgb(w, h, 6)).save(b, "JPEG", quality=90, subsampling=ss)
            s = b.getvalue()
            for out_c in (12, 1):  # RGB, RGBA
                ls = vc_get_linesize(w, out_c)
                for pitch in (ls, ls + 40):
                    for cs in ("Y709", "Y601", "Y601full", "auto"):
                        out = torch.empty(pitch * h, dtype=torch.uint8, device="cuda")
                        dec6.decode(s, out_c, shifts=(8, 16, 0) if out_c == 1 else (0, 8, 16), device=True, pitch=pitch, out=out, color_space=cs)
                        n += 1
    dec6.close()
# LDGM FEC: encode from host (packets of 4-, 8- and 16-byte words) and from a device frame at offsets 4 and 1 into a tight device buffer;
# decode with losses peeling can repair (several levels) and with losses it cannot
import ldgm_cases as lc
for k, m, c in ([] if ONLY in ("jpeg", "staged") else ((64, 64, 2), (512, 384, 5))):
    coder = api.LdgmCoder(lc.matrix(k, m, c, 1), k, m)
    for size in (1, 4 * k * 3 - 12, 4 * k * 4 - 8, 20_011):
        frame = util.rng_bytes(size, size)
        enc_h = coder.encode(frame, b"hdr")
        for off in (4, 1):
            dev = torch.zeros(size + 8, dtype=torch.uint8, device="cuda")
            dev[off:off + size] = torch.from_numpy(frame).cuda()
            tight = torch.empty(enc_h.size, dtype=torch.uint8, device="cuda")
            coder.encode(dev[off:off + size], b"hdr", out=tight)
        n += 3
        ps = lc.layout(k, 3 + size)[1]
        rng = np.random.default_rng(size)
        for loss in (0.1, 0.3, 0.7):
            buf = enc_h.copy()
            coder.decode(buf, lc.packets_received(k + m, ps, rng.random(k + m) >= loss))
            n += 1
    coder.close()
# libavcodec bridge: every to_lavc pair at odd sizes (v210 -> YUV420P10LE at odd height included) into tight, padded and odd-padded planes and into
# planes 2 bytes into their buffers; every from_lavc pair the library accepts at odd sizes, with a tight and a wider pitch
if ONLY not in ("jpeg", "staged"):
    import test_lavc_exact as tle
    L2, _ = tle.lib_and_torch()
    for inc, fmt in tle.to_lavc_pairs():
        for w, h in ((47, 5), (49, 3), (1, 1)):
            src = tle.make_source(inc, w, h, 1)
            for _, lss, off in tle.plane_modes(fmt, w, h):
                assert tle.gpu_to_lavc(L2, torch, inc, fmt, src, w, h, lss, off)[0] == 0
                n += 1
    for fmt, outc in tle.from_lavc_pairs():
        for w, h in ((47, 5), (15, 3)):
            pl = tle.av_planes_in(fmt, w, h, 2, pad=3)
            planes = [torch.from_numpy(a.reshape(-1).copy()).cuda() for a, _ in pl]
            for pitch in (vc_get_linesize(w, outc), vc_get_linesize(w, outc) + 40):
                dst = torch.zeros(pitch * h, dtype=torch.uint8, device="cuda")
                api.from_lavc(fmt, outc, planes, [ls for _, ls in pl], w, h, dst, pitch)
                n += 1
# interlaced video: vc_deinterlace_ex on tight buffers (dst ends at row lines-1's src_linesize), in place and out of place, lines 1-6, odd
# line sizes, R12L's partial group and 16-bit rows that are not whole 16-byte chunks; vc_deinterlace at odd line sizes and addresses;
# il_* in place and out of place
if ONLY not in ("jpeg", "staged"):
    for codec, ls in ((2, 3838), (2, 47), (7, 1004), (5, 68), (6, 36 * 5 + 8), (6, 8640), (27, 11508), (30, 20), (31, 14), (12, 5757)):
        for lines in range(1, 7):
            src = torch.randint(0, 256, (ls * lines,), dtype=torch.uint8, device="cuda")
            dst = torch.zeros(ls * lines, dtype=torch.uint8, device="cuda")
            api.deinterlace_ex(codec, src, ls, lines, dst=dst)
            api.deinterlace_ex(codec, src, ls, lines, dst=src)
            n += 2
    for ls in (16, 17, 31, 52, 3841):
        for lines in range(1, 8):
            for off in (0, 1):
                buf = torch.randint(0, 256, (ls * lines + off,), dtype=torch.uint8, device="cuda")
                api.deinterlace(buf[off:], ls, lines)
                n += 1
    for ls, h in ((1, 1), (3, 7), (3841, 6)):
        src = torch.randint(0, 256, (ls * h,), dtype=torch.uint8, device="cuda")
        api.il_upper_to_merged(src, ls, h, dst=torch.empty_like(src))
        api.il_merged_to_upper(src, ls, h)
        n += 2
    # field-rate postprocessors on tight buffers (sources L * h, dst ends at row h-1's L bytes): R10k and R12L at line sizes
    # off 16 and 36, an odd 8-bit line size, odd h and h = 2, both calls, `:d` fused (pitch L) and composed (pitch > L)
    for codec, ls in ((5, 68), (5, 7680 * 4), (6, 36 * 5 + 8), (6, 36 * 3 + 4), (2, 47), (7, 1004 // 4 * 4), (27, 11508)):
        for h in (2, 3, 5, 7):
            for pitch in (ls, ls + 12):
                prev = torch.randint(0, 256, (ls * h,), dtype=torch.uint8, device="cuda")
                cur = torch.randint(0, 256, (ls * h,), dtype=torch.uint8, device="cuda")
                dst = torch.zeros(pitch * (h - 1) + ls, dtype=torch.uint8, device="cuda")
                for call in (0, 1):
                    api.deinterlace_bob(cur, ls, h, call, dst=dst, pitch=pitch)
                    api.deinterlace_linear(codec, cur, ls, h, call, dst=dst, pitch=pitch)
                    api.double_framerate(codec, prev, cur, ls, h, call, dst=dst, pitch=pitch)
                    if pitch == ls or pitch % 4 == 0:
                        api.double_framerate(codec, prev, cur, ls, h, call, True, dst=dst, pitch=pitch)
                        n += 1
                    n += 3
                api.interlace(cur, prev, ls, h, dst=dst, pitch=pitch)
                n += 1
    # colour capture filters on tight buffers (input and output frames exactly vf_alloc_desc's length) at odd sizes:
    # matrix UYVY at odd widths (the output stops at 3 * w * h), v210 off multiples of 48, RG48 / Y416 at 2-byte offsets
    cf_g = api.gamma(2.2)
    for w, h in ((1, 1), (3, 5), (47, 3), (49, 7), (131, 2), (1919, 3)):
        m = api.Y601_TO_Y709
        for c in (2, 12, 27):
            src = torch.randint(0, 256, (vc_get_linesize(w, c) * h,), dtype=torch.uint8, device="cuda")
            for b in (True, False):
                api.matrix(c, src, w, h, m, b)
                n += 1
        for c in (2, 7, 31):
            src = torch.randint(0, 256, (vc_get_linesize(w, c) * h,), dtype=torch.uint8, device="cuda")
            api.matrix2(c, src, w, h, m)
            n += 1
        api.grayscale(torch.randint(0, 256, (vc_get_linesize(w, 2) * h,), dtype=torch.uint8, device="cuda"), w, h)
        n += 1
        for c in (12, 27):
            raw = torch.randint(0, 256, (vc_get_linesize(w, c) * h + 2,), dtype=torch.uint8, device="cuda")
            for d in (0, 8, 16):
                cf_g(c, raw[2:], w, h, d)
                n += 1
    cf_g.close()
torch.cuda.synchronize()
print("exercised", n, "calls")
