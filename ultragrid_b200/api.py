"""Thin torch-tensor front end over the C ABI (tests and bench only; plumbing, not the product).

All tensors are ``torch.uint8`` CUDA tensors; results are bit-identical to the reference functions named in
``include/*.h``.  Every call requires the CUDA library — there is no CPU path.
"""
import ctypes

import torch

from . import _lib
from .codec import Codec, vc_get_linesize

_L = _lib.load()


def _stream(stream=None):
    s = stream if stream is not None else torch.cuda.current_stream()
    return ctypes.c_void_p(s.cuda_stream)


def _check(rc, what):
    if rc != 0:
        raise RuntimeError(f"{what} failed with code {rc}")


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def dxt_out_bytes(width, height, dxt_type):
    h = abs(height)
    return width * h // 2 if dxt_type == 1 else width * h


def compat_to_dxt(name, src, width, height, out=None, stream=None):
    """Synchronous reference-ABI entry points: name in cuda_{rgb,yuv}_to_dxt{1,6}."""
    dxt_type = 1 if name.endswith("dxt1") else 6
    if out is None:
        out = torch.empty(dxt_out_bytes(width, height, dxt_type), dtype=torch.uint8, device=src.device)
    _check(getattr(_L, name)(_ptr(src), _ptr(out), width, height, _stream(stream)), name)
    return out


def uyvy_to_dxt(src, width, height, dxt_type=1, pitch=0, out=None, stream=None):
    """Fused UYVY -> DXT1 / DXT5-YCoCg, asynchronous on the stream."""
    if out is None:
        out = torch.empty(dxt_out_bytes(width, height, dxt_type), dtype=torch.uint8, device=src.device)
    fn = _L.ugb200_uyvy_to_dxt1_async if dxt_type == 1 else _L.ugb200_uyvy_to_dxt6_async
    _check(fn(_ptr(src), _ptr(out), width, height, pitch, _stream(stream)), "ugb200_uyvy_to_dxt")
    return out


def yuv422_to_yuv444(src, pix_count, out=None, stream=None):
    if out is None:
        out = torch.empty(pix_count * 3, dtype=torch.uint8, device=src.device)
    _check(_L.cuda_yuv422_to_yuv444(_ptr(src), _ptr(out), pix_count, _stream(stream)), "cuda_yuv422_to_yuv444")
    return out


def pixfmt_supported(in_codec, out_codec):
    return bool(_L.ugb200_pixfmt_supported(int(in_codec), int(out_codec)))


def pixfmt_convert(in_codec, out_codec, src, width, height, dst=None, dst_len=None, src_pitch=None, dst_pitch=None,
                   shifts=(0, 8, 16), stream=None):
    """Device form of the reference row loop (tools/convert.cpp:148-152)."""
    src_pitch = vc_get_linesize(width, in_codec) if src_pitch is None else src_pitch
    dst_pitch = vc_get_linesize(width, out_codec) if dst_pitch is None else dst_pitch
    dst_len = vc_get_linesize(width, out_codec) if dst_len is None else dst_len
    if dst is None:
        dst = torch.zeros(dst_pitch * height, dtype=torch.uint8, device=src.device)
    rc = _L.ugb200_pixfmt_convert(int(in_codec), int(out_codec), _ptr(dst), dst_pitch, _ptr(src), src_pitch, dst_len, height,
                                  src.numel(), shifts[0], shifts[1], shifts[2], _stream(stream))
    _check(rc, f"ugb200_pixfmt_convert({Codec(in_codec).name}->{Codec(out_codec).name})")
    return dst


def pixfmt_staged_mode(mode):
    """-1 default (per converter), 0 never, 1 always staged through shared memory; returns the previous mode"""
    return _L.ugb200_pixfmt_staged_mode(int(mode))


LINE_FUNCS = {"ABGRtoRGB": 1, "BGRAtoRGB": 2, "ToRGBA_inplace": 3, "UYVYtoGrayscale": 4}


def vc_copyline(func, src, dst, dst_len, height, src_pitch, dst_pitch, shifts=(0, 8, 16), stream=None):
    """the exported line converters outside decoders[] (pixfmt_conv.h:93-101); func = a key of LINE_FUNCS; dst may be src for ToRGBA_inplace"""
    rc = _L.ugb200_vc_copyline(LINE_FUNCS[func], _ptr(dst), dst_pitch, _ptr(src), src_pitch, dst_len, height, src.numel(), shifts[0], shifts[1], shifts[2],
                               _stream(stream))
    _check(rc, f"ugb200_vc_copyline({func})")
    return dst


class ToPlanarData(ctypes.Structure):
    _fields_ = [("width", ctypes.c_int), ("height", ctypes.c_int), ("out_data", ctypes.c_void_p * 4),
                ("out_linesize", ctypes.c_uint * 4), ("in_data", ctypes.c_void_p)]


def v210_to_p010le(src, width, height, out_y=None, out_c=None, ls_y=None, ls_c=None, stream=None):
    ls_y = width * 2 if ls_y is None else ls_y
    ls_c = width * 2 if ls_c is None else ls_c
    if out_y is None:
        out_y = torch.zeros(ls_y * height, dtype=torch.uint8, device=src.device)
    if out_c is None:
        out_c = torch.zeros(ls_c * ((height + 1) // 2), dtype=torch.uint8, device=src.device)
    d = ToPlanarData()
    d.width, d.height = width, height
    d.out_data[0], d.out_data[1] = out_y.data_ptr(), out_c.data_ptr()
    d.out_linesize[0], d.out_linesize[1] = ls_y, ls_c
    d.in_data = src.data_ptr()
    _check(_L.ugb200_v210_to_p010le(ctypes.byref(d), 0, _stream(stream)), "ugb200_v210_to_p010le")
    return out_y, out_c


def dxt_to_rgb(src, width, height, dxt_type=1, bgr=False, out=None, out_pitch=0, stream=None):
    """ugb200_dxt1_to_rgb / ugb200_dxt5ycocg_to_rgb: device blocks -> packed RGB (or BGR) on the device"""
    if out is None:
        out = torch.zeros((out_pitch or width * 3) * height, dtype=torch.uint8, device=src.device)
    fn = _L.ugb200_dxt1_to_rgb if dxt_type == 1 else _L.ugb200_dxt5ycocg_to_rgb
    _check(fn(_ptr(src), _ptr(out), width, height, out_pitch, int(bgr), _stream(stream)), "ugb200_dxt_to_rgb")
    return out


class FromPlanarData(ctypes.Structure):
    """struct from_planar_data (src/from_planar.h:58-70) with device pointers"""
    _fields_ = [("width", ctypes.c_int), ("height", ctypes.c_int), ("out_data", ctypes.c_void_p), ("out_pitch", ctypes.c_uint),
                ("in_data", ctypes.c_void_p * 4), ("in_linesize", ctypes.c_uint * 4), ("in_depth", ctypes.c_int),
                ("log2_chroma_h", ctypes.c_int), ("rgb_shift", ctypes.c_int * 3)]


def to_planar(name, src, width, height, planes, linesizes, stream=None):
    """decode_buffer_func_t `name` of src/to_planar.h:65-74 (e.g. "uyvy_to_nv12") on device tensors"""
    d = ToPlanarData()
    d.width, d.height, d.in_data = width, height, src.data_ptr()
    for i, (t, ls) in enumerate(zip(planes, linesizes)):
        d.out_data[i], d.out_linesize[i] = t.data_ptr(), ls
    _check(getattr(_L, "ugb200_" + name)(ctypes.byref(d), _stream(stream)), "ugb200_" + name)
    return planes


def from_planar(name, planes, linesizes, width, height, out, out_pitch, in_depth=0, rgb_shift=(0, 8, 16), stream=None):
    """decode_planar_func_t `name` of src/from_planar.h:88-115 (e.g. "gbrp10le_to_rgb") on device tensors"""
    d = FromPlanarData()
    d.width, d.height, d.out_data, d.out_pitch, d.in_depth = width, height, out.data_ptr(), out_pitch, in_depth
    for i, (t, ls) in enumerate(zip(planes, linesizes)):
        d.in_data[i], d.in_linesize[i] = t.data_ptr(), ls
    d.rgb_shift[0], d.rgb_shift[1], d.rgb_shift[2] = rgb_shift
    _check(getattr(_L, "ugb200_" + name)(ctypes.byref(d), _stream(stream)), "ugb200_" + name)
    return out


def deinterlace_ex(codec, src, src_linesize, lines, dst=None, dst_pitch=None, stream=None):
    """vc_deinterlace_ex (src/video_codec.c:722-854) on device tensors; dst=src for the in-place form"""
    dst_pitch = src_linesize if dst_pitch is None else dst_pitch
    if dst is None:
        dst = torch.zeros(dst_pitch * lines, dtype=torch.uint8, device=src.device)
    rc = _L.ugb200_vc_deinterlace_ex(int(codec), _ptr(src), src_linesize, _ptr(dst), dst_pitch, lines, _stream(stream))
    _check(rc, f"ugb200_vc_deinterlace_ex({Codec(codec).name})")
    return dst


def deinterlace(buf, linesize, lines, stream=None):
    """vc_deinterlace (src/video_codec.c:597-711), in place on a device tensor"""
    _check(_L.ugb200_vc_deinterlace(_ptr(buf), linesize, lines, _stream(stream)), "ugb200_vc_deinterlace")
    return buf


def il_upper_to_merged(src, linesize, height, dst=None, stream=None):
    """il_upper_to_merged (src/video_frame.c:332-355); dst=None works in place"""
    dst = src if dst is None else dst
    _check(_L.ugb200_il_upper_to_merged(_ptr(dst), _ptr(src), linesize, height, _stream(stream)), "ugb200_il_upper_to_merged")
    return dst


def il_merged_to_upper(src, linesize, height, dst=None, stream=None):
    """il_merged_to_upper (src/video_frame.c:357-379); dst=None works in place"""
    dst = src if dst is None else dst
    _check(_L.ugb200_il_merged_to_upper(_ptr(dst), _ptr(src), linesize, height, _stream(stream)), "ugb200_il_merged_to_upper")
    return dst


def _pp_out(src, linesize, height, dst, pitch):
    """dst=None allocates a zeroed frame: double_framerate's call 0 at odd height leaves row height-1 as it finds it
    (and `:d` blends it into row height-2), as the reference does"""
    pitch = linesize if pitch is None else pitch
    if dst is None:
        dst = torch.zeros(pitch * height, dtype=torch.uint8, device=src.device)
    return dst, pitch


def double_framerate(codec, prev, cur, linesize, height, call, deinterlace=False, dst=None, pitch=None, stream=None):
    """double_framerate (src/vo_postprocess/temporal-deint.c:240-277) on device tensors: call 0 weaves cur's even rows
    with prev's odd rows, call 1 is cur; deinterlace=True is the `:d` option.  At odd height call 0 leaves row height-1 of
    dst as it is, and `:d` blends it into row height-2, as the reference does: pass dst=None for a zeroed frame."""
    dst, pitch = _pp_out(cur, linesize, height, dst, pitch)
    rc = _L.ugb200_pp_double_framerate(int(codec), _ptr(prev), _ptr(cur), linesize, height, call, int(bool(deinterlace)), _ptr(dst), pitch,
                                       _stream(stream))
    _check(rc, f"ugb200_pp_double_framerate({Codec(codec).name})")
    return dst


def deinterlace_bob(cur, linesize, height, call, dst=None, pitch=None, stream=None):
    """deinterlace_bob (src/vo_postprocess/temporal-deint.c:279-300): call 0 doubles the even rows, call 1 the odd"""
    dst, pitch = _pp_out(cur, linesize, height, dst, pitch)
    _check(_L.ugb200_pp_bob(_ptr(cur), linesize, height, call, _ptr(dst), pitch, _stream(stream)), "ugb200_pp_bob")
    return dst


def deinterlace_linear(codec, cur, linesize, height, call, dst=None, pitch=None, stream=None):
    """deinterlace_linear (src/vo_postprocess/temporal-deint.c:442-466): the call's field, missing rows interpolated"""
    dst, pitch = _pp_out(cur, linesize, height, dst, pitch)
    rc = _L.ugb200_pp_linear(int(codec), _ptr(cur), linesize, height, call, _ptr(dst), pitch, _stream(stream))
    _check(rc, f"ugb200_pp_linear({Codec(codec).name})")
    return dst


def interlace(even_rows, odd_rows, linesize, height, dst=None, pitch=None, stream=None):
    """interlace (src/vo_postprocess/interlace.c:159-190): out row i from even_rows for even i, from odd_rows for odd i"""
    dst, pitch = _pp_out(even_rows, linesize, height, dst, pitch)
    _check(_L.ugb200_pp_interlace(_ptr(even_rows), _ptr(odd_rows), linesize, height, _ptr(dst), pitch, _stream(stream)), "ugb200_pp_interlace")
    return dst


# matrix2.c's y601_y709_matrix (`matrix2:y601_to_y709`), as UGB200_CF_Y601_TO_Y709 in include/ugb200.h
Y601_TO_Y709 = (1, -0.11555, -0.207938, 0, 1.01864, 0.114618, 0, 0.075049, 1.025327)


def _cf_out(src, nbytes, dst):
    """dst=None allocates a zeroed frame: grayscale leaves the last 2 * h bytes of an odd-width frame as it finds them"""
    return torch.zeros(nbytes, dtype=torch.uint8, device=src.device) if dst is None else dst


def _matrix9(m):
    m = (ctypes.c_double * 9)(*[float(x) for x in m])
    assert len(m) == 9
    return m


class gamma:
    """gamma:g[:8|:16] (src/capture_filter/gamma.cpp): holds the four tables, built once on the host, on the device"""

    def __init__(self, g):
        self.g = float(g)
        self._h = _L.ugb200_cf_gamma_create(self.g)
        if not self._h:
            raise RuntimeError("ugb200_cf_gamma_create failed")

    def __call__(self, codec, src, width, height, out_depth=0, dst=None, stream=None):
        """RGB or RG48 in; out_depth 0 keeps the depth, 8 gives RGB, 16 RG48"""
        in_bits = 8 if Codec(codec) == Codec.RGB else 16
        out_bits = out_depth or in_bits
        dst = _cf_out(src, width * height * 3 * out_bits // 8, dst)
        rc = _L.ugb200_cf_gamma(self._h, int(codec), int(out_depth), width, height, _ptr(src), _ptr(dst), _stream(stream))
        _check(rc, f"ugb200_cf_gamma({Codec(codec).name}, {out_depth})")
        return dst

    def close(self):
        if self._h:
            _L.ugb200_cf_gamma_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()


def matrix(codec, src, width, height, m, check_bounds=True, dst=None, stream=None):
    """matrix:a:...:i[:no-bound-check] (src/capture_filter/matrix.c): UYVY -> RGB, RGB -> RGB, RG48 -> RG48"""
    out_codec = Codec.RGB if Codec(codec) == Codec.UYVY else codec
    dst = _cf_out(src, vc_get_linesize(width, out_codec) * height, dst)
    rc = _L.ugb200_cf_matrix(int(codec), width, height, _matrix9(m), int(bool(check_bounds)), _ptr(src), _ptr(dst), _stream(stream))
    _check(rc, f"ugb200_cf_matrix({Codec(codec).name})")
    return dst


def matrix2(codec, src, width, height, m=Y601_TO_Y709, dst=None, stream=None):
    """matrix2:a:...:i (src/capture_filter/matrix2.c) on UYVY, v210 or Y416, in the same codec"""
    dst = _cf_out(src, vc_get_linesize(width, codec) * height, dst)
    rc = _L.ugb200_cf_matrix2(int(codec), width, height, _matrix9(m), _ptr(src), _ptr(dst), _stream(stream))
    _check(rc, f"ugb200_cf_matrix2({Codec(codec).name})")
    return dst


def grayscale(src, width, height, dst=None, stream=None):
    """grayscale (src/capture_filter/grayscale.c) on UYVY: chroma 127, luma copied over the first 2 * w * h bytes"""
    dst = _cf_out(src, vc_get_linesize(width, Codec.UYVY) * height, dst)
    _check(_L.ugb200_cf_grayscale(width, height, _ptr(src), _ptr(dst), _stream(stream)), "ugb200_cf_grayscale")
    return dst


class AvPlanes(ctypes.Structure):
    """struct ugb200_av_planes (include/ugb200_lavc.h): AVFrame::data / AVFrame::linesize"""
    _fields_ = [("data", ctypes.c_void_p * 4), ("linesize", ctypes.c_int * 4)]


AV_PIXFMT = {n: i for i, n in enumerate(["NONE", "YUV420P", "YUV422P", "YUV444P", "NV12", "P010LE", "YUV420P10LE", "YUV422P10LE", "YUV444P10LE", "YUV422P12LE",
                                          "YUV444P12LE", "YUV422P16LE", "YUV444P16LE", "GBRP"])}


def av_plane_shapes(av_pixfmt, width, height, pad=0):
    """[(linesize bytes, rows)] of the planes of a frame of `av_pixfmt` (name), rows padded by `pad` bytes"""
    f = av_pixfmt
    bps = 1 if f in ("YUV420P", "YUV422P", "YUV444P", "NV12", "GBRP") else 2
    hs = 0 if "444" in f or f == "GBRP" else 1
    vs = 1 if "420" in f or f in ("NV12", "P010LE") else 0
    cw, ch = (width + (1 << hs) - 1) >> hs, (height + (1 << vs) - 1) >> vs
    if f in ("NV12", "P010LE"):
        return [(width * bps + pad, height), (cw * 2 * bps + pad, ch)]
    return [(width * bps + pad, height), (cw * bps + pad, ch), (cw * bps + pad, ch)]


def to_lavc(in_codec, av_pixfmt, src, width, height, planes=None, pad=0, stream=None):
    """ugb200_to_lavc_convert: device frame of `in_codec` -> list of device plane tensors of `av_pixfmt` (a name of AV_PIXFMT)"""
    shapes = av_plane_shapes(av_pixfmt, width, height, pad)
    if planes is None:
        planes = [torch.zeros(ls * rows, dtype=torch.uint8, device=src.device) for ls, rows in shapes]
    p = AvPlanes()
    for i, (t, (ls, _)) in enumerate(zip(planes, shapes)):
        p.data[i], p.linesize[i] = t.data_ptr(), ls
    _check(_L.ugb200_to_lavc_convert(int(in_codec), AV_PIXFMT[av_pixfmt], ctypes.byref(p), _ptr(src), width, height, _stream(stream)), "ugb200_to_lavc_convert")
    return planes


def from_lavc(av_pixfmt, out_codec, planes, linesizes, width, height, dst, pitch, rgb_shift=(0, 8, 16), stream=None):
    """get_av_to_uv_cuda_conversion + av_to_uv_convert_cuda shape: device planes -> device frame of `out_codec`"""
    st = _L.ugb200_get_av_to_uv_conversion(AV_PIXFMT[av_pixfmt], int(out_codec))
    if not st:
        raise RuntimeError(f"no av -> uv conversion {av_pixfmt} -> {out_codec}")
    p = AvPlanes()
    for i, (t, ls) in enumerate(zip(planes, linesizes)):
        p.data[i], p.linesize[i] = t.data_ptr(), ls
    shifts = (ctypes.c_int * 3)(*rgb_shift)
    try:
        _check(_L.ugb200_av_to_uv_convert(st, _ptr(dst), ctypes.byref(p), width, height, pitch, shifts, _stream(stream)), "ugb200_av_to_uv_convert")
        torch.cuda.current_stream().synchronize()
    finally:
        h = ctypes.c_void_p(st)
        _L.ugb200_av_to_uv_conversion_destroy(ctypes.byref(h))
    return dst


def bind_host_to_device(device):
    """cuda_wrapper_bind_thread_to_device: CPU affinity + preferred memory node of the calling thread := the GPU's NUMA node; returns the node or -1"""
    return _L.cuda_wrapper_bind_thread_to_device(int(device))


def pinned_near(nbytes, device):
    """pinned host buffer whose pages live on the GPU's NUMA node (cuda_wrapper_malloc_host_near); returns a numpy uint8 view (never freed: bench buffers)"""
    import numpy as np
    p = ctypes.c_void_p()
    _check(_L.cuda_wrapper_malloc_host_near(ctypes.byref(p), nbytes, int(device)), "cuda_wrapper_malloc_host_near")
    return np.ctypeslib.as_array(ctypes.cast(p, ctypes.POINTER(ctypes.c_uint8)), shape=(nbytes,))


class JpegParams(ctypes.Structure):
    _fields_ = [("quality", ctypes.c_int), ("restart_interval", ctypes.c_int), ("interleaved", ctypes.c_int)]


class JpegParamsEx(ctypes.Structure):
    """struct ugb200_jpeg_params_ex: subsampling 0 (native) / 444 / 422 / 420, or 4444 with Codec.RGBA (R G B A, the alpha channel
    as a fourth component); color_space one of JPEG_CS"""
    _fields_ = [("base", JpegParams), ("subsampling", ctypes.c_int), ("color_space", ctypes.c_int)]


JPEG_CS = {"native": 0, "Y601": 1, "Y601full": 2, "Y709": 3, "RGB": 4}  # UGB200_JPEG_CS_* = gpujpeg_opts::internal_cs


class JpegEncoder:
    """ugb200_jpeg_* (include/ugb200_jpeg.h): the stage src/video_compress/gpujpeg.cpp delegates to libgpujpeg."""

    def __init__(self, stream=None):
        self._stream = stream if stream is not None else torch.cuda.current_stream()
        self._h = _L.ugb200_jpeg_encoder_create(ctypes.c_void_p(self._stream.cuda_stream))
        if not self._h:
            raise RuntimeError("ugb200_jpeg_encoder_create failed")

    def close(self):
        if self._h and _L is not None:
            _L.ugb200_jpeg_encoder_destroy(self._h)
        self._h = None

    def __del__(self):
        self.close()

    def _params(self, quality, restart_interval, interleaved=False):
        p = JpegParams()
        _L.ugb200_jpeg_default_params(ctypes.byref(p))
        if quality is not None:
            p.quality = quality
        p.restart_interval = restart_interval
        p.interleaved = 1 if interleaved else 0
        return p

    def _params_ex(self, quality, restart_interval, interleaved, subsampling, color_space):
        p = JpegParamsEx()
        _L.ugb200_jpeg_default_params_ex(ctypes.byref(p))
        p.base = self._params(quality, restart_interval, interleaved)
        p.subsampling, p.color_space = subsampling, color_space
        return p

    @staticmethod
    def _use_ex(codec, subsampling, color_space):
        """the _ex entry points only for what the plain ones cannot do: existing callers keep the calls they make"""
        return bool(subsampling or color_space) or int(codec) == int(Codec.I420)

    def encode_device(self, src, width, height, codec, quality=None, restart_interval=0, pitch=0, interleaved=False, subsampling=0, color_space=0):
        """asynchronous; returns nothing — call result() for the bytes.  subsampling / color_space: see JpegParamsEx"""
        if self._use_ex(codec, subsampling, color_space):
            p = self._params_ex(quality, restart_interval, interleaved, subsampling, color_space)
            _check(_L.ugb200_jpeg_encode_device_ex(self._h, _ptr(src), pitch, width, height, int(codec), ctypes.byref(p)), "ugb200_jpeg_encode_device_ex")
            return
        p = self._params(quality, restart_interval, interleaved)
        _check(_L.ugb200_jpeg_encode_device(self._h, _ptr(src), pitch, width, height, int(codec), ctypes.byref(p)), "ugb200_jpeg_encode_device")

    def result(self):
        """waits for the encode; returns the stream as bytes"""
        ptr, n = ctypes.c_void_p(), ctypes.c_size_t()
        _check(_L.ugb200_jpeg_result_device(self._h, ctypes.byref(ptr), ctypes.byref(n)), "ugb200_jpeg_result_device")
        host = (ctypes.c_uint8 * n.value)()
        _check(_L.cuda_wrapper_memcpy(host, ptr, n.value, 1), "cuda_wrapper_memcpy")
        return bytes(host)

    def encode(self, src, width, height, codec, quality=None, restart_interval=0, pitch=0, interleaved=False, subsampling=0, color_space=0):
        """gpujpeg_encoder_encode: src is a host numpy array or a CUDA tensor; returns the JPEG bytes"""
        if isinstance(src, torch.Tensor):
            sp, is_dev = _ptr(src), 1
        else:
            sp, is_dev = ctypes.c_void_p(src.ctypes.data), 0
        if self._use_ex(codec, subsampling, color_space):
            import numpy as np
            p = self._params_ex(quality, restart_interval, interleaved, subsampling, color_space)
            dst, n = np.empty(width * height * 3 + 4096, dtype=np.uint8), ctypes.c_size_t()
            _check(_L.ugb200_jpeg_encode_into_ex(self._h, sp, is_dev, pitch, width, height, int(codec), ctypes.byref(p), ctypes.c_void_p(dst.ctypes.data),
                                                 dst.size, ctypes.byref(n)), "ugb200_jpeg_encode_into_ex")
            return dst[:n.value].tobytes()
        p = self._params(quality, restart_interval, interleaved)
        out, n = ctypes.c_void_p(), ctypes.c_size_t()
        _check(_L.ugb200_jpeg_encode(self._h, sp, is_dev, pitch, width, height, int(codec), ctypes.byref(p), ctypes.byref(out), ctypes.byref(n)),
               "ugb200_jpeg_encode")
        return ctypes.string_at(out.value, n.value)

    def result_size(self):
        """waits for the encode; returns the stream length only (the stream stays on the device)"""
        n = ctypes.c_size_t()
        _check(_L.ugb200_jpeg_result_device(self._h, None, ctypes.byref(n)), "ugb200_jpeg_result_device")
        return n.value

    def stage_timing(self, enable=True):
        _check(_L.ugb200_jpeg_encoder_stage_timing(self._h, 1 if enable else 0), "ugb200_jpeg_encoder_stage_timing")

    def stage_times(self):
        """device microseconds of the last encode: (DCT + entropy kernel, segment assembly kernel, offset scan, compaction)"""
        us = (ctypes.c_float * 4)()
        _check(_L.ugb200_jpeg_encoder_stage_times(self._h, us), "ugb200_jpeg_encoder_stage_times")
        return tuple(float(x) for x in us)

    def coefficients(self):
        ptr, n = ctypes.c_void_p(), ctypes.c_size_t()
        _check(_L.ugb200_jpeg_debug_coefficients(self._h, ctypes.byref(ptr), ctypes.byref(n)), "ugb200_jpeg_debug_coefficients")
        import numpy as np
        host = np.empty(n.value, dtype=np.int16)
        _check(_L.cuda_wrapper_memcpy(ctypes.c_void_p(host.ctypes.data), ptr, n.value * 2, 1), "cuda_wrapper_memcpy")
        return host


def _bytes_ptr(b):
    """address of a bytes object's buffer without copying it (the C side only reads)"""
    return ctypes.cast(ctypes.c_char_p(b), ctypes.c_void_p)


class JpegImageInfo(ctypes.Structure):
    _fields_ = [("width", ctypes.c_int), ("height", ctypes.c_int), ("components", ctypes.c_int), ("h_samp", ctypes.c_int), ("v_samp", ctypes.c_int),
                ("adobe_transform", ctypes.c_int), ("restart_interval", ctypes.c_int), ("native_codec", ctypes.c_int)]


def jpeg_image_info(stream):
    """gpujpeg_decoder_get_image_info (src/video_decompress/gpujpeg.c:212): host-only header probe"""
    info = JpegImageInfo()
    _check(_L.ugb200_jpeg_get_image_info(_bytes_ptr(stream), len(stream), ctypes.byref(info)), "ugb200_jpeg_get_image_info")
    return info


class JpegSyncStats(ctypes.Structure):
    _fields_ = [("scans", ctypes.c_int), ("rounds", ctypes.c_int), ("subsequences", ctypes.c_long)]


class JpegDecoder:
    """ugb200_jpeg_decode*: the stage src/video_decompress/gpujpeg.c delegates to libgpujpeg."""

    def __init__(self, stream=None):
        self._stream = stream if stream is not None else torch.cuda.current_stream()
        self._h = _L.ugb200_jpeg_decoder_create(ctypes.c_void_p(self._stream.cuda_stream))
        if not self._h:
            raise RuntimeError("ugb200_jpeg_decoder_create failed")

    def close(self):
        if self._h and _L is not None:
            _L.ugb200_jpeg_decoder_destroy(self._h)
        self._h = None

    def __del__(self):
        self.close()

    def last_sync(self):
        """what the last decode's self-synchronising Huffman route did: {"scans", "subsequences", "rounds"} (scans 0: one thread per restart segment)"""
        st = JpegSyncStats()
        _check(_L.ugb200_jpeg_decoder_last_sync(self._h, ctypes.byref(st)), "ugb200_jpeg_decoder_last_sync")
        return {"scans": st.scans, "subsequences": st.subsequences, "rounds": st.rounds}

    def set_upsampling(self, mode):
        """ugb200_jpeg_decoder_set_upsampling: chroma of RGB / RGBA output in a colour space, ``"replicate"`` (the default) or ``"fancy"``
        (libjpeg's interpolation; 4:2:2 and 4:2:0 streams), or its value, for every later decode"""
        m = JPEG_UPSAMPLE[mode] if isinstance(mode, str) else int(mode)
        _check(_L.ugb200_jpeg_decoder_set_upsampling(self._h, m), "ugb200_jpeg_decoder_set_upsampling")

    def decode(self, stream, out_codec, shifts=(0, 8, 16), device=False, pitch=0, out=None, sync=True, color_space=None, out_cs=None):
        """bytes -> numpy array (host) or CUDA tensor (device=True) holding height rows of vc_get_linesize(width, out_codec) bytes.
        ``color_space`` None: ugb200_jpeg_decode (the stream's samples, RGB / RGBA through UltraGrid's line converters); else one of
        JPEG_CS (``"native"``, ``"Y709"``, ``"Y601"``, ``"Y601full"``, ``"auto"``) or its value: ugb200_jpeg_decode_cs.  ``out_cs`` not None (``"native"``, ``"Y709"``, ``"Y601"``, ``"Y601full"`` or its value):
        ugb200_jpeg_decode_to, UYVY / I420 / VUYA output converted from ``color_space`` (None: native) to ``out_cs``"""
        info = jpeg_image_info(stream)
        ls = pitch or vc_get_linesize(info.width, out_codec)
        nbytes = ls * info.height
        if int(out_codec) == int(Codec.I420):  # three tight planes
            nbytes = info.width * info.height + 2 * ((info.width + 1) // 2) * ((info.height + 1) // 2)
        buf = _bytes_ptr(stream)
        if device:
            if out is None:
                out = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
            elif out.numel() * out.element_size() < nbytes:
                raise ValueError(f"out holds {out.numel() * out.element_size()} bytes, the stream decodes to {nbytes}")
            self._decode(buf, len(stream), _ptr(out), 1, ls, out_codec, shifts, color_space, out_cs)
            if sync:
                self._stream.synchronize()
            return out
        import numpy as np
        out = np.zeros(nbytes, dtype=np.uint8)
        self._decode(buf, len(stream), ctypes.c_void_p(out.ctypes.data), 0, ls, out_codec, shifts, color_space, out_cs)
        return out

    def decode_to(self, stream, out_codec, stream_cs="auto", out_cs="Y709", **kw):
        """ugb200_jpeg_decode_to: decode() with UYVY / I420 / VUYA output converted from ``stream_cs`` to the colour space ``out_cs``; RGB / RGBA
        output is decode(color_space=stream_cs).  Also decodes grayscale streams."""
        return self.decode(stream, out_codec, color_space=stream_cs, out_cs=out_cs, **kw)

    def _decode(self, buf, n, dst, is_device, pitch, out_codec, shifts, color_space, out_cs=None):
        to_cs = lambda c: 0 if c is None else JPEG_CS[c] if isinstance(c, str) else int(c)
        if out_cs is not None:
            _check(_L.ugb200_jpeg_decode_to(self._h, buf, n, dst, is_device, pitch, int(out_codec), *shifts, to_cs(color_space), to_cs(out_cs)),
                   "ugb200_jpeg_decode_to")
        elif color_space is None:
            _check(_L.ugb200_jpeg_decode(self._h, buf, n, dst, is_device, pitch, int(out_codec), *shifts), "ugb200_jpeg_decode")
        else:
            cs = JPEG_CS[color_space] if isinstance(color_space, str) else int(color_space)
            _check(_L.ugb200_jpeg_decode_cs(self._h, buf, n, dst, is_device, pitch, int(out_codec), *shifts, cs), "ugb200_jpeg_decode_cs")


# UGB200_JPEG_CS_* of include/ugb200_jpeg.h
JPEG_CS = {"native": 0, "Y601": 1, "Y601full": 2, "Y709": 3, "RGB": 4, "auto": 5}
# UGB200_JPEG_UPSAMPLE_*
JPEG_UPSAMPLE = {"replicate": 0, "fancy": 1}


def jpeg_stream_color_space(stream):
    """ugb200_jpeg_stream_color_space: the colour space the stream declares, as a key of JPEG_CS (raises on a refusal)"""
    rc = _L.ugb200_jpeg_stream_color_space(_bytes_ptr(stream), len(stream))
    _check(min(rc, 0), "ugb200_jpeg_stream_color_space")
    return {v: k for k, v in JPEG_CS.items()}[rc]


class LdgmCoder:
    """ugb200_ldgm_* (include/ugb200_ldgm.h): LDGM FEC of the reference's LDGM_session (ldgm/src/ldgm-session.h), on the GPU.
    ``pcm`` is the compact parity-check matrix as set_pcMatrix reads it: an int32 array of m rows of w_f entries."""

    def __init__(self, pcm, k, m, stream=None):
        self._stream = stream if stream is not None else torch.cuda.current_stream()
        self._h = _L.ugb200_ldgm_create(ctypes.c_void_p(self._stream.cuda_stream))
        if not self._h:
            raise RuntimeError("ugb200_ldgm_create failed")
        self.set_matrix(pcm, k, m)

    def set_matrix(self, pcm, k, m):
        import numpy as np
        pcm = np.ascontiguousarray(pcm, dtype=np.int32).reshape(m, -1)
        _check(_L.ugb200_ldgm_set_matrix(self._h, ctypes.c_void_p(pcm.ctypes.data), k, m, pcm.shape[1]), "ugb200_ldgm_set_matrix")
        self.k, self.m = k, m

    def close(self):
        if self._h and _L is not None:
            _L.ugb200_ldgm_destroy(self._h)
        self._h = None

    def __del__(self):
        self.close()

    def buffer_size(self, payload_size):
        """(encoded length, packet size) for a header + frame of payload_size bytes"""
        ps = ctypes.c_int()
        n = _L.ugb200_ldgm_buffer_size(self._h, payload_size, ctypes.byref(ps))
        if n < 0:
            raise RuntimeError(f"ugb200_ldgm_buffer_size failed with code {n}")
        return n, ps.value

    def encode(self, frame, hdr=b"", out=None):
        """encode_hdr_frame.  ``frame`` is bytes / a uint8 numpy array (host) or a uint8 CUDA tensor (device, may be a view at any
        offset); returns a uint8 numpy array, or for a device frame a CUDA tensor (``out`` may supply either).  A device encode is
        asynchronous and ordered after, and before, the work of the current torch stream."""
        import numpy as np
        hdr = bytes(hdr)
        n_out = ctypes.c_int()
        if isinstance(frame, torch.Tensor):
            total, _ = self.buffer_size(len(hdr) + frame.numel())
            if out is None:
                out = torch.empty(total, dtype=torch.uint8, device=frame.device)
            # the coder runs on its own stream: it starts after the work queued so far on the caller's stream (which made the frame),
            # and the caller's stream continues after the encode; the allocator keeps both tensors until the coder's stream is done
            caller = torch.cuda.current_stream(frame.device)
            if caller != self._stream:
                self._stream.wait_stream(caller)
            _check(_L.ugb200_ldgm_encode_device(self._h, hdr, len(hdr), _ptr(frame), frame.numel(), _ptr(out), out.numel(),
                                                ctypes.byref(n_out)), "ugb200_ldgm_encode_device")
            if caller != self._stream:
                frame.record_stream(self._stream)
                out.record_stream(self._stream)
                caller.wait_stream(self._stream)
            return out[:n_out.value]
        src = np.frombuffer(frame, dtype=np.uint8) if isinstance(frame, (bytes, bytearray)) else np.ascontiguousarray(frame, dtype=np.uint8)
        total, _ = self.buffer_size(len(hdr) + src.size)
        if out is None:
            out = np.empty(total, dtype=np.uint8)
        _check(_L.ugb200_ldgm_encode_frame(self._h, hdr, len(hdr), ctypes.c_void_p(src.ctypes.data), src.size, ctypes.c_void_p(out.ctypes.data),
                                           out.size, ctypes.byref(n_out)), "ugb200_ldgm_encode_frame")
        return out[:n_out.value]

    def decode(self, buf, ranges):
        """decode_frame on a writable uint8 numpy array, in place; ``ranges`` is a dict or a list of (offset, length) of received bytes.
        Returns the frame size of the header (the payload starts at buf[4:]), or 0 when the frame cannot be recovered."""
        import numpy as np
        items = list(ranges.items()) if isinstance(ranges, dict) else list(ranges)
        r = np.ascontiguousarray(np.array(items, dtype=np.int32).reshape(-1, 2))
        fs = ctypes.c_int()
        _check(_L.ugb200_ldgm_decode(self._h, ctypes.c_void_p(buf.ctypes.data), buf.size, ctypes.c_void_p(r.ctypes.data), len(items),
                                     ctypes.byref(fs)), "ugb200_ldgm_decode")
        return fs.value
