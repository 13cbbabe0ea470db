"""ctypes loader of the in-tree C-ABI library.  Fails loudly when it is missing (no fallback)."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libugb200.so")

# every symbol include/*.h declares, with (restype, argtypes); tests check the export list against this
_vp, _i, _l, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_long, ctypes.c_size_t
SIGNATURES = {
    # include/cuda_dxt.h
    "cuda_rgb_to_dxt1": (_i, [_vp, _vp, _i, _i, _vp]),
    "cuda_yuv_to_dxt1": (_i, [_vp, _vp, _i, _i, _vp]),
    "cuda_rgb_to_dxt6": (_i, [_vp, _vp, _i, _i, _vp]),
    "cuda_yuv_to_dxt6": (_i, [_vp, _vp, _i, _i, _vp]),
    "cuda_yuv422_to_yuv444": (_i, [_vp, _vp, _i, _vp]),
    # include/cuda_wrapper.h
    "cuda_wrapper_free": (_i, [_vp]),
    "cuda_wrapper_free_host": (_i, [_vp]),
    "cuda_wrapper_host_alloc": (_i, [ctypes.POINTER(_vp), _sz, ctypes.c_uint]),
    "cuda_wrapper_malloc": (_i, [ctypes.POINTER(_vp), _sz]),
    "cuda_wrapper_malloc_host": (_i, [ctypes.POINTER(_vp), _sz]),
    "cuda_wrapper_memcpy": (_i, [_vp, _vp, _sz, _i]),
    "cuda_wrapper_last_error_string": (ctypes.c_char_p, []),
    "cuda_wrapper_set_device": (_i, [_i]),
    "cuda_wrapper_get_last_error": (_i, []),
    "cuda_wrapper_get_error_string": (ctypes.c_char_p, [_i]),
    "cuda_wrapper_print_devices_info": (None, [ctypes.c_bool]),
    "cuda_wrapper_device_reset": (None, []),
    "cuda_wrapper_get_device_count": (_i, [ctypes.POINTER(_i)]),
    "cuda_wrapper_stream_create": (_i, [ctypes.POINTER(_vp)]),
    "cuda_wrapper_stream_destroy": (_i, [_vp]),
    "cuda_wrapper_stream_synchronize": (_i, [_vp]),
    "cuda_wrapper_memcpy_async": (_i, [_vp, _vp, _sz, _i, _vp]),
    "cuda_wrapper_memcpy2d": (_i, [_vp, _sz, _vp, _sz, _sz, _sz, _i]),
    "cuda_wrapper_device_numa_node": (_i, [_i]),
    "cuda_wrapper_bind_thread_to_device": (_i, [_i]),
    "cuda_wrapper_malloc_host_near": (_i, [ctypes.POINTER(_vp), _sz, _i]),
    # include/ugb200.h
    "ugb200_rgb_to_dxt1_async": (_i, [_vp, _vp, _i, _i, _vp]),
    "ugb200_yuv_to_dxt1_async": (_i, [_vp, _vp, _i, _i, _vp]),
    "ugb200_rgb_to_dxt6_async": (_i, [_vp, _vp, _i, _i, _vp]),
    "ugb200_yuv_to_dxt6_async": (_i, [_vp, _vp, _i, _i, _vp]),
    "ugb200_uyvy_to_dxt1_async": (_i, [_vp, _vp, _i, _i, _l, _vp]),
    "ugb200_uyvy_to_dxt6_async": (_i, [_vp, _vp, _i, _i, _l, _vp]),
    "ugb200_dxt1_to_rgb": (_i, [_vp, _vp, _i, _i, _l, _i, _vp]),
    "ugb200_dxt5ycocg_to_rgb": (_i, [_vp, _vp, _i, _i, _l, _i, _vp]),
    "ugb200_vc_copyline": (_i, [_i, _vp, _l, _vp, _l, _i, _i, _l, _i, _i, _i, _vp]),
    "ugb200_pixfmt_supported": (_i, [_i, _i]),
    "ugb200_pixfmt_staged_mode": (_i, [_i]),
    "ugb200_pixfmt_convert": (_i, [_i, _i, _vp, _l, _vp, _l, _i, _i, _l, _i, _i, _i, _vp]),
    "ugb200_v210_to_p010le": (_i, [_vp, _l, _vp]),
    # the other to_planar.h / from_planar.h functions: (struct *, stream)
    "ugb200_y216_to_p010le": (_i, [_vp, _vp]),
    "ugb200_uyvy_to_nv12": (_i, [_vp, _vp]),
    "ugb200_rgba_to_bgra": (_i, [_vp, _vp]),
    "ugb200_vuya_to_i444": (_i, [_vp, _vp]),
    "ugb200_uyvy_to_i420": (_i, [_vp, _vp]),
    "ugb200_r12l_to_gbrp12le": (_i, [_vp, _vp]),
    "ugb200_r12l_to_gbrp16le": (_i, [_vp, _vp]),
    "ugb200_r12l_to_rgbp12le": (_i, [_vp, _vp]),
    "ugb200_gbrap_to_rgb": (_i, [_vp, _vp]),
    "ugb200_gbrap_to_rgba": (_i, [_vp, _vp]),
    "ugb200_gbrp10le_to_rgb": (_i, [_vp, _vp]),
    "ugb200_gbrp12le_to_rgb": (_i, [_vp, _vp]),
    "ugb200_gbrp16le_to_rgb": (_i, [_vp, _vp]),
    "ugb200_rgbpXX_to_rgb": (_i, [_vp, _vp]),
    "ugb200_gbrp10le_to_rgba": (_i, [_vp, _vp]),
    "ugb200_gbrp12le_to_rgba": (_i, [_vp, _vp]),
    "ugb200_gbrp16le_to_rgba": (_i, [_vp, _vp]),
    "ugb200_gbrp10le_to_rg48": (_i, [_vp, _vp]),
    "ugb200_gbrp12le_to_rg48": (_i, [_vp, _vp]),
    "ugb200_gbrp16le_to_rg48": (_i, [_vp, _vp]),
    "ugb200_rgbpXXle_to_rg48": (_i, [_vp, _vp]),
    "ugb200_gbrp10le_to_r10k": (_i, [_vp, _vp]),
    "ugb200_gbrp12le_to_r10k": (_i, [_vp, _vp]),
    "ugb200_gbrp16le_to_r10k": (_i, [_vp, _vp]),
    "ugb200_rgbpXXle_to_r10k": (_i, [_vp, _vp]),
    "ugb200_gbrp12le_to_r12l": (_i, [_vp, _vp]),
    "ugb200_gbrp16le_to_r12l": (_i, [_vp, _vp]),
    "ugb200_rgbpXXle_to_r12l": (_i, [_vp, _vp]),
    "ugb200_yuv444p_to_vuya": (_i, [_vp, _vp]),
    "ugb200_yuv420p_to_uyvy": (_i, [_vp, _vp]),
    "ugb200_yuv420_to_i420": (_i, [_vp, _vp]),
    "ugb200_yuv422p_to_uyvy": (_i, [_vp, _vp]),
    "ugb200_yuv422p_to_yuyv": (_i, [_vp, _vp]),
    "ugb200_yuv422pXX_to_uyvy": (_i, [_vp, _vp]),
    "ugb200_yuv422p10le_to_uyvy": (_i, [_vp, _vp]),
    "ugb200_yuv422p10le_to_v210": (_i, [_vp, _vp]),
    "ugb200_vc_deinterlace_ex": (_i, [_i, _vp, _sz, _vp, _sz, _sz, _vp]),
    "ugb200_vc_deinterlace": (_i, [_vp, _l, _i, _vp]),
    "ugb200_il_upper_to_merged": (_i, [_vp, _vp, _i, _i, _vp]),
    "ugb200_il_merged_to_upper": (_i, [_vp, _vp, _i, _i, _vp]),
    "ugb200_pp_double_framerate": (_i, [_i, _vp, _vp, _sz, _i, _i, _i, _vp, _sz, _vp]),
    "ugb200_pp_bob": (_i, [_vp, _sz, _i, _i, _vp, _sz, _vp]),
    "ugb200_pp_linear": (_i, [_i, _vp, _sz, _i, _i, _vp, _sz, _vp]),
    "ugb200_pp_interlace": (_i, [_vp, _vp, _sz, _i, _vp, _sz, _vp]),
    "ugb200_cf_gamma_create": (_vp, [ctypes.c_double]),
    "ugb200_cf_gamma_destroy": (None, [_vp]),
    "ugb200_cf_gamma": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "ugb200_cf_matrix": (_i, [_i, _i, _i, _vp, _i, _vp, _vp, _vp]),
    "ugb200_cf_matrix2": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp]),
    "ugb200_cf_grayscale": (_i, [_i, _i, _vp, _vp, _vp]),
    "ugb200_cf_flip": (_i, [_i, _i, _i, _vp, _vp, _vp]),
    "ugb200_cf_mirror": (_i, [_i, _i, _i, _vp, _vp, _vp]),
    "ugb200_cf_crop_geometry": (_i, [_i, _i, _i, _i, _i, _i, _i, ctypes.POINTER(_i)]),
    "ugb200_cf_crop": (_i, [_i, _i, _i, _i, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "ugb200_cf_split": (_i, [_i, _i, _i, _i, _i, _vp, ctypes.POINTER(_vp), _vp]),
    "ugb200_pp_border": (_i, [_i, _i, _i, ctypes.POINTER(ctypes.c_uint8), ctypes.c_uint, ctypes.c_uint, _vp, _vp, _vp]),
    "ugb200_pp_interlaced_3d": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp]),
    "ugb200_cf_logo_create": (_vp, [ctypes.POINTER(ctypes.c_uint8), ctypes.c_uint, ctypes.c_uint]),
    "ugb200_cf_logo_destroy": (None, [_vp]),
    "ugb200_cf_logo": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "ugb200_cf_r12l_to_y416_fake": (_i, [_i, _i, _i, _vp, _vp, _vp]),
    "ugb200_pp_y416_to_r12l_fake": (_i, [_i, _i, _i, _vp, _vp, _sz, _vp]),
    "ugb200_cf_resize_create": (_vp, [_i, ctypes.c_double, _i, _i, _i]),
    "ugb200_cf_resize_create2": (_vp, [_i, ctypes.c_double, _i, _i, _i]),
    "ugb200_cf_resize_destroy": (None, [_vp]),
    "ugb200_cf_resize_geometry": (_i, [_vp, _i, _i, _i, ctypes.POINTER(_i)]),
    "ugb200_cf_resize": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp]),
    # include/ugb200_jpeg.h
    "ugb200_jpeg_default_params": (None, [_vp]),
    "ugb200_jpeg_encoder_create": (_vp, [_vp]),
    "ugb200_jpeg_encoder_destroy": (None, [_vp]),
    "ugb200_jpeg_encode_device": (_i, [_vp, _vp, _l, _i, _i, _i, _vp]),
    "ugb200_jpeg_result_device": (_i, [_vp, ctypes.POINTER(_vp), ctypes.POINTER(_sz)]),
    "ugb200_jpeg_encode": (_i, [_vp, _vp, _i, _l, _i, _i, _i, _vp, ctypes.POINTER(_vp), ctypes.POINTER(_sz)]),
    "ugb200_jpeg_encode_into": (_i, [_vp, _vp, _i, _l, _i, _i, _i, _vp, _vp, _sz, ctypes.POINTER(_sz)]),
    "ugb200_jpeg_default_params_ex": (None, [_vp]),
    "ugb200_jpeg_encode_device_ex": (_i, [_vp, _vp, _l, _i, _i, _i, _vp]),
    "ugb200_jpeg_encode_into_ex": (_i, [_vp, _vp, _i, _l, _i, _i, _i, _vp, _vp, _sz, ctypes.POINTER(_sz)]),
    "ugb200_jpeg_encoder_stage_timing": (_i, [_vp, _i]),
    "ugb200_jpeg_encoder_stage_times": (_i, [_vp, ctypes.POINTER(ctypes.c_float)]),
    "ugb200_jpeg_get_image_info": (_i, [_vp, _sz, _vp]),
    "ugb200_jpeg_debug_segments": (_l, [_vp, _sz, _vp, _vp, _l]),
    "ugb200_jpeg_decoder_last_segments": (_l, [_vp, _vp, _vp, _l]),
    "ugb200_jpeg_decoder_last_sync": (_i, [_vp, _vp]),
    "ugb200_jpeg_decoder_create": (_vp, [_vp]),
    "ugb200_jpeg_decoder_destroy": (None, [_vp]),
    "ugb200_jpeg_decoder_expect": (_i, [_vp, _i, _i]),
    "ugb200_jpeg_decoder_set_upsampling": (_i, [_vp, _i]),
    "ugb200_jpeg_decode": (_i, [_vp, _vp, _sz, _vp, _i, _l, _i, _i, _i, _i]),
    "ugb200_jpeg_decode_cs": (_i, [_vp, _vp, _sz, _vp, _i, _l, _i, _i, _i, _i, _i]),
    "ugb200_jpeg_decode_to": (_i, [_vp, _vp, _sz, _vp, _i, _l, _i, _i, _i, _i, _i, _i]),
    "ugb200_jpeg_stream_color_space": (_i, [_vp, _sz]),
    "ugb200_jpeg_debug_coefficients": (_i, [_vp, ctypes.POINTER(_vp), ctypes.POINTER(_sz)]),
    # include/ugb200_ldgm.h
    "ugb200_ldgm_create": (_vp, [_vp]),
    "ugb200_ldgm_destroy": (None, [_vp]),
    "ugb200_ldgm_set_matrix": (_i, [_vp, _vp, _i, _i, _i]),
    "ugb200_ldgm_buffer_size": (_l, [_vp, _i, ctypes.POINTER(_i)]),
    "ugb200_ldgm_encode": (_i, [_vp, _vp, _vp, _i]),
    "ugb200_ldgm_encode_frame": (_i, [_vp, _vp, _i, _vp, _i, _vp, _sz, ctypes.POINTER(_i)]),
    "ugb200_ldgm_encode_device": (_i, [_vp, _vp, _i, _vp, _i, _vp, _sz, ctypes.POINTER(_i)]),
    "ugb200_ldgm_decode": (_i, [_vp, _vp, _i, _vp, _i, ctypes.POINTER(_i)]),
    # include/ugb200_lavc.h
    "ugb200_to_lavc_supported": (_i, [_i, _i]),
    "ugb200_to_lavc_convert": (_i, [_i, _i, _vp, _vp, _i, _i, _vp]),
    "ugb200_to_lavc_vid_conv_init": (_vp, [_i, _i, _i, _i]),
    "ugb200_to_lavc_vid_conv": (_vp, [_vp, _vp, _i]),
    "ugb200_to_lavc_vid_conv_destroy": (None, [_vp]),
    "ugb200_get_av_to_uv_conversion": (_vp, [_i, _i]),
    "ugb200_av_to_uv_convert": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "ugb200_av_to_uv_conversion_destroy": (None, [_vp]),
    # include/ugb200_vcompress.h
    "ugb200_set_cuda_devices": (_i, [ctypes.POINTER(_i), _i]),
    "ugb200_compress_init": (_vp, [ctypes.c_char_p]),
    "ugb200_compress_push": (_i, [_vp, _vp, _i, _i, _i, _i, ctypes.c_double]),
    "ugb200_compress_pop": (_i, [_vp, _vp, _sz, ctypes.POINTER(_sz), ctypes.POINTER(_i), ctypes.POINTER(ctypes.c_uint)]),
    "ugb200_compress_pop_ref": (_i, [_vp, ctypes.POINTER(_vp), ctypes.POINTER(_sz), ctypes.POINTER(_i), ctypes.POINTER(ctypes.c_uint)]),
    "ugb200_compress_done": (None, [_vp]),
    "ugb200_decompress_init": (_vp, [_i, _i]),
    "ugb200_decompress_module": (ctypes.c_char_p, [_vp]),
    "ugb200_decompress_reconfigure": (_i, [_vp, _i, _i, _i, _i, _i, _i, _i, _i]),
    "ugb200_decompress_frame": (_i, [_vp, _vp, _vp, ctypes.c_uint, _i, _vp]),
    "ugb200_decompress_done": (None, [_vp]),
    "ugb200_get_best_decoder_from": (_i, [_i, ctypes.POINTER(_i), _i]),
}

_lib = None


def load():
    """Load libugb200.so and bind the signatures.  Raises RuntimeError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C ultragrid_b200/csrc`). There is no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here means the library is stale
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
