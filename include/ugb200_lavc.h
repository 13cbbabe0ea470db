/* libavcodec bridge conversions on the device (SURVEY.md section 8f rank 3).
 *
 * What it replaces: the per-frame CPU conversions between UltraGrid's packed pixel formats and libavcodec's planar ones,
 * src/libavcodec/to_lavc_vid_conv.c (table uv_to_av_conversions[], :1458-1531) and src/libavcodec/from_lavc_vid_conv.c, and it fills the
 * CUDA hooks the reference ships EMPTY: to_lavc_vid_conv_cuda_init / to_lavc_vid_conv_cuda / to_lavc_vid_conv_cuda_destroy
 * (src/libavcodec/to_lavc_vid_conv_cuda.h:60-65, .cu:55-79) and get_av_to_uv_cuda_conversion / av_to_uv_convert_cuda /
 * av_to_uv_conversion_cuda_destroy (from_lavc_vid_conv_cuda.h:61-69, .cu:54-72).
 *
 * FFmpeg's headers are not part of this library's contract: a frame is described by the only AVFrame fields the conversions touch
 * (to_lavc_vid_conv.c:115-128) - plane pointers and line sizes - and the pixel format by the enum below (INTEGRATION.md shows the
 * AV_PIX_FMT_* switch of the binding).  Pointers are DEVICE pointers (the planes are what an NVENC / hardware frame context consumes).
 *
 * PARITY: to_lavc_vid_conv.c and from_lavc_vid_conv.c cannot be compiled here (libavutil / libavcodec headers absent), so this bridge is NOT
 * pinned against lavc itself.  tests/test_lavc_exact.py pins every pair it admits to a numpy restatement of the cited reference lines, and pins that
 * restatement to what the tree does allow: the colour coefficients against the reference build, identities through the unmodified to_planar.c /
 * from_planar.c objects (the idea of test/ff_codec_conversions_test.cpp:346-401), a bound of the float64 BT.709 matrix, and oracle/lavc_oracle.c. */
#ifndef UGB200_LAVC_H
#define UGB200_LAVC_H
#include "ugb200.h"

#ifdef __cplusplus
extern "C" {
#endif

enum ugb200_av_pixfmt {          /* libavutil/pixfmt.h name */
        UGB_AV_NONE = 0,
        UGB_AV_YUV420P,          /* AV_PIX_FMT_YUV420P  (and YUVJ420P) */
        UGB_AV_YUV422P,          /* AV_PIX_FMT_YUV422P  (and YUVJ422P) */
        UGB_AV_YUV444P,          /* AV_PIX_FMT_YUV444P  (and YUVJ444P) */
        UGB_AV_NV12,             /* AV_PIX_FMT_NV12 */
        UGB_AV_P010LE,           /* AV_PIX_FMT_P010LE */
        UGB_AV_YUV420P10LE, UGB_AV_YUV422P10LE, UGB_AV_YUV444P10LE,
        UGB_AV_YUV422P12LE, UGB_AV_YUV444P12LE,
        UGB_AV_YUV422P16LE, UGB_AV_YUV444P16LE,
        UGB_AV_GBRP,             /* AV_PIX_FMT_GBRP: planes G, B, R */
        UGB_AV_PIXFMT_COUNT
};

struct ugb200_av_planes {        /* AVFrame::data / AVFrame::linesize */
        unsigned char *data[4];
        int linesize[4];
};

/* Is there a device conversion for this pair (the role of get_uv_to_av_conversions(), to_lavc_vid_conv.c:1458)? */
UGB_API int ugb200_to_lavc_supported(int in_codec, int av_pixfmt);
/* One frame: `in_data` = device frame of `in_codec`, rows vc_get_linesize(width, in_codec) apart, -> planes.  Asynchronous on `stream`.
 * 0 ok, -1 bad arguments / unsupported pair / a 16-bit plane at an odd address or line size / a v210 source that is not 4-byte aligned (the
 * reference asserts both; nothing is written), -2 launch failure.  Loop bounds as the reference functions (whole v210 groups of 6, R12L groups
 * of 8, UYVY pixel pairs ...), except that no sample is written beyond a plane row's linesize. */
UGB_API int ugb200_to_lavc_convert(int in_codec, int av_pixfmt, const struct ugb200_av_planes *out, const void *in_data, int width, int height,
                                   cuda_wrapper_stream_t stream);

/* The hook shape of to_lavc_vid_conv_cuda.h:60-65.  The state owns device planes of the right size (AVFrame role); `in_data` is a HOST frame
 * (as the reference's hook gets it) unless in_is_device.  Returns the planes (device memory, valid until the next call), NULL on error. */
struct ugb200_to_lavc_conv;
UGB_API struct ugb200_to_lavc_conv *ugb200_to_lavc_vid_conv_init(int in_codec, int width, int height, int av_pixfmt);
UGB_API const struct ugb200_av_planes *ugb200_to_lavc_vid_conv(struct ugb200_to_lavc_conv *state, const char *in_data, int in_is_device);
UGB_API void ugb200_to_lavc_vid_conv_destroy(struct ugb200_to_lavc_conv **state);

/* from_lavc: planar frame of the decoder -> any UltraGrid codec (from_lavc_vid_conv_cuda.h:61-69; the reference declares YUV422P as the format the
 * CUDA path must accept).  Planes and dst are device memory; conversions go through the planar kernels (src/from_planar.c names) and, for a
 * destination the planar stage does not produce, one line converter.  rgb_shift as av_to_uv_convert_cuda. */
struct ugb200_av_to_uv_conv;
UGB_API struct ugb200_av_to_uv_conv *ugb200_get_av_to_uv_conversion(int av_pixfmt, int out_codec);
UGB_API int ugb200_av_to_uv_convert(struct ugb200_av_to_uv_conv *state, char *dst_buffer, const struct ugb200_av_planes *in_frame, int width, int height,
                                    int pitch, const int *rgb_shift, cuda_wrapper_stream_t stream);
UGB_API void ugb200_av_to_uv_conversion_destroy(struct ugb200_av_to_uv_conv **state);

#ifdef __cplusplus
}
#endif
#endif
