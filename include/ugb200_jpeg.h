/* Baseline-JPEG encode stage — the C ABI that stands where UltraGrid's GPUJPEG module calls libgpujpeg
 * (src/video_compress/gpujpeg.cpp: gpujpeg_encoder_create :353, gpujpeg_encoder_input_set_image /
 * _set_gpu_image :617-622, gpujpeg_encoder_encode :624, gpujpeg_encoder_destroy :639).
 *
 * Stream contract (what the reference configures at gpujpeg.cpp:256-369):
 *   UGB_UYVY input -> YCbCr stored as-is (no colour transform), 4:2:2, ONE interleaved scan (MCU 16x8 = Y0 Y1 Cb Cr)
 *   UGB_RGB  input -> R,G,B stored as-is, 4:4:4, THREE scans (non-interleaved), Adobe APP14 transform=0
 *   baseline sequential DCT (SOF0), Annex K Huffman tables, Annex K quantisation tables scaled by IJG quality,
 *   restart interval `restart_interval` MCUs (0 = default: 4 for UYVY, 8 for RGB — gpujpeg.cpp:351), RSTn markers.
 * The _ex calls add what GPUJPEG's `subsampling` and internal colour space options ask for (gpujpeg.cpp:262-266,292-304,332):
 *   UGB_I420 input (native 4:2:0, BT.709) -> YCbCr 4:2:0, one interleaved scan (MCU 16x16 = Y0 Y1 Y2 Y3 Cb Cr); the planes are read in place
 *   UGB_UYVY input, subsampling 420          -> the same stream; chroma of two rows averaged as uyvy_to_i420 (to_planar.c:343-378)
 *   UGB_RGB  input, Y709 | Y601 | Y601FULL   -> YCbCr 4:4:4 / 4:2:2 / 4:2:0 (subsampling 0 = 444), one scan per component (T.81 A.2: a
 *                                               component's blocks are not padded to whole MCUs) or one interleaved scan with `interleaved`;
 *                                               integer RGB_TO_Y/CB/CR of the reference at 8 bits (Y601FULL: JFIF full range)
 *   every YCbCr stream carries JFIF APP0; restart interval default 8 for RGB input, 4 otherwise.  Native parameters give the bytes of
 *   the calls without _ex.  Anything else returns -4: chroma upsampling, YCbCr -> RGB, one YCbCr matrix -> another, subsampled RGB.
 * Output capacity is width*height*3 + 4096 bytes like the reference's pool frames (gpujpeg.cpp:355).
 */
#ifndef UGB200_JPEG_H
#define UGB200_JPEG_H

#include <stddef.h>
#include <stdint.h>

#include "cuda_wrapper.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ugb200_jpeg_encoder ugb200_jpeg_encoder;

struct ugb200_jpeg_params {
        int quality;          /* 1..100; gpujpeg_set_default_parameters() gives 75 */
        int restart_interval; /* MCUs per restart segment; 0 = default for the input format */
        int interleaved;      /* RGB input only: one scan of R G B MCUs instead of one scan per component (the `interleaved` option of the
                               * reference module, gpujpeg.cpp:303,397-398); UYVY input is a single interleaved scan either way */
};

/* gpujpeg_set_default_parameters */
UGB_API void ugb200_jpeg_default_params(struct ugb200_jpeg_params *p);

/* gpujpeg_encoder_create(stream).  Uses the current CUDA device (cuda_wrapper_set_device first, like
 * gpujpeg_set_device at gpujpeg.cpp:559).  NULL on failure. */
UGB_API ugb200_jpeg_encoder *ugb200_jpeg_encoder_create(cuda_wrapper_stream_t stream);
UGB_API void ugb200_jpeg_encoder_destroy(ugb200_jpeg_encoder *enc);

/* Asynchronous device-side encode: src is a DEVICE pointer (gpujpeg_encoder_input_set_gpu_image), `codec` is UGB_UYVY or
 * UGB_RGB, pitch 0 = tightly packed.  The stream ends up in an encoder-owned device buffer.  0 ok, -1 bad args,
 * -2 CUDA failure, -4 unsupported codec, -5 (from the result call) the stream is larger than the w * h * 3 + 4096 byte output
 * buffer, the capacity the reference gives libgpujpeg at gpujpeg.cpp:355 (noise at quality ~100 only). */
UGB_API int ugb200_jpeg_encode_device(ugb200_jpeg_encoder *enc, const void *src, long pitch, int width, int height, int codec,
                                      const struct ugb200_jpeg_params *params);
enum { UGB200_JPEG_CS_NATIVE = 0, UGB200_JPEG_CS_Y601, UGB200_JPEG_CS_Y601FULL, UGB200_JPEG_CS_Y709, UGB200_JPEG_CS_RGB };  /* = gpujpeg_opts::internal_cs */
struct ugb200_jpeg_params_ex {
        struct ugb200_jpeg_params base;
        int subsampling;   /* 0 = native for the input (RGB 444, UYVY 422, I420 420), else 444 / 422 / 420 */
        int color_space;   /* UGB200_JPEG_CS_* */
};
UGB_API void ugb200_jpeg_default_params_ex(struct ugb200_jpeg_params_ex *p);
/* ugb200_jpeg_encode_device with the layouts above; `codec` also takes UGB_I420 (pitch must be 0) */
UGB_API int ugb200_jpeg_encode_device_ex(ugb200_jpeg_encoder *enc, const void *src, long pitch, int width, int height, int codec,
                                         const struct ugb200_jpeg_params_ex *params);

/* Waits for the encode and returns the device pointer and byte size of the JPEG stream. */
UGB_API int ugb200_jpeg_result_device(ugb200_jpeg_encoder *enc, const void **dev_ptr, size_t *size);

/* gpujpeg_encoder_encode: synchronous; src is host memory unless src_is_device; *out points to an encoder-owned PINNED host
 * buffer that stays valid until the next call (the reference memcpy's it into its pool frame, gpujpeg.cpp:629-630). */
UGB_API int ugb200_jpeg_encode(ugb200_jpeg_encoder *enc, const void *src, int src_is_device, long pitch, int width, int height,
                               int codec, const struct ugb200_jpeg_params *params, uint8_t **out, size_t *out_size);

/* Same, but the stream goes straight into the caller's host buffer `dst` (capacity dst_cap; pinned memory keeps the copy
 * asynchronous to other streams) - the module writes into its pooled output frame without the memcpy of gpujpeg.cpp:629-630.
 * -5 if the stream does not fit. */
UGB_API int ugb200_jpeg_encode_into(ugb200_jpeg_encoder *enc, const void *src, int src_is_device, long pitch, int width, int height,
                                    int codec, const struct ugb200_jpeg_params *params, uint8_t *dst, size_t dst_cap, size_t *out_size);

/* ugb200_jpeg_encode_into with the layouts of ugb200_jpeg_encode_device_ex; a host I420 source is vc_get_datalen bytes */
UGB_API int ugb200_jpeg_encode_into_ex(ugb200_jpeg_encoder *enc, const void *src, int src_is_device, long pitch, int width, int height,
                                       int codec, const struct ugb200_jpeg_params_ex *params, uint8_t *dst, size_t dst_cap, size_t *out_size);

/* Measurement: with stage timing on, every encode records CUDA events between its kernels on the encoder's stream;
 * ugb200_jpeg_encoder_stage_times waits for the last encode and returns the device time in microseconds of
 * us[0] the DCT + entropy kernel (one-kernel form: the whole fused kernel; split path: the DCT + Huffman pair), us[1] the restart-segment
 * assembly kernel of the two-kernel form (0 otherwise), us[2] the offset scan, us[3] the compaction. */
UGB_API int ugb200_jpeg_encoder_stage_timing(ugb200_jpeg_encoder *enc, int enable);
UGB_API int ugb200_jpeg_encoder_stage_times(ugb200_jpeg_encoder *enc, float us[4]);

/* Stage access for tests: quantised zig-zag coefficients (int16[blocks][64], scan order) of the last encode, device ptr. */
UGB_API int ugb200_jpeg_debug_coefficients(ugb200_jpeg_encoder *enc, const int16_t **dev_ptr, size_t *count);

/* ---- decode (SURVEY.md section 8f rank 1): what src/video_decompress/gpujpeg.c:74-145,268-330 asks of libgpujpeg ---------------
 * Baseline sequential Huffman JPEG, 3 components, luma sampling 1x1 / 2x1 / 2x2, interleaved or one scan per component, restart
 * intervals (the unit of GPU parallelism), tables taken from the stream.  No colour transform inside the codec: a 4:2:2 / 4:2:0
 * YCbCr stream decodes to UYVY, a 4:4:4 RGB stream (Adobe transform 0) to RGB, a 4:4:4 YCbCr stream to VUYA; any other requested
 * output goes through UltraGrid's own line converters (ugb200_pixfmt_convert). */
typedef struct ugb200_jpeg_decoder ugb200_jpeg_decoder;
struct ugb200_jpeg_image_info {
        int width, height, components;
        int h_samp, v_samp;      /* sampling factors of component 0 */
        int adobe_transform;     /* APP14 transform flag, -1 without an Adobe marker */
        int restart_interval;
        int native_codec;        /* enum ugb200_codec the stream decodes to without conversion */
};
/* gpujpeg_decoder_get_image_info (gpujpeg.c:212): host only, reads the headers up to the first SOS */
UGB_API int ugb200_jpeg_get_image_info(const uint8_t *stream, size_t len, struct ugb200_jpeg_image_info *info);
/* host only, for tests: the restart segments the stream parser found ([begin, end) byte offsets of their entropy-coded data);
 * returns their number (may exceed cap) or a negative error */
UGB_API long ugb200_jpeg_debug_segments(const uint8_t *stream, size_t len, uint32_t *begin, uint32_t *end, long cap);
/* Where the restart segments are found: a stream of at least 1 MB with ONE scan that holds all components (UltraGrid's UYVY streams) or with one scan
 * per component in component order (RGB as GPUJPEG stores it, gpujpeg.cpp:303-305) has its RSTn markers located on the device (the host only reads the
 * header segments in front of the first SOS and copies the stream to pinned memory; for the second form the device also checks the later SOS headers
 * and hands an irregular stream back to the host parser); other streams are scanned by a few host threads.  UGB200_JPEG_MARKER_SCAN=host|device at
 * decoder creation forces one way (device: at any size).  The stream is uploaded on a copy stream of the decoder, under the kernels of the frame before.
 * ugb200_jpeg_decoder_last_segments returns the segment table of the last decode as the device holds it (waits for the decoder's stream). */
UGB_API long ugb200_jpeg_decoder_last_segments(ugb200_jpeg_decoder *dec, uint32_t *begin, uint32_t *end, long cap);
UGB_API ugb200_jpeg_decoder *ugb200_jpeg_decoder_create(cuda_wrapper_stream_t stream);   /* gpujpeg_decoder_create, gpujpeg.c:93 */
UGB_API void ugb200_jpeg_decoder_destroy(ugb200_jpeg_decoder *dec);                      /* gpujpeg_decoder_destroy */
/* The destination of ugb200_jpeg_decode is sized by the CALLER (video_desc of reconfigure(), gpujpeg.c:176-203) while the stream's SOF0
 * says how much is written: after this call a stream whose dimensions differ is refused with -3 before anything is decoded
 * (width = height = 0 switches the check off).  The decompress modules always set it. */
UGB_API int ugb200_jpeg_decoder_expect(ugb200_jpeg_decoder *dec, int width, int height);
/* gpujpeg_decoder_decode (gpujpeg.c:289,300): `stream` is a HOST buffer; dst is a host (synchronous) or device (asynchronous on the
 * decoder's stream) buffer of dst_pitch bytes per row (0 = vc_get_linesize); out_codec UGB_UYVY, UGB_RGB or UGB_RGBA (shifts).
 * 0 ok, -1 bad arguments, -2 CUDA failure, -3 malformed stream, -4 unsupported stream or output codec. */
UGB_API int ugb200_jpeg_decode(ugb200_jpeg_decoder *dec, const uint8_t *stream, size_t len, void *dst, int dst_is_device, long dst_pitch,
                               int out_codec, int rshift, int gshift, int bshift);

#ifdef __cplusplus
}
#endif
#endif
