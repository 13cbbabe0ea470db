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
 *   UGB_RGBA input, subsampling 4444, colour space NATIVE or RGB (the GPUJPEG module's `alpha`: GPUJPEG_SUBSAMPLING_4444 with
 *                                               GPUJPEG_4444_U8_P0123, gpujpeg.cpp:227-236,316-328) -> R, G, B, A stored as-is, the frame read in
 *                                               place at 4 B/px: Adobe APP14 transform 0, SOF0 with four components (ids 1..4, all 1x1,
 *                                               quantisation and Huffman tables 0 1 1 1 - GPUJPEG's own choice for alpha is unpinned, the library
 *                                               being absent), four scans (one per component, gpujpeg.cpp:303) or one scan of R G B A MCUs with
 *                                               `interleaved`, restart interval default 8.  The first three scans are byte for byte the scans of
 *                                               the RGB stream of the frame's R, G, B bytes; the fourth is coded like the third (table 1).
 *   every YCbCr stream carries JFIF APP0; restart interval default 8 for RGB and RGBA input, 4 otherwise.  Native parameters give the bytes
 *   of the calls without _ex.  Anything else returns -4: chroma upsampling, YCbCr -> RGB, one YCbCr matrix -> another, subsampled RGB, RGBA
 *   without subsampling 4444 or with a YCbCr colour space, and RGBA through ugb200_jpeg_encode_device / _encode / _encode_into.
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
enum { UGB200_JPEG_CS_NATIVE = 0, UGB200_JPEG_CS_Y601, UGB200_JPEG_CS_Y601FULL, UGB200_JPEG_CS_Y709, UGB200_JPEG_CS_RGB,  /* = gpujpeg_opts::internal_cs */
       UGB200_JPEG_CS_AUTO = 5 /* decode only: the colour space the stream declares (ugb200_jpeg_stream_color_space) */ };
struct ugb200_jpeg_params_ex {
        struct ugb200_jpeg_params base;
        int subsampling;   /* 0 = native for the input (RGB 444, UYVY 422, I420 420), else 444 / 422 / 420 */
        int color_space;   /* UGB200_JPEG_CS_* */
};
UGB_API void ugb200_jpeg_default_params_ex(struct ugb200_jpeg_params_ex *p);
/* ugb200_jpeg_encode_device with the layouts above; `codec` also takes UGB_I420 (pitch must be 0) and UGB_RGBA (subsampling 4444) */
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
 * us[0] the DCT + entropy kernel (fused path: the whole fused kernel; split path: the DCT + Huffman pair), us[1] always 0 (it was the
 * restart-segment assembly kernel of a retired two-kernel form; the slot keeps the layout), us[2] the offset scan, us[3] the compaction. */
UGB_API int ugb200_jpeg_encoder_stage_timing(ugb200_jpeg_encoder *enc, int enable);
UGB_API int ugb200_jpeg_encoder_stage_times(ugb200_jpeg_encoder *enc, float us[4]);

/* Stage access for tests: quantised zig-zag coefficients (int16[blocks][64], scan order) of the last encode, device ptr. */
UGB_API int ugb200_jpeg_debug_coefficients(ugb200_jpeg_encoder *enc, const int16_t **dev_ptr, size_t *count);

/* ---- decode (SURVEY.md section 8f rank 1): what src/video_decompress/gpujpeg.c:74-145,268-330 asks of libgpujpeg ---------------
 * Baseline sequential Huffman JPEG, 3 components (or 1, below), luma sampling 1x1 / 2x1 / 2x2, interleaved or one scan per component, restart
 * intervals (the unit of GPU parallelism), tables taken from the stream.  No colour transform inside the codec: a 4:2:2 / 4:2:0
 * YCbCr stream decodes to UYVY, a 4:4:4 RGB stream (Adobe transform 0) to RGB, a 4:4:4 YCbCr stream to VUYA; any other requested
 * output goes through UltraGrid's own line converters (ugb200_pixfmt_convert).
 * Also 4 components, all sampled 1x1, without an Adobe marker or with Adobe transform 0 (the GPUJPEG module's `alpha` stream): native
 * codec UGB_RGBA, samples as stored.  To RGBA with shifts (0, 8, 16): R G B A, alpha in byte 3, at any pitch; with other shifts that
 * result re-shifted by the RGBA -> RGBA line converter (vc_copylineRGBA: the unused byte becomes 0xFF).  To any other codec: the first three
 * planes as an RGB stream decodes.  Four-component streams with Adobe transform 1 or 2 (YCCK) or subsampled components return -4.
 * Also 1 component (grayscale: IR and machine-vision cameras, libavcodec's `gray` MJPEG), one scan with or without DRI; the sampling factors are
 * ignored (T.81 A.2.2).  ugb200_jpeg_get_image_info reports components 1, h_samp = v_samp = 1, native codec UGB_UYVY.  ugb200_jpeg_decode_to decodes
 * it as a YCbCr stream with Cb = Cr = 128 everywhere: UYVY `128 Y 128 Y`, I420 with 128-filled chroma planes, RGB / RGBA by the formula of
 * stream_cs (Y601FULL gives R = G = B = Y; NATIVE: the BT.709 line converters).  VUYA output of a grayscale stream returns -4, as of every stream whose
 * native codec is UYVY (there is no UYVY -> VUYA line converter).  ugb200_jpeg_decode and ugb200_jpeg_decode_cs refuse it with -4,
 * as they always have. */
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
/* Huffman decoding.  A restart segment of fewer than 64 MCUs is decoded by one GPU thread.  Longer segments - every scan of a stream without DRI (RTSP
 * cameras, webcam MJPEG, libjpeg's defaults) - take a self-synchronising route: the segment's bytes are cut into subsequences of 64 bytes, one thread
 * each; every thread decodes from a guessed state until its exit state (bit position, block of the MCU, zig-zag position at the first symbol boundary
 * behind the next subsequence's start) stops changing from round to round, which proves every start state; a prefix sum of block counts and DC
 * differences then places the blocks.  Both routes give the same coefficients for any bytes, damaged ones included (DESIGN.md section 2).
 * ugb200_jpeg_decoder_last_sync reports what the last decode did (waits for the decoder's stream): the scans that took the self-synchronising route
 * (0: none), its subsequences over all segments and its rounds.  Test hook, read at decoder creation: UGB200_JPEG_SYNC=off forces one thread per
 * segment, UGB200_JPEG_SYNC=on[:<bytes>] forces the self-synchronising route for every stream, optionally with another subsequence length. */
struct ugb200_jpeg_sync_stats {
        int scans;           /* scans of the last decode that took the self-synchronising route */
        int rounds;          /* synchronisation rounds (1: every guessed start state was right at once) */
        long subsequences;   /* subsequences over all restart segments of those scans */
};
UGB_API int ugb200_jpeg_decoder_last_sync(ugb200_jpeg_decoder *dec, struct ugb200_jpeg_sync_stats *st);
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

/* Decode in a colour space.  ugb200_jpeg_decode writes the stream's samples (no colour transform in the codec); its RGB and RGBA output of a YCbCr
 * stream is that of UltraGrid's line converters, which take every stream as BT.709 limited range.  A JFIF stream (libjpeg, PIL, webcams) holds
 * full-range BT.601 (T.871), so its colours come out wrong that way.
 *
 * ugb200_jpeg_stream_color_space (host only) returns the colour space the stream declares, or < 0 (-1 bad arguments, -3 malformed, -4 unsupported):
 *   RGB and RGBA streams (Adobe transform 0, component ids 'R' 'G' 'B', four components) -> UGB200_JPEG_CS_RGB, whatever else they carry;
 *   else a SPIFF APP8: colour space 1 -> Y709, 4 -> Y601, 3 -> Y601FULL, 10 -> RGB, any other code -> -4, a segment too short for the field -> -3;
 *   else Adobe APP14 transform 1 -> Y601FULL; else JFIF APP0 -> Y601FULL; else (no marker) -> Y709, what UltraGrid assumes for unmarked streams.
 *   A one-component stream never resolves to RGB: SPIFF colour space 8 (grayscale) -> Y601FULL, as UltraGrid's reader takes it
 *   (src/utils/jpeg_reader.c:682-685), SPIFF 10 -> -4, everything else as above.
 *
 * ugb200_jpeg_decode_cs is ugb200_jpeg_decode, except that RGB and RGBA output of a YCbCr stream is converted from `color_space`:
 *   UGB200_JPEG_CS_NATIVE: the bytes of ugb200_jpeg_decode.
 *   UGB200_JPEG_CS_Y709 | _Y601 | _Y601FULL: what the stream's YCbCr holds.  R = clamp((y_scale * (Y - o) + r_cr * (Cr - 128)) >> 14, 0, 255), G and B
 *     likewise (UltraGrid's YCBCR_TO_R/G/B) with the coefficients coeffs_709(8), coeffs_601(8), coeffs_601(0) of UltraGrid's color_space.c, o = 16,
 *     16, 0, and >> a floor.  Chroma is replicated from its pixel pair (4:2:2) or quad (4:2:0) unless the decoder interpolates it
 *     (ugb200_jpeg_decoder_set_upsampling).  RGBA places R, G and B at the
 *     shifts and sets every other bit (alpha 0xFF).  Y709 RGB output of a 4:2:2 or 4:2:0 stream is the RGB of ugb200_jpeg_decode byte for byte.
 *   UGB200_JPEG_CS_AUTO: as ugb200_jpeg_stream_color_space resolves it; a stream that declares RGB is not transformed, a refusal is returned.
 * RGB and four-component streams, and UYVY, I420 and VUYA output, keep the stream's samples in every mode (ugb200_jpeg_decode_to converts those).
 * As in ugb200_jpeg_decode, RGB and RGBA rows of a 4:2:2 / 4:2:0 stream of odd width get whole pixel pairs only (DESIGN.md section 8).
 * Any other color_space returns -1.  On every error the output buffer is not touched.
 * Known limitation: this library's encoder writes JFIF APP0 on its UYVY and I420 streams although they hold BT.709 limited-range samples, so
 * AUTO reads them as Y601FULL; callers that decode this encoder's streams pass Y709 or NATIVE. */
UGB_API int ugb200_jpeg_stream_color_space(const uint8_t *stream, size_t len);
UGB_API int ugb200_jpeg_decode_cs(ugb200_jpeg_decoder *dec, const uint8_t *stream, size_t len, void *dst, int dst_is_device, long dst_pitch,
                                  int out_codec, int rshift, int gshift, int bshift, int color_space);

/* Decode to a colour space.  UltraGrid's receiver asks libgpujpeg for BT.709 limited-range UYVY / I420 whatever the stream holds
 * (src/video_decompress/gpujpeg.c:103-138); a camera's JFIF stream holds full-range BT.601, so its samples have to be converted, not only packed.
 *   stream_cs: as color_space of ugb200_jpeg_decode_cs (NATIVE, Y709, Y601, Y601FULL, AUTO).
 *   out_cs:    NATIVE, Y709, Y601 or Y601FULL - the space that YCbCr output (UYVY, I420, VUYA) shall hold.  Anything else returns -1.
 * RGB / RGBA output: exactly ugb200_jpeg_decode_cs(..., stream_cs); out_cs is ignored.
 * YCbCr output of a YCbCr (or grayscale) stream: when stream_cs or out_cs is NATIVE, or both resolve to the same space, the bytes of
 * ugb200_jpeg_decode.  Otherwise every decoded sample is converted at the stream's own sampling (nothing is resampled) and then packed as
 * ugb200_jpeg_decode packs that sampling for that output codec - "convert, then pack":
 *   Y'  = clamp(((m_yy * (Y - o_in) + m_yb * (Cb - 128) + m_yr * (Cr - 128) + 8192) >> 14) + o_out, 0, 255)   per luma sample, with the chroma
 *                                                                                                             of its pair (4:2:2) or quad (4:2:0)
 *   Cb' = clamp(((m_bb * (Cb - 128) + m_br * (Cr - 128) + 8192) >> 14) + 128, 0, 255)                          per chroma sample
 *   Cr' = clamp(((m_rb * (Cb - 128) + m_rr * (Cr - 128) + 8192) >> 14) + 128, 0, 255)                          per chroma sample
 * with o = 16 for Y709 and Y601, 0 for Y601FULL, `>>` a floor, and the seven coefficients round(2^14 * M), M = (RGB -> YCbCr of out_cs) *
 * (YCbCr -> RGB of stream_cs) formed in double from the kr, kb and range scales of UltraGrid's color_space.c and rounded once
 * (compute_ycc_matrix, csrc/color_space.h).  Chroma of the target does not depend on luma of the source, which makes the conversion exact at
 * 4:2:2 and 4:2:0.  A grayscale stream takes the luma line alone (the chroma terms vanish).  The clamp is 0..255: UltraGrid's CLAMP_LIMITED_* are
 * identities (color_space.h:93-94); libgpujpeg's own rounding is unpinned, the library being absent.  Each result lies within 1 of the unrounded
 * matrix product (tests/test_jpeg_decode_yuv.py derives and checks the bound over every triple).
 * YCbCr output of an RGB or four-component stream (or one that declares RGB under AUTO, which is never matrixed): out_cs NATIVE or Y709 give the
 * bytes of ugb200_jpeg_decode (UltraGrid's line converters are BT.709); Y601 and Y601FULL return -4.
 * Errors as ugb200_jpeg_decode_cs; on every error the output buffer is not touched. */
UGB_API int ugb200_jpeg_decode_to(ugb200_jpeg_decoder *dec, const uint8_t *stream, size_t len, void *dst, int dst_is_device, long dst_pitch,
                                  int out_codec, int rshift, int gshift, int bshift, int stream_cs, int out_cs);

/* Chroma upsampling of RGB and RGBA output in a colour space.  REPLICATE (the default) gives every pixel the chroma of its pair or quad, as above.
 * FANCY interpolates it as libjpeg-turbo (and so every libjpeg- or ffmpeg-based viewer) does, so that saturated edges show no 2-pixel colour steps.
 * FANCY changes only RGB and RGBA output of a 4:2:2 or 4:2:0 YCbCr stream from ugb200_jpeg_decode_cs and ugb200_jpeg_decode_to, and only when the
 * colour space is Y709, Y601 or Y601FULL, or AUTO resolving to one of them.  For those outputs:
 *   1. Each chroma plane (Cb, Cr) is upsampled to full resolution with integers and `>>` a floor.  The plane has cw = ceil(w / 2) columns and
 *      ch = h rows (4:2:2) or ceil(h / 2) rows (4:2:0); a neighbour outside [0, cw - 1] x [0, ch - 1] takes the value of the nearest edge sample, so
 *      the padded block area beyond cw / ch is never read.
 *        4:2:2, chroma sample c[x] of a row:  out[2x] = (3 c[x] + c[x-1] + 1) >> 2,  out[2x+1] = (3 c[x] + c[x+1] + 2) >> 2
 *        4:2:0, chroma rows c (this row) and n (the row above for output row 2y, the row below for 2y + 1), s[x] = 3 c[x] + n[x]:
 *                                             out[2x] = (3 s[x] + s[x-1] + 8) >> 4,  out[2x+1] = (3 s[x] + s[x+1] + 7) >> 4
 *      When cw <= 2 the chroma is replicated instead, in both directions, as libjpeg-turbo does for planes that narrow (jdsample.c).  Output
 *      columns and rows past w / h are dropped.
 *   2. Every pixel then gets YCBCR_TO_R/G/B of ugb200_jpeg_decode_cs with its own luma and its own upsampled Cb, Cr, clamped 0..255; RGBA as there.
 *   3. Every pixel of every row is written, w * 3 or w * 4 bytes and nothing beyond - the last pixel of an odd width included, which REPLICATE
 *      leaves unwritten.
 * Byte for byte the same under FANCY as under REPLICATE: ugb200_jpeg_decode, colour space NATIVE, UYVY / I420 / VUYA output, 4:4:4, grayscale, RGB
 * and four-component streams, AUTO resolving to RGB, and every refusal.  The filter and its edge rule equal libjpeg-turbo's YCbCr output sample for
 * sample (tests/test_jpeg_decode_fancy.py).
 * mode applies to every later decode call on this decoder.  0 ok, -1 bad arguments (NULL decoder, unknown mode). */
enum { UGB200_JPEG_UPSAMPLE_REPLICATE = 0, UGB200_JPEG_UPSAMPLE_FANCY = 1 };
UGB_API int ugb200_jpeg_decoder_set_upsampling(ugb200_jpeg_decoder *dec, int mode);

#ifdef __cplusplus
}
#endif
#endif
