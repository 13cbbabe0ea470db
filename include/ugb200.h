/* Additions (H100-native, sm_90a) to the UltraGrid hot-path C ABI: fused / asynchronous block-compression entry
 * points, whole-buffer pixel-format conversion (device form of decoder_t line functions) and
 * packed->planar conversion.  Plain C, device pointers + sizes only.
 *
 * All functions here are ASYNCHRONOUS on `stream` (no implicit synchronisation) and return
 *   0 ok, -1 bad arguments / alignment, -2 launch failure, -4 unsupported conversion.
 */
#ifndef UGB200_H
#define UGB200_H

#include "cuda_wrapper.h"

#ifdef __cplusplus
extern "C" {
#endif

/* codec_t values — numerically identical to UltraGrid's enum (src/types.h:62-112) */
enum ugb200_codec {
        UGB_VIDEO_CODEC_NONE = 0,
        UGB_RGBA, UGB_UYVY, UGB_YUYV, UGB_VUYA, UGB_R10k, UGB_R12L, UGB_v210, UGB_DVS10, UGB_DXT1, UGB_DXT1_YUV,
        UGB_DXT5, UGB_RGB, UGB_JPEG, UGB_JPEG_XS, UGB_RAW, UGB_H264, UGB_H265, UGB_VP8, UGB_VP9, UGB_BGR, UGB_J2K,
        UGB_J2KR, UGB_HW_VDPAU, UGB_HFYU, UGB_FFV1, UGB_CFHD, UGB_RG48, UGB_AV1, UGB_I420, UGB_Y216, UGB_Y416,
        UGB_PRORES, UGB_PRORES_4444, UGB_PRORES_4444_XQ, UGB_PRORES_422_HQ, UGB_PRORES_422, UGB_PRORES_422_PROXY,
        UGB_PRORES_422_LT, UGB_APV, UGB_PYROWAVE, UGB_DRM_PRIME,
        UGB_VIDEO_CODEC_COUNT
};

/* ---- block compression (see cuda_dxt.h for the synchronous reference-compatible entry points) ---- */

/* same as cuda_{rgb,yuv}_to_dxt{1,6} (cuda_dxt/cuda_dxt.h:30-88) minus the cudaStreamSynchronize */
UGB_API int ugb200_rgb_to_dxt1_async(const void *src, void *out, int size_x, int size_y, cuda_wrapper_stream_t stream);
UGB_API int ugb200_yuv_to_dxt1_async(const void *src, void *out, int size_x, int size_y, cuda_wrapper_stream_t stream);
UGB_API int ugb200_rgb_to_dxt6_async(const void *src, void *out, int size_x, int size_y, cuda_wrapper_stream_t stream);
UGB_API int ugb200_yuv_to_dxt6_async(const void *src, void *out, int size_x, int size_y, cuda_wrapper_stream_t stream);

/* Fused UYVY -> DXT: replaces the pair cuda_yuv422_to_yuv444 + cuda_yuv_to_dxt{1,6} that
 * src/video_compress/cuda_dxt.cpp:223-257 runs (results are bit-identical to that pair).
 * src: device UYVY, 8-byte aligned (16 for the fast path); src_pitch bytes per row (0 = size_x*2);
 * size_x, size_y multiples of 4; negative size_y mirrors vertically. */
UGB_API int ugb200_uyvy_to_dxt1_async(const void *src, void *out, int size_x, int size_y, long src_pitch,
                              cuda_wrapper_stream_t stream);
UGB_API int ugb200_uyvy_to_dxt6_async(const void *src, void *out, int size_x, int size_y, long src_pitch,
                              cuda_wrapper_stream_t stream);

/* ---- pixel-format line converters over a whole buffer ---------------------------------------------
 * Device form of   for (y < height) decoder(dst + y*dst_pitch, src + y*src_pitch, dst_len, rs, gs, bs);
 * with decoder = get_decoder_from_to(in, out)  (src/pixfmt_conv.h:62-63, src/pixfmt_conv.c:3110-3125,
 * row loop as tools/convert.cpp:148-152).  Per-row results are byte-identical to the reference decoder,
 * including how many bytes of dst_len each loop really writes.  src_size = readable bytes from src
 * (0 = src_pitch*height): some reference loops over-read a partial pixel group; reads past src_size give 0. */
UGB_API int ugb200_pixfmt_supported(int in_codec, int out_codec); /* get_decoder_from_to() != NULL */
UGB_API int ugb200_pixfmt_convert(int in_codec, int out_codec, void *dst, long dst_pitch, const void *src, long src_pitch,
                          int dst_len, int height, long src_size, int rshift, int gshift, int bshift,
                          cuda_wrapper_stream_t stream);

/* Launch form of the line converters: -1 (default) = per converter, whichever measured faster at 8K (staged through shared memory with coalesced 16-byte
 * accesses, or one chunk per thread straight from / to global memory); 0 = never staged; 1 / 2 / 3 = input and output / output only / input only staged whenever pointers and pitches are 16-byte aligned.
 * The results are identical; the knob exists for the sweep (tools/pixfmt_sweep.py) and the tests.  Env UGB200_LINE_STAGED sets the initial value.
 * Returns the previous mode. */
UGB_API int ugb200_pixfmt_staged_mode(int mode);

/* The line converters pixfmt_conv.h exports OUTSIDE the decoders[] table (pixfmt_conv.h:93-101; callers: screen capture, DeckLink): same
 * whole-buffer form and return codes as ugb200_pixfmt_convert.  rshift/gshift/bshift are used by UGB_LINE_TO_RGBA_INPLACE only (SOURCE shifts). */
enum ugb200_line_func {
        UGB_LINE_ABGR_TO_RGB = 1,      /* vc_copylineABGRtoRGB, pixfmt_conv.c:809-843 */
        UGB_LINE_BGRA_TO_RGB,          /* vc_copylineBGRAtoRGB, :845-860 */
        UGB_LINE_TO_RGBA_INPLACE,      /* vc_copylineToRGBA_inplace, :907-921 (dst may equal src) */
        UGB_LINE_UYVY_TO_GRAYSCALE,    /* vc_copylineUYVYtoGrayscale, :927-938 */
};
UGB_API int ugb200_vc_copyline(int func, void *dst, long dst_pitch, const void *src, long src_pitch, int dst_len, int height, long src_size,
                               int rshift, int gshift, int bshift, cuda_wrapper_stream_t stream);

/* ---- block decoders (SURVEY.md section 8f rank 1) --------------------------------------------------- */
/* DXT5-YCoCg -> RGB exactly as the reference's CPU tool cuda_dxt/dxt62tga.c:24-108 (double arithmetic); DXT1 -> RGB by the same rule
 * for the colour block (+ the 3-colour mode).  src: device blocks in raster block order (what the encoders write), out: device, 3 B/px,
 * out_pitch bytes per row (0 = 3 * w); bgr != 0 swaps R and B (the TGA order of the tool).  w, h multiples of 4.  Asynchronous. */
UGB_API int ugb200_dxt1_to_rgb(const void *src, void *out, int w, int h, long out_pitch, int bgr, cuda_wrapper_stream_t stream);
UGB_API int ugb200_dxt5ycocg_to_rgb(const void *src, void *out, int w, int h, long out_pitch, int bgr, cuda_wrapper_stream_t stream);

/* ---- packed -> planar (src/to_planar.h:53-59) ----------------------------------------------------- */
struct ugb200_to_planar_data { /* same fields as struct to_planar_data; pointers are DEVICE pointers */
        int            width;
        int            height;
        unsigned char *out_data[4];
        unsigned       out_linesize[4];
        const unsigned char *in_data;
};
/* v210_to_p010le (src/to_planar.c:64-155). in_linesize 0 = vc_get_linesize(width, v210). */
UGB_API int ugb200_v210_to_p010le(const struct ugb200_to_planar_data *d, long in_linesize, cuda_wrapper_stream_t stream);
/* The other decode_buffer_func_t of src/to_planar.h:65-74, same names.  Input rows are vc_get_linesize(width, <in codec>) apart
 * (uyvy_to_nv12: width * 2, as to_planar.c:215).  Asynchronous on `stream`; 0 ok, -1 bad arguments, -2 launch failure. */
UGB_API int ugb200_y216_to_p010le(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t stream);   /* to_planar.c:164-200 */
UGB_API int ugb200_uyvy_to_nv12(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t stream);     /* :207-302 */
UGB_API int ugb200_rgba_to_bgra(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t stream);     /* :304-319 */
UGB_API int ugb200_vuya_to_i444(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t stream);     /* :321-337 */
UGB_API int ugb200_uyvy_to_i420(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t stream);     /* :343-378 */
UGB_API int ugb200_r12l_to_gbrp12le(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t stream); /* :381-481 */
UGB_API int ugb200_r12l_to_gbrp16le(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_r12l_to_rgbp12le(const struct ugb200_to_planar_data *d, cuda_wrapper_stream_t stream);

/* ---- planar -> packed (src/from_planar.h:58-70) ---------------------------------------------------- */
struct ugb200_from_planar_data { /* same fields as struct from_planar_data; pointers are DEVICE pointers */
        int            width;
        int            height;
        unsigned char *out_data;
        unsigned       out_pitch;
        const unsigned char *in_data[4];
        unsigned       in_linesize[4];
        int            in_depth;       /* the XX (generic) conversions */
        int            log2_chroma_h;  /* unused on the device (only decode_planar_parallel's row split needs it) */
        int            rgb_shift[3];   /* RGBA output only */
};
/* decode_planar_func_t of src/from_planar.h:88-115, same names.  Asynchronous on `stream`; 0 ok, -1 bad arguments, -2 launch failure. */
UGB_API int ugb200_gbrap_to_rgb(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);  /* from_planar.c:335-366 (8-bit planes G, B, R, A) */
UGB_API int ugb200_gbrap_to_rgba(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_gbrp10le_to_rgb(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);  /* :465-484, :521-563 (XX: in_depth; 8 = byte planes) */
UGB_API int ugb200_gbrp12le_to_rgb(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_gbrp16le_to_rgb(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_rgbpXX_to_rgb(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_gbrp10le_to_rgba(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);  /* :486-517 (rgb_shift[]) */
UGB_API int ugb200_gbrp12le_to_rgba(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_gbrp16le_to_rgba(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_gbrp10le_to_rg48(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);  /* :157-201 */
UGB_API int ugb200_gbrp12le_to_rg48(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_gbrp16le_to_rg48(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_rgbpXXle_to_rg48(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_gbrp10le_to_r10k(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);  /* :203-250 */
UGB_API int ugb200_gbrp12le_to_r10k(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_gbrp16le_to_r10k(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_rgbpXXle_to_r10k(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_gbrp12le_to_r12l(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);  /* :61-155 */
UGB_API int ugb200_gbrp16le_to_r12l(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_rgbpXXle_to_r12l(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_yuv444p_to_vuya(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);  /* :565-580 */
UGB_API int ugb200_yuv420p_to_uyvy(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);  /* :582-683 */
UGB_API int ugb200_yuv420_to_i420(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);  /* :368-390 (out = contiguous I420, out_pitch ignored) */
UGB_API int ugb200_yuv422p_to_uyvy(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);  /* :392-463 */
UGB_API int ugb200_yuv422p_to_yuyv(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_yuv422pXX_to_uyvy(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_yuv422p10le_to_uyvy(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);
UGB_API int ugb200_yuv422p10le_to_v210(const struct ugb200_from_planar_data *d, cuda_wrapper_stream_t stream);  /* :295-333 (whole 6-pixel groups) */

/* ---- interlaced video (src/video_codec.c, src/video_frame.c) ------------------------------------------ */
/* vc_deinterlace_ex (video_codec.c:722-854): linear blend, out row y = (row y + row y+1 + 1) >> 1 per sample, then
 * row lines-1 = out row lines-2 (src_linesize bytes).  Byte-exact on every byte the reference writes, in place
 * (dst == src, dst_pitch == src_linesize) or out of place.  Differences (DESIGN.md §8): 16-bit codecs blend the
 * whole row and R12L every whole 36-byte group, where the reference leaves the row's tail unwritten; opaque
 * codecs are refused with -4.  lines == 1 copies the row for every non-opaque codec, as the reference does.
 * -1: lines == 0, dst_pitch < src_linesize, partial overlap, or a 16-bit (word) codec at an address or pitch that
 * is not a multiple of 2 (4).  -4: opaque codec, or DVS10 with lines > 1. */
UGB_API int ugb200_vc_deinterlace_ex(int codec, const void *src, size_t src_linesize, void *dst, size_t dst_pitch, size_t lines,
                                     cuda_wrapper_stream_t stream);
/* vc_deinterlace (video_codec.c:597-711, the SSE2 form an x86-64 build runs): in-place recursive filter, any buffer
 * address, byte-exact for linesize >= 16 (-1 below), including the last 16-byte column's re-filter of the next row's
 * first bytes.  lines <= 4 leaves the buffer as it is. */
UGB_API int ugb200_vc_deinterlace(void *buf, long linesize, int lines, cuda_wrapper_stream_t stream);
/* il_upper_to_merged / il_merged_to_upper (video_frame.c:332-379): (height+1)/2 upper-field rows then height/2
 * lower-field rows <-> interleaved rows.  dst == src works (stream-ordered scratch, no host wait); partial overlap
 * is -1. */
UGB_API int ugb200_il_upper_to_merged(void *dst, void *src, int linesize, int height, cuda_wrapper_stream_t stream);
UGB_API int ugb200_il_merged_to_upper(void *dst, void *src, int linesize, int height, cuda_wrapper_stream_t stream);

/* ---- field-rate postprocessors (src/vo_postprocess/temporal-deint.c, src/vo_postprocess/interlace.c) -------- */
/* Stateless: the caller keeps the two frame buffers, as common_getf does.  `call` 0 is the module's postprocess(in =
 * frame) and 1 the follow-up postprocess(in = NULL); `cur` is the merged frame just received, `prev` the one before.
 * Rows [0, height) of dst get the reference's bytes [0, linesize) and nothing else is written or read, except where
 * noted.  Differences (DESIGN.md §8): nothing past linesize (the reference rounds 8/16-bit rows up to 16 bytes and
 * writes 4 x linesize for R10k) nor row `height` (double_framerate at odd height) is touched; height < 2 is -1;
 * opaque codecs are -4 for linear and :d.
 * -1: a null pointer, height < 2, linesize == 0, pitch < linesize, call not 0 / 1, dst overlapping a source, or a
 * 16-bit (word) codec whose addresses, linesize or pitch are not multiples of 2 (4) where the codec matters.
 * Every refusal (-1, -4) writes nothing; -2 (a CUDA launch or scratch allocation failed) can leave dst partly written. */
/* double_framerate (temporal-deint.c:240-277): call 0 = cur's even rows and prev's odd rows (at odd height row
 * height-1 stays as it is), call 1 = cur.  deinterlace != 0 is `:d`: then vc_deinterlace_ex in place at pitch linesize,
 * as ugb200_vc_deinterlace_ex computes it (-4 where that refuses); at pitch == linesize weave and blend are one pass,
 * otherwise the first linesize * height bytes of dst are blended as the reference blends them. */
UGB_API int ugb200_pp_double_framerate(int codec, const void *prev, const void *cur, size_t linesize, int height, int call,
                                       int deinterlace, void *dst, size_t pitch, cuda_wrapper_stream_t stream);
/* deinterlace_bob (:279-300): call 0 doubles rows 0, 2, ...; call 1 writes row 1 to rows 0-2, then doubles 3, 5, ...;
 * a left-over last row repeats the row above it */
UGB_API int ugb200_pp_bob(const void *cur, size_t linesize, int height, int call, void *dst, size_t pitch, cuda_wrapper_stream_t stream);
/* deinterlace_linear (:442-466, avg_lines :307-440): rows of the call's parity are copied, the row between two of
 * them is avg_lines of the two, the last row(s) repeat the last copied row.  avg_lines as the reference computes
 * it: 8/16-bit c1/2 + c2/2 + (c1 & 1), v210 whole 16-byte groups, R10k byte-swapped with bits 0-1 zero, R12L
 * over linesize/16 groups of 4 words with the last word dropped unless 3 divides linesize/16; DVS10 copies */
UGB_API int ugb200_pp_linear(int codec, const void *cur, size_t linesize, int height, int call, void *dst, size_t pitch,
                             cuda_wrapper_stream_t stream);
/* interlace (interlace.c:159-190): out row i = row i of even_rows (the module's s->odd) for even i, of odd_rows
 * (s->even) for odd i */
UGB_API int ugb200_pp_interlace(const void *even_rows, const void *odd_rows, size_t linesize, int height, void *dst, size_t pitch,
                                cuda_wrapper_stream_t stream);

/* ---- colour capture filters (src/capture_filter/gamma.cpp, matrix.c, matrix2.c, grayscale.c) -------------------- */
/* The filters' filter() on device frames; each is also a postprocessor through ADD_VO_PP_CAPTURE_FILTER_WRAPPER.
 * Frames are tight (vc_get_linesize pitch, which the vo_pp wrapper insists on); input and output lengths follow
 * from codec, width and height as vf_alloc_desc derives them.  Every double -> integer conversion is x86's
 * cvttsd2si with a 32-bit destination (truncation, INT_MIN for NaN and out-of-range values), then the low 8 or 16
 * bits; FP64 sums run left to right without FMA.  Differences (DESIGN.md §8): gamma maps every sample (the
 * reference skips the last len % hardware_concurrency() ones); nothing is written past the output frame (matrix
 * UYVY at odd widths stops at 3 * w * h, matrix2 v210 at the frame's length); matrix2 on v210 maps every 16-byte
 * group of the frame, including those >= w * h / 6 whose reference bytes are indeterminate.
 * -1: a null pointer or handle, width or height <= 0, out_depth not 0 / 8 / 16, dst overlapping src, or a 16-bit
 * buffer at an odd address (v210: not a multiple of 4).  -4: a codec the filter does not take (the reference
 * returns NULL for gamma and matrix, its input for grayscale, and a frame of uninitialised memory for matrix2).
 * Every refusal (-1, -4) writes nothing; -2 is a failed launch. */

/* gamma:g[:8|:16] (gamma.cpp): the four tables pow(i / max_in, g) * max_out (8->8, 16->16, 8->16, 16->8), built
 * on the host with the C library's pow at create; NULL when the device allocation fails */
typedef struct ugb200_cf_gamma *ugb200_cf_gamma_t;
UGB_API ugb200_cf_gamma_t ugb200_cf_gamma_create(double gamma);
UGB_API void ugb200_cf_gamma_destroy(ugb200_cf_gamma_t g);
/* codec RGB or RG48; out_depth 0 keeps the depth, 8 writes RGB, 16 RG48 */
UGB_API int ugb200_cf_gamma(ugb200_cf_gamma_t g, int codec, int out_depth, int width, int height, const void *src, void *dst,
                            cuda_wrapper_stream_t stream);
/* matrix:a:...:i[:no-bound-check] (matrix.c): UYVY -> RGB (U Y0 V Y1 -> (Y0-16, U-128, V-128), (Y1-16, ...)),
 * RGB -> RGB, RG48 -> RG48; out = (m0*a0 + m1*a1) + m2*a2 per row.  check_bounds != 0 clamps the int32 to
 * [0, 255], RG48 included; 0 keeps its low bits.  UYVY at odd widths drifts across rows as the reference does. */
UGB_API int ugb200_cf_matrix(int codec, int width, int height, const double m[9], int check_bounds, const void *src, void *dst,
                             cuda_wrapper_stream_t stream);
/* matrix2:a:...:i or matrix2:y601_to_y709 (matrix2.c): YCbCr in place of its own codec, no clamping.
 * UYVY: Y' = ((16 + m0*y) + m1*u) + m2*v, U' / V' the same with offset 128 and y = (y1 + y2) / 2.
 * Y416: offsets 1<<12 / 1<<15 per pixel, A = 0xFFFF.  v210: the 16-byte group x of the frame -> 6 Y416 pixels
 * (vc_copylineV210toY416) -> the Y416 matrix -> vc_copylineY416toV210 (pair-averaged chroma, >> 6) -> group x. */
UGB_API int ugb200_cf_matrix2(int codec, int width, int height, const double m[9], const void *src, void *dst,
                              cuda_wrapper_stream_t stream);
/* matrix2.c's y601_y709_matrix, the coefficients of `matrix2:y601_to_y709` */
#define UGB200_CF_Y601_TO_Y709 { 1, -0.11555, -0.207938, 0, 1.01864, 0.114618, 0, 0.075049, 1.025327 }
/* grayscale (grayscale.c): UYVY, chroma bytes 127 and luma copied over the first 2 * w * h bytes; at odd widths
 * the last 2 * h bytes of the frame are left as they are, as the reference leaves them */
UGB_API int ugb200_cf_grayscale(int width, int height, const void *src, void *dst, cuda_wrapper_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif
