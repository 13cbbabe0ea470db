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
 * (0 = src_pitch*height): some reference loops over-read a partial pixel group; reads past src_size give 0.  The plain copies
 * (in == out, and RGB -> RGB / RGBA -> RGBA with the default shifts 0, 8, 16) follow the same rule: nothing past src_size is read, and
 * the bytes of dst_len that would come from there are written as 0. */
UGB_API int ugb200_pixfmt_supported(int in_codec, int out_codec); /* get_decoder_from_to() != NULL */
UGB_API int ugb200_pixfmt_convert(int in_codec, int out_codec, void *dst, long dst_pitch, const void *src, long src_pitch,
                          int dst_len, int height, long src_size, int rshift, int gshift, int bshift,
                          cuda_wrapper_stream_t stream);

/* Colour space of the RGB <-> YCbCr converters: the values of UltraGrid's enum colorspace (src/color_space.h:129-133).  A binding passes
 * get_default_cs(), which is UGB_CS_601 under `--param color-601` and UGB_CS_709 otherwise. */
enum ugb200_colorspace {
        UGB_CS_DFL = 0,  /* BT.709, UltraGrid's default */
        UGB_CS_601 = 1,  /* BT.601 */
        UGB_CS_709 = 2,  /* BT.709 */
};
/* ugb200_pixfmt_convert with the Q14 coefficients of `cs` (get_color_coeffs(CS_DFL, depth) of an UltraGrid whose default colour space is `cs`)
 * in every converter whose reference body reads them; the others give the same bytes for every `cs`.  ugb200_pixfmt_convert is this with
 * UGB_CS_709.  A `cs` outside enum ugb200_colorspace returns -1 and writes nothing. */
UGB_API int ugb200_pixfmt_convert_cs(int in_codec, int out_codec, void *dst, long dst_pitch, const void *src, long src_pitch, int dst_len, int height,
                                     long src_size, int rshift, int gshift, int bshift, int cs, cuda_wrapper_stream_t stream);

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

/* ---- geometry filters (src/capture_filter/flip.c, mirror.c, src/vo_postprocess/crop.c, src/utils/vf_split.cpp,
 * src/vo_postprocess/border.c, 3d-interlaced.c) -------------------------------------------------------------------
 * The filters that move bytes without changing them (interlaced_3d averages two rows).  Stateless: the caller keeps
 * the module's options.  Frames are tight (vc_get_linesize pitch) unless a pitch is taken.  Every byte the reference
 * writes inside the output frame from bytes inside the sources gets the reference's value.  Differences (DESIGN.md
 * §8): nothing is written past the output frame, into the tails of split's tile rows or into pitch padding the
 * reference leaves alone; bytes the reference computes from memory past a source are left unwritten.
 * -1: a null pointer, width or height <= 0, dst overlapping a source, or the arguments under which the reference
 * asserts, crashes or writes outside the frame (noted per function).  -4: a codec the filter does not take.
 * Every refusal (-1, -4) writes nothing; -2 is a failed launch or scratch allocation. */
/* flip (flip.c:65-80): out row h-1-y = in row y, vc_get_linesize(width) bytes; any codec with a byte layout */
UGB_API int ugb200_cf_flip(int codec, int width, int height, const void *src, void *dst, cuda_wrapper_stream_t stream);
/* mirror (mirror.c:50-95): UYVY only (-4 otherwise, where the reference returns its input): group k of a row,
 * (U Y0 V Y1), lands at byte L - 4 - 4k as (U Y1 V Y0) */
UGB_API int ugb200_cf_mirror(int codec, int width, int height, const void *src, void *dst, cuda_wrapper_stream_t stream);
/* crop:[size=WxH][:width=W][:height=H][:xoff=X][:yoff=Y] (crop.c): out = {output width, output height, xoff, yoff}
 * exactly as crop_postprocess_reconfigure (:118-136) and crop_postprocess (:165-172) compute them: the width rounded
 * to whole pixel blocks in double arithmetic, the offsets compared in unsigned arithmetic (a negative offset is
 * clamped to in - out only when the sum wraps).  width / height 0 keep the input's.  -4: a codec without a pixel
 * block (opaque, planar or DXT). */
UGB_API int ugb200_cf_crop_geometry(int codec, int in_width, int in_height, int width, int height, int xoff, int yoff, int out[4]);
/* crop_postprocess (:160-185): out row y, at y * pitch, gets `pitch` bytes from source byte (yoff + y) * src_linesize
 * + xoff_bytes (xoff_bytes = xoff * bpp rounded down to whole blocks), reading on into the rest of the source row and
 * the next; bytes past the source frame are left unwritten.  pitch 0 is the capture filter's
 * vc_get_linesize(output width) (cf_crop_filter :214); the postprocessor passes the display's pitch.
 * An empty output frame (a window narrower than one pixel block) writes nothing and returns 0; dst may then be NULL.
 * -1 also: an unclamped negative offset that makes the first row start before the source. */
UGB_API int ugb200_cf_crop(int codec, int in_width, int in_height, int width, int height, int xoff, int yoff, const void *src,
                           void *dst, size_t pitch, cuda_wrapper_stream_t stream);
/* split:X:Y (split.c, vo_postprocess/split.c, vf_split.cpp:14-84): tiles[(line / tile_h) * x + i] row line % tile_h, at
 * vc_get_linesize(tile_w) pitch, gets (size_t) (tile_w * bpp) bytes from source row `line` at byte offset
 * `unsigned byte += tile_w * bpp` (truncated at every step); the rest of each tile row is left unwritten.  All
 * x * y tiles in one launch; the tile table goes to stream-ordered scratch.  -1 also: width % x or height % y != 0
 * (the reference asserts).  -4: a codec without a pixel block. */
UGB_API int ugb200_cf_split(int codec, int width, int height, int x, int y, const void *src, void *const *tiles,
                            cuda_wrapper_stream_t stream);
/* border[:color=rrggbb][:width=W][:height=H] (border.c:104-190): color = the module state's four RGBA bytes (as
 * border_init parses them), border_width / border_height as the state holds them.  Rows [bh, h - bh) are copied
 * outside the side bands, every other byte is the fill, each byte written once.  UYVY: the 4 bytes
 * vc_copylineRGBAtoUYVY makes from two pixels of the colour, over whole rows and over bytes [0, 4g) and [L - 4g, L)
 * of every row, g = (border_width + 1) / 2.  RGB / RGBA: color[b % bpp] over whole rows and border_width pixels on
 * each side.  -4: other codecs (the reference copies the middle rows, then fails).  -1 also: 2 * border_height >
 * height, or a side band wider than the row. */
UGB_API int ugb200_pp_border(int codec, int width, int height, const unsigned char color[4], unsigned border_width, unsigned border_height,
                             const void *src, void *dst, cuda_wrapper_stream_t stream);
/* interlaced_3d (3d-interlaced.c:131-167): left and right eye tiles -> one frame; out row x is written from byte
 * x * Lc, Lc = L rounded up to 16, in 16-byte chunks, chunk c = pavgb ((a + b + 1) >> 1) of bytes [16c, 16c + 16) of
 * rows x/2*2 and x/2*2+1 of tile x % 2 (L = vc_get_linesize(width)).  Rows drift when L % 16 != 0, as the
 * reference's do.  Bytes at or past L * height, and bytes whose sources lie past a tile (the last row at odd height
 * reads row `height` of the left tile), are not written. */
UGB_API int ugb200_pp_interlaced_3d(int codec, int width, int height, const void *left, const void *right, void *dst,
                                    cuda_wrapper_stream_t stream);

/* ---- logo and the R12L <-> Y416 pass-through filters (src/capture_filter/logo.c, r12l_to_y416_fake.c,
 * src/vo_postprocess/y416_to_r12l_fake.c) ----------------------------------------------------------------------------
 * Frames are tight (vc_get_linesize pitch) unless a pitch is taken.  Differences (DESIGN.md §8): logo widths whose
 * RGB segment the reference allocates too short are blended as the reference blends them with a long enough
 * segment; where the reference writes past a row or the frame, or asserts, the call returns -1.
 * -1: a null pointer or handle, a size <= 0, and the cases noted per function.  -4: a codec the filter does not
 * take.  Every refusal (-1, -4) writes nothing; -2 is a failed launch. */
/* logo:<file>[:<x>[:<y>]] (logo.c:162-235): the module state's logo, s->logo (RGBA; load_logo_data_from_file widens
 * 3-channel PAMs to alpha 0xFF), copied to the device; NULL when a size is 0 or the device allocation fails */
typedef struct ugb200_cf_logo *ugb200_cf_logo_t;
UGB_API ugb200_cf_logo_t ugb200_cf_logo_create(const unsigned char *rgba, unsigned width, unsigned height);
UGB_API void ugb200_cf_logo_destroy(ugb200_cf_logo_t logo);
/* filter() in place on a w x h logo over a width x height frame of RGB, RGBA, UYVY, RG48 or R12L (-4 otherwise, where
 * the reference returns its input).  x, y: the state's ints, -1 the default (bottom right).  rect_x = x, or width - w
 * when x < 0 or x + w > width, then C-truncated to a multiple of get_pf_block_bytes (bytes, counted in pixels);
 * rect_y = y, or height - h.  A negative rect_x or rect_y returns 0 and writes nothing.  Rows [rect_y, rect_y + h)
 * get bytes [off, off + vc_get_linesize(w)), off = vc_get_linesize(rect_x), and nothing else: the span is decoded
 * to RGB (the decoder_t of get_decoder_from_to(codec, RGB), default shifts), its first w pixels blended with the
 * logo as (p * (255 - a) + l * a) / 255 in int, and the span encoded back (get_decoder_from_to(RGB, codec)).  Every
 * pixel of the span makes the round trip: UYVY through A4 then A5, RG48 with its low bytes zeroed, RGBA with alpha
 * 0xFF and the decoder's SSSE3 tail (pixels [d - 4, d) of the row, d = w rounded up to 4, all take pixel d - 4's
 * colour before the blend), R12L through 8 bits.  -1 also: off + vc_get_linesize(w) > vc_get_linesize(width) (the
 * reference writes into the next row or past the frame), RG48 / R12L frames at an address not a multiple of 2 / 4. */
UGB_API int ugb200_cf_logo(ugb200_cf_logo_t logo, int codec, int width, int height, int x, int y, void *frame,
                           cuda_wrapper_stream_t stream);
/* r12l_to_y416_fake[:full-range] (r12l_to_y416_fake.c:85-191): tight R12L -> tight Y416, each pixel (R', G', B',
 * 0xFFFF) as uint16: full range c << 4; limited 14 * R + 4096, 13 * G + 4096, 14 * B + 4096.
 * -1 also: width % 8 != 0 (the reference asserts), src not 4-byte aligned, dst at an odd address, dst overlapping src. */
UGB_API int ugb200_cf_r12l_to_y416_fake(int width, int height, int full_range, const void *src, void *dst, cuda_wrapper_stream_t stream);
/* y416_to_r12l_fake[:full-range] (y416_to_r12l_fake.c:117-238): tight Y416 -> R12L rows at `pitch`, row y at
 * y * pitch (the reference's single-task layout, DESIGN.md §8), alpha dropped: full range min(v >> 4, 4095);
 * limited min((max(v, 4096) - 4096) / 14, 4095) for R and B, / 13 for G.  Pitch padding is not written.
 * -1 also: width % 8 != 0, pitch < vc_get_linesize(width, R12L), src at an odd address, dst not 4-byte aligned,
 * dst overlapping src. */
UGB_API int ugb200_pp_y416_to_r12l_fake(int width, int height, int full_range, const void *src, void *dst, size_t pitch,
                                        cuda_wrapper_stream_t stream);

/* ---- resize (src/capture_filter/resize.c; capture filter and, through its wrapper, postprocessor) ------------------
 * The resampling is not the reference's bytes (it runs in OpenCV): it follows the exact integer / float32 contract
 * of DESIGN.md §2 "Resize", modelled on OpenCV's generic path.  Everything resize.c itself decides (route, output
 * codec and size, letterbox) is the reference's.  Frames are tight (vc_get_linesize pitch; I420 as three planes).
 * The handle keeps the tables of the last input descriptor and, for codecs outside the resize set, a staging frame
 * in the route codec; calls on one handle must be ordered (one stream, or synchronised).  Every refusal writes
 * nothing. */
/* the module's struct resize_param values: mode 1 = fraction (factor), 2 = dimensions (tw, th); algo = cv::INTER_*
 * (0 nearest, 1 linear, 2 cubic, 3 area, 4 lanczos4) or -1 (RESIZE_ALGO_DFL: linear).  NULL on other values, a
 * factor that is not finite and > 0, or tw / th <= 0. */
typedef struct ugb200_cf_resize *ugb200_cf_resize_t;
UGB_API ugb200_cf_resize_t ugb200_cf_resize_create(int mode, double factor, int tw, int th, int algo);
/* The same parameters and NULL cases.  Its handles also resample with cubic, lanczos4, and area at ratios that are
 * not integer downscales (area upscaling included), each to the contract of DESIGN.md §2 "Resize"; nearest, linear
 * and integer area give the bytes of a ugb200_cf_resize_create handle.  -4 from them means only "no route". */
UGB_API ugb200_cf_resize_t ugb200_cf_resize_create2(int mode, double factor, int tw, int th, int algo);
UGB_API void ugb200_cf_resize_destroy(ugb200_cf_resize_t r);
/* out[0..7]: route codec (the input codec if in {RGB, RGBA, I420, UYVY, YUYV, RG48}, else get_best_decoder_from over
 * that set), out codec (RG48 for a 16-bit route, else RGB), out_w, out_h (fraction: (int) (w * factor); dimensions:
 * tw, th), the resampled rectangle x, y, w, h (resize_utils.cpp's letterbox; the whole frame in fraction mode).
 * Returns 0, -1 (null handle, size <= 0, an output or rectangle of size 0, an odd width on a UYVY / YUYV route, an
 * odd width or height on I420) or -4 (no route; on a ugb200_cf_resize_create handle also cubic, lanczos4, or area
 * at other than integer downscales). */
UGB_API int ugb200_cf_resize_geometry(ugb200_cf_resize_t r, int codec, int width, int height, int out[8]);
/* filter() of one tile into `dst` (vc_get_linesize(out_w, out codec) * out_h bytes, every one written: margins 0).
 * Codecs outside the resize set are first converted to the route codec (ugb200_pixfmt_convert) into the handle's
 * staging frame on `stream`.  0, -1 (also: null pointers, dst overlapping src), -2 (launch or device allocation
 * failure) or -4 as ugb200_cf_resize_geometry. */
UGB_API int ugb200_cf_resize(ugb200_cf_resize_t r, int codec, int width, int height, const void *src, void *dst,
                             cuda_wrapper_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif
