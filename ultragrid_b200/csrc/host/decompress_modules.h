// The three decompress modules of this library (gpujpeg, gpujpeg_to_dxt, dxt_cuda), written once against the type and function NAMES that UltraGrid's
// headers and the mirror headers of this directory share (codec_t, struct video_desc, struct pixfmt_desc, decompress_status, video_decompress_info,
// REGISTER_MODULE, cuda_devices, vc_get_linesize).  Included by
//   host/video_decompress.cpp            mirror types (host/ug_types.h): part of libugb200.so, used by the Python driver and bench
//   module/ug_decompress_module.cpp      the reference's REAL headers (-I$(REF)/src): ultragrid_b200/modules/ultragrid_vdecompress_*.so, what an
//                                        unmodified UltraGrid dlopen()s (src/video_decompress.c:100-230 selects them by priority)
// UGB_DECOMPRESS_MODULES selects which modules a translation unit registers: bit 0 gpujpeg, bit 1 gpujpeg_to_dxt, bit 2 dxt_cuda (default: all).
// Everything CUDA happens behind the C ABI of libugb200.so (include/*.h).
#pragma once
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "../../../include/cuda_dxt.h"
#include "../../../include/cuda_wrapper.h"
#include "../../../include/ugb200.h"
#include "../../../include/ugb200_jpeg.h"

#ifndef UGB_DECOMPRESS_MODULES
#define UGB_DECOMPRESS_MODULES 7
#endif
static int no_corrupted_frames(void *, int property, void *val, size_t *len)  // gpujpeg.c:325-343 and the others alike
{
        if (property == DECOMPRESS_PROPERTY_ACCEPTS_CORRUPTED_FRAME && *len >= sizeof(int)) {
                *(int *) val = 0, *len = sizeof(int);
                return 1;
        }
        return 0;
}
/// The colour space the JPEG modules take a stream's YCbCr to be, read when a module instance is created: UGB200_JPEG_DECODE_CS=auto|y709|y601|y601full
/// makes gpujpeg and gpujpeg_to_dxt ask for BT.709 output converted from that space (what gpujpeg.c:81,103-138 asks of libgpujpeg: GPUJPEG_YCBCR_BT709
/// for UYVY / I420, RGB converted from the stream's space).  Unset (NATIVE): the stream's samples as they are, the bytes of ugb200_jpeg_decode - this
/// library's encoder labels its BT.709 streams with JFIF APP0, which `auto` would read as full-range BT.601.
static int jpeg_decode_cs_from_env()
{
        const char *e = getenv("UGB200_JPEG_DECODE_CS");
        if (e == nullptr || e[0] == 0) {
                return UGB200_JPEG_CS_NATIVE;
        }
        if (strcmp(e, "auto") == 0) {
                return UGB200_JPEG_CS_AUTO;
        }
        if (strcmp(e, "y709") == 0) {
                return UGB200_JPEG_CS_Y709;
        }
        if (strcmp(e, "y601") == 0) {
                return UGB200_JPEG_CS_Y601;
        }
        if (strcmp(e, "y601full") == 0) {
                return UGB200_JPEG_CS_Y601FULL;
        }
        fprintf(stderr, "[GPUJPEG dec.] UGB200_JPEG_DECODE_CS=%s is not one of auto, y709, y601, y601full: ignored\n", e);
        return UGB200_JPEG_CS_NATIVE;
}
/// The chroma upsampling of the JPEG modules' RGB / RGBA output, read when a module instance is created next to UGB200_JPEG_DECODE_CS:
/// UGB200_JPEG_DECODE_UPSAMPLE=fancy|replicate (ugb200_jpeg_decoder_set_upsampling).  It acts only together with a colour space, because FANCY changes
/// nothing of the native bytes; unset, the chroma is replicated as before.
static int jpeg_decode_upsample_from_env(int stream_cs)
{
        const char *e = getenv("UGB200_JPEG_DECODE_UPSAMPLE");
        if (e == nullptr || e[0] == 0) {
                return UGB200_JPEG_UPSAMPLE_REPLICATE;
        }
        int mode;
        if (strcmp(e, "fancy") == 0) {
                mode = UGB200_JPEG_UPSAMPLE_FANCY;
        } else if (strcmp(e, "replicate") == 0) {
                mode = UGB200_JPEG_UPSAMPLE_REPLICATE;
        } else {
                fprintf(stderr, "[GPUJPEG dec.] UGB200_JPEG_DECODE_UPSAMPLE=%s is not one of fancy, replicate: ignored\n", e);
                return UGB200_JPEG_UPSAMPLE_REPLICATE;
        }
        if (stream_cs == UGB200_JPEG_CS_NATIVE) {
                fprintf(stderr, "[GPUJPEG dec.] note: UGB200_JPEG_DECODE_UPSAMPLE=%s has an effect only together with UGB200_JPEG_DECODE_CS\n", e);
        }
        return mode;
}
/// ugb200_jpeg_decode_to with the module's colour space: NATIVE gives the bytes of ugb200_jpeg_decode (and decodes grayscale streams, which that call refuses)
static int jpeg_module_decode(ugb200_jpeg_decoder *dec, int stream_cs, const unsigned char *buffer, size_t len, void *dst, int dst_is_device, long pitch, int out_codec,
                              int rshift, int gshift, int bshift)
{
        return ugb200_jpeg_decode_to(dec, buffer, len, dst, dst_is_device, pitch, out_codec, rshift, gshift, bshift, stream_cs,
                                     stream_cs == UGB200_JPEG_CS_NATIVE ? UGB200_JPEG_CS_NATIVE : UGB200_JPEG_CS_Y709);
}

// ---- gpujpeg ---------------------------------------------------------------------------------------------------------------------
#if UGB_DECOMPRESS_MODULES & 1
namespace {
struct state_decompress_gpujpeg {  // gpujpeg.c:63-70
        ugb200_jpeg_decoder *decoder = nullptr;
        struct video_desc desc{};
        int rshift = 0, gshift = 0, bshift = 0, pitch = 0;
        codec_t out_codec = VIDEO_CODEC_NONE;
        int stream_cs = jpeg_decode_cs_from_env();
        int upsampling = jpeg_decode_upsample_from_env(stream_cs);
};
}  // namespace

static void *gpujpeg_decompress_init(void)
{
        if (cuda_wrapper_set_device((int) cuda_devices[0]) != CUDA_WRAPPER_SUCCESS) {  // gpujpeg_init_device, gpujpeg.c:163
                fprintf(stderr, "[GPUJPEG dec.] initializing CUDA device %u failed.\n", cuda_devices[0]);
                return nullptr;
        }
        return new state_decompress_gpujpeg();
}
static int gpujpeg_decompress_reconfigure(void *state, struct video_desc desc, int rshift, int gshift, int bshift, int pitch, codec_t out_codec)
{
        auto *s = (state_decompress_gpujpeg *) state;
        if (out_codec != RGB && out_codec != RGBA && out_codec != UYVY && out_codec != I420 && out_codec != VIDEO_CODEC_NONE) {
                return 0;  // the reference asserts this set, gpujpeg.c:181-182
        }
        s->desc = desc, s->rshift = rshift, s->gshift = gshift, s->bshift = bshift, s->pitch = pitch, s->out_codec = out_codec;
        if (!s->decoder) {
                s->decoder = ugb200_jpeg_decoder_create(nullptr);
                if (s->decoder) {
                        ugb200_jpeg_decoder_set_upsampling(s->decoder, s->upsampling);
                }
        }
        // dst holds pitch * desc.height bytes: a stream that declares another size must not be decoded into it
        return s->decoder != nullptr && ugb200_jpeg_decoder_expect(s->decoder, (int) desc.width, (int) desc.height) == 0;
}
/// gpujpeg_probe_internal_codec, gpujpeg.c:205-262
static decompress_status gpujpeg_probe_internal_codec(unsigned char *buffer, size_t len, struct pixfmt_desc *internal_prop)
{
        struct ugb200_jpeg_image_info info;
        if (ugb200_jpeg_get_image_info(buffer, len, &info) != 0) {
                fprintf(stderr, "[GPUJPEG dec.] probe - cannot get image info!\n");
                return DECODER_NO_FRAME;
        }
        internal_prop->depth = 8;
        internal_prop->rgb = info.native_codec == RGB || info.native_codec == RGBA;  // four components: R G B A (gpujpeg.c:254-260)
        internal_prop->subsampling = info.components == 4 ? SUBS_4444 : info.h_samp == 1 ? SUBS_444 : info.v_samp == 1 ? SUBS_422 : SUBS_420;
        return DECODER_GOT_CODEC;
}
static decompress_status gpujpeg_decompress(void *state, unsigned char *dst, unsigned char *buffer, unsigned int src_len, int, struct video_frame_callbacks *,
                                            struct pixfmt_desc *internal_prop)
{
        auto *s = (state_decompress_gpujpeg *) state;
        if (s->out_codec == VIDEO_CODEC_NONE) {
                return gpujpeg_probe_internal_codec(buffer, src_len, internal_prop);
        }
        cuda_wrapper_set_device((int) cuda_devices[0]);
        // the device path writes any pitch and any RGBA shifts directly (the reference needs a second CPU pass for those, gpujpeg.c:295-318)
        const int rc = jpeg_module_decode(s->decoder, s->stream_cs, buffer, src_len, dst, 0, s->pitch, s->out_codec, s->rshift, s->gshift, s->bshift);
        return rc == 0 ? DECODER_GOT_FRAME : DECODER_NO_FRAME;
}
static void gpujpeg_decompress_done(void *state)
{
        auto *s = (state_decompress_gpujpeg *) state;
        ugb200_jpeg_decoder_destroy(s->decoder);
        delete s;
}
static int gpujpeg_decompress_get_priority(codec_t compression, struct pixfmt_desc, codec_t ugc)  // gpujpeg.c:355-367
{
        if (compression != JPEG) {
                return -1;
        }
        if (ugc == VIDEO_CODEC_NONE) {
                return VDEC_PRIO_PROBE_HI;
        }
        return ugc == I420 || ugc == RGB || ugc == RGBA || ugc == UYVY ? VDEC_PRIO_PREFERRED : VDEC_PRIO_NA;
}
static const struct video_decompress_info gpujpeg_dec_info = { gpujpeg_decompress_init, gpujpeg_decompress_reconfigure, gpujpeg_decompress, no_corrupted_frames,
                                                               gpujpeg_decompress_done, gpujpeg_decompress_get_priority };
REGISTER_MODULE(gpujpeg, &gpujpeg_dec_info, LIBRARY_CLASS_VIDEO_DECOMPRESS, VIDEO_DECOMPRESS_ABI_VERSION);
#endif  // gpujpeg

// ---- gpujpeg_to_dxt ------------------------------------------------------------------------------------------------------------------
#if UGB_DECOMPRESS_MODULES & 2
namespace {
struct state_gpujpeg_to_dxt {
        ugb200_jpeg_decoder *decoder = nullptr;
        void *rgb = nullptr, *dxt = nullptr;  // device
        size_t rgb_cap = 0, dxt_cap = 0;
        int stream_cs = jpeg_decode_cs_from_env();
        int upsampling = jpeg_decode_upsample_from_env(stream_cs);
        struct video_desc desc{};
        codec_t out_codec = VIDEO_CODEC_NONE;
};
}  // namespace
static void *gpujpeg_to_dxt_init(void)
{
        if (cuda_wrapper_set_device((int) cuda_devices[0]) != CUDA_WRAPPER_SUCCESS) {
                return nullptr;
        }
        auto *s = new state_gpujpeg_to_dxt();
        s->decoder = ugb200_jpeg_decoder_create(nullptr);
        if (!s->decoder) {
                delete s;
                return nullptr;
        }
        ugb200_jpeg_decoder_set_upsampling(s->decoder, s->upsampling);
        return s;
}
static int gpujpeg_to_dxt_reconfigure(void *state, struct video_desc desc, int, int, int, int pitch, codec_t out_codec)
{
        auto *s = (state_gpujpeg_to_dxt *) state;
        if ((out_codec != DXT1 && out_codec != DXT5) || desc.width % 4 || desc.height % 4 || pitch != (int) vc_get_linesize(desc.width, out_codec)) {
                return 0;  // gpujpeg_to_dxt.cpp:230-236
        }
        const size_t rgb = (size_t) desc.width * desc.height * 3, dxt = (size_t) desc.width * desc.height / (out_codec == DXT1 ? 2 : 1);
        if (rgb > s->rgb_cap) {
                cuda_wrapper_free(s->rgb);
                if (cuda_wrapper_malloc(&s->rgb, rgb) != CUDA_WRAPPER_SUCCESS) {
                        return 0;
                }
                s->rgb_cap = rgb;
        }
        if (dxt > s->dxt_cap) {
                cuda_wrapper_free(s->dxt);
                if (cuda_wrapper_malloc(&s->dxt, dxt) != CUDA_WRAPPER_SUCCESS) {
                        return 0;
                }
                s->dxt_cap = dxt;
        }
        s->desc = desc, s->out_codec = out_codec;
        return ugb200_jpeg_decoder_expect(s->decoder, (int) desc.width, (int) desc.height) == 0;  // s->rgb holds width * height * 3 bytes
}
/// worker_thread, gpujpeg_to_dxt.cpp:134-166: decode to RGB on the device, encode with mirrored height, copy the blocks out
static decompress_status gpujpeg_to_dxt_decompress(void *state, unsigned char *dst, unsigned char *buffer, unsigned int src_len, int, struct video_frame_callbacks *,
                                                   struct pixfmt_desc *)
{
        auto *s = (state_gpujpeg_to_dxt *) state;
        cuda_wrapper_set_device((int) cuda_devices[0]);
        if (jpeg_module_decode(s->decoder, s->stream_cs, buffer, src_len, s->rgb, 1, 0, RGB, 0, 8, 16) != 0) {
                return DECODER_NO_FRAME;
        }
        const int w = (int) s->desc.width, h = (int) s->desc.height;
        const int rc = s->out_codec == DXT1 ? cuda_rgb_to_dxt1(s->rgb, s->dxt, w, -h, nullptr) : cuda_rgb_to_dxt6(s->rgb, s->dxt, w, -h, nullptr);
        if (rc != 0 || cuda_wrapper_memcpy(dst, s->dxt, (size_t) w * h / (s->out_codec == DXT1 ? 2 : 1), CUDA_WRAPPER_MEMCPY_DEVICE_TO_HOST) != CUDA_WRAPPER_SUCCESS) {
                return DECODER_NO_FRAME;
        }
        return DECODER_GOT_FRAME;
}
static void gpujpeg_to_dxt_done(void *state)
{
        auto *s = (state_gpujpeg_to_dxt *) state;
        ugb200_jpeg_decoder_destroy(s->decoder);
        cuda_wrapper_free(s->rgb), cuda_wrapper_free(s->dxt);
        delete s;
}
static int gpujpeg_to_dxt_get_priority(codec_t compression, struct pixfmt_desc, codec_t ugc)  // gpujpeg_to_dxt.cpp:364-369
{
        return compression == JPEG && (ugc == DXT1 || ugc == DXT5) ? 900 : -1;
}
static const struct video_decompress_info gpujpeg_to_dxt_info = { gpujpeg_to_dxt_init, gpujpeg_to_dxt_reconfigure, gpujpeg_to_dxt_decompress, no_corrupted_frames,
                                                                  gpujpeg_to_dxt_done, gpujpeg_to_dxt_get_priority };
REGISTER_MODULE(gpujpeg_to_dxt, &gpujpeg_to_dxt_info, LIBRARY_CLASS_VIDEO_DECOMPRESS, VIDEO_DECOMPRESS_ABI_VERSION);
#endif  // gpujpeg_to_dxt

// ---- dxt_cuda: DXT1 / DXT5-YCoCg -> RGB / RGBA / UYVY ----------------------------------------------------------------------------------
#if UGB_DECOMPRESS_MODULES & 4
namespace {
struct state_dxt_cuda {
        void *blocks = nullptr, *rgb = nullptr, *conv = nullptr;  // device
        size_t blocks_cap = 0, rgb_cap = 0, conv_cap = 0;
        struct video_desc desc{};
        int rshift = 0, gshift = 8, bshift = 16, pitch = 0;
        codec_t out_codec = VIDEO_CODEC_NONE;
};
bool dev_grow(void *&p, size_t &cap, size_t need)
{
        if (need <= cap) {
                return true;
        }
        cuda_wrapper_free(p);
        p = nullptr, cap = 0;
        if (cuda_wrapper_malloc(&p, need) != CUDA_WRAPPER_SUCCESS) {
                return false;
        }
        cap = need;
        return true;
}
}  // namespace
static void *dxt_cuda_init(void) { return cuda_wrapper_set_device((int) cuda_devices[0]) == CUDA_WRAPPER_SUCCESS ? new state_dxt_cuda() : nullptr; }
static int dxt_cuda_reconfigure(void *state, struct video_desc desc, int rshift, int gshift, int bshift, int pitch, codec_t out_codec)
{
        auto *s = (state_dxt_cuda *) state;
        if ((desc.color_spec != DXT1 && desc.color_spec != DXT5) || (out_codec != RGB && out_codec != RGBA && out_codec != UYVY) || desc.width % 4 || desc.height % 4) {
                return 0;
        }
        s->desc = desc, s->rshift = rshift, s->gshift = gshift, s->bshift = bshift, s->pitch = pitch, s->out_codec = out_codec;
        return dev_grow(s->blocks, s->blocks_cap, (size_t) desc.width * desc.height) && dev_grow(s->rgb, s->rgb_cap, (size_t) desc.width * desc.height * 3 + 64) &&
               dev_grow(s->conv, s->conv_cap, (size_t) desc.width * desc.height * 4 + 64);
}
static decompress_status dxt_cuda_decompress(void *state, unsigned char *dst, unsigned char *buffer, unsigned int src_len, int, struct video_frame_callbacks *,
                                             struct pixfmt_desc *)
{
        auto *s = (state_dxt_cuda *) state;
        const int w = (int) s->desc.width, h = (int) s->desc.height;
        const size_t need = (size_t) w * h / (s->desc.color_spec == DXT1 ? 2 : 1);
        if (src_len < need) {
                return DECODER_NO_FRAME;
        }
        cuda_wrapper_set_device((int) cuda_devices[0]);
        if (cuda_wrapper_memcpy(s->blocks, buffer, need, CUDA_WRAPPER_MEMCPY_HOST_TO_DEVICE) != CUDA_WRAPPER_SUCCESS) {
                return DECODER_NO_FRAME;
        }
        int rc = s->desc.color_spec == DXT1 ? ugb200_dxt1_to_rgb(s->blocks, s->rgb, w, h, 0, 0, nullptr) : ugb200_dxt5ycocg_to_rgb(s->blocks, s->rgb, w, h, 0, 0, nullptr);
        const void *res = s->rgb;
        const long ls = (long) vc_get_linesize((unsigned) w, s->out_codec);
        if (rc == 0 && s->out_codec != RGB) {
                rc = ugb200_pixfmt_convert(RGB, s->out_codec, s->conv, ls, s->rgb, (long) w * 3, (int) ls, h, 0, s->rshift, s->gshift, s->bshift, nullptr);
                res = s->conv;
        }
        if (rc != 0) {
                return DECODER_NO_FRAME;
        }
        const long pitch = s->pitch ? s->pitch : ls;
        if (pitch == ls) {
                rc = cuda_wrapper_memcpy(dst, res, (size_t) ls * h, CUDA_WRAPPER_MEMCPY_DEVICE_TO_HOST);
        } else {
                rc = cuda_wrapper_memcpy2d(dst, (size_t) pitch, res, (size_t) ls, (size_t) ls, (size_t) h, CUDA_WRAPPER_MEMCPY_DEVICE_TO_HOST);
        }
        return rc == CUDA_WRAPPER_SUCCESS ? DECODER_GOT_FRAME : DECODER_NO_FRAME;
}
static void dxt_cuda_done(void *state)
{
        auto *s = (state_dxt_cuda *) state;
        cuda_wrapper_free(s->blocks), cuda_wrapper_free(s->rgb), cuda_wrapper_free(s->conv);
        delete s;
}
static int dxt_cuda_get_priority(codec_t compression, struct pixfmt_desc, codec_t ugc)  // same contract as dxt_glsl.c:228-237 (+ RGB)
{
        if (compression != DXT1 && compression != DXT5) {
                return -1;
        }
        return ugc == RGBA || ugc == UYVY || ugc == RGB ? 500 : -1;
}
static const struct video_decompress_info dxt_cuda_info = { dxt_cuda_init, dxt_cuda_reconfigure, dxt_cuda_decompress, no_corrupted_frames, dxt_cuda_done,
                                                            dxt_cuda_get_priority };
REGISTER_MODULE(dxt_cuda, &dxt_cuda_info, LIBRARY_CLASS_VIDEO_DECOMPRESS, VIDEO_DECOMPRESS_ABI_VERSION);
#endif  // dxt_cuda

