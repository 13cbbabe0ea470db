// codec_t registry and converter selection — host mirror of src/video_codec.{h,c} and of the lookup half of
// src/pixfmt_conv.c (get_decoder_from_to :3110-3125, get_best_decoder_from :3148-3172).  On the device a "decoder"
// is a whole-buffer kernel, so decoder_t here is just the (in, out) pair accepted by ugb200_pixfmt_convert.
#pragma once
#include "ug_types.h"

// The layout of every codec id (codec_info[], video_codec.c:120-206); ids outside [NONE, COUNT) have none: sizes 0.
long vc_linesize64(long width, codec_t codec);                                   // vc_get_linesize without the int overflow
int vc_get_linesize(unsigned int width, codec_t codec);                          // video_codec.c:507-521
size_t vc_get_datalen(unsigned int width, unsigned int height, codec_t codec);   // :543-560, in 64 bits
int get_bits_per_component(codec_t codec);
double get_bpp(codec_t codec);
int get_pf_block_bytes(codec_t codec);
bool is_codec_opaque(codec_t codec);
bool codec_is_planar(codec_t codec);                                             // only I420
const char *get_codec_name(codec_t codec);
struct pixfmt_desc get_pixfmt_desc(codec_t pixfmt);                              // :1134-1143
int compare_pixdesc(const pixfmt_desc *a, const pixfmt_desc *b, const pixfmt_desc *src);  // :1148-1192

struct decoder_t {
        codec_t in, out;
        explicit operator bool() const { return in != VIDEO_CODEC_NONE; }
};
decoder_t get_decoder_from_to(codec_t in, codec_t out);
decoder_t get_best_decoder_from(codec_t in, const codec_t *out_candidates, codec_t *out);
