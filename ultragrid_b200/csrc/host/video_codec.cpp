#include "video_codec.h"

#include <algorithm>
#include <cassert>
#include <vector>

namespace {
struct info_t {
        const char *name;
        int block_bytes, block_pixels, h_align, bits;
        bool rgb, opaque;
        enum subsampling subs;
};
// codec_info[] (src/video_codec.c:120-206), one row per codec id.  HW_VDPAU and DRM_PRIME are constant-size handles with
// no byte layout: their block bytes are 0 here (the reference's are the handle's size), so every size of them is 0.
const info_t infos[] = {
        [UGB_VIDEO_CODEC_NONE] = { "(none)", 0, 0, 0, 0, false, true, SUBS_UNKNOWN },
        [UGB_RGBA] = { "RGBA", 4, 1, 1, 8, true, false, SUBS_4444 },
        [UGB_UYVY] = { "UYVY", 4, 2, 2, 8, false, false, SUBS_422 },
        [UGB_YUYV] = { "YUYV", 4, 2, 2, 8, false, false, SUBS_422 },
        [UGB_VUYA] = { "VUYA", 4, 1, 1, 8, false, false, SUBS_4444 },
        [UGB_R10k] = { "R10k", 4, 1, 64, 10, true, false, SUBS_444 },
        [UGB_R12L] = { "R12L", 36, 8, 8, 12, true, false, SUBS_444 },
        [UGB_v210] = { "v210", 16, 6, 48, 10, false, false, SUBS_422 },
        [UGB_DVS10] = { "DVS10", 16, 6, 48, 10, false, false, SUBS_422 },
        [UGB_DXT1] = { "DXT1", 1, 2, 0, 2, true, true, SUBS_UNKNOWN },
        [UGB_DXT1_YUV] = { "DXT1_YUV", 1, 2, 0, 2, false, true, SUBS_UNKNOWN },
        [UGB_DXT5] = { "DXT5", 1, 1, 0, 4, false, true, SUBS_UNKNOWN },
        [UGB_RGB] = { "RGB", 3, 1, 1, 8, true, false, SUBS_444 },
        [UGB_JPEG] = { "JPEG", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_JPEG_XS] = { "JPEG_XS", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_RAW] = { "raw", 1, 1, 0, 0, false, true, SUBS_UNKNOWN },
        [UGB_H264] = { "H.264", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_H265] = { "H.265", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_VP8] = { "VP8", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_VP9] = { "VP9", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_BGR] = { "BGR", 3, 1, 1, 8, true, false, SUBS_444 },
        [UGB_J2K] = { "J2K", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_J2KR] = { "J2KR", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_HW_VDPAU] = { "HW_VDPAU", 0, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_HFYU] = { "HFYU", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_FFV1] = { "FFV1", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_CFHD] = { "CFHD", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_RG48] = { "RG48", 6, 1, 1, 16, true, false, SUBS_444 },
        [UGB_AV1] = { "AV1", 1, 1, 0, 8, true, true, SUBS_UNKNOWN },
        [UGB_I420] = { "I420", 3, 2, 2, 8, false, false, SUBS_420 },
        [UGB_Y216] = { "Y216", 8, 2, 2, 16, false, false, SUBS_422 },
        [UGB_Y416] = { "Y416", 8, 1, 1, 16, false, false, SUBS_4444 },
        [UGB_PRORES] = { "PRORES", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_PRORES_4444] = { "PRORES_4444", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_PRORES_4444_XQ] = { "PRORES_4444_XQ", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_PRORES_422_HQ] = { "PRORES_422_HQ", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_PRORES_422] = { "PRORES_422", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_PRORES_422_PROXY] = { "PRORES_422_PROXY", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_PRORES_422_LT] = { "PRORES_422_LT", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_APV] = { "APV", 1, 1, 0, 0, false, true, SUBS_UNKNOWN },
        [UGB_PYROWAVE] = { "PYROWAVE", 1, 1, 0, 8, false, true, SUBS_UNKNOWN },
        [UGB_DRM_PRIME] = { "DRM_PRIME", 0, 1, 0, 8, false, true, SUBS_UNKNOWN },
};
static_assert(sizeof infos / sizeof infos[0] == UGB_VIDEO_CODEC_COUNT, "one row per codec id");

// ids outside the table have no layout
const info_t *find(codec_t c) { return (unsigned) c < UGB_VIDEO_CODEC_COUNT ? &infos[c] : nullptr; }
const char pixfmt_conv_pref[] = "dsc";  // video_codec.c:80
}  // namespace

long vc_linesize64(long width, codec_t codec)
{
        const info_t *i = find(codec);
        if (!i || i->block_pixels == 0) {
                return 0;
        }
        if (i->h_align) {
                width = (width + i->h_align - 1) / i->h_align * i->h_align;
        }
        return (width + i->block_pixels - 1) / i->block_pixels * i->block_bytes;
}
int vc_get_linesize(unsigned int width, codec_t codec) { return (int) vc_linesize64(width, codec); }
size_t vc_get_datalen(unsigned int width, unsigned int height, codec_t codec)
{
        if (codec_is_planar(codec)) {
                return (size_t) width * height + 2 * (size_t) ((width + 1) / 2) * ((height + 1) / 2);
        }
        return (size_t) vc_linesize64(width, codec) * height;
}
int get_bits_per_component(codec_t codec)
{
        const info_t *i = find(codec);
        return i ? i->bits : 0;
}
double get_bpp(codec_t codec)
{
        const info_t *i = find(codec);
        return i && i->block_pixels ? (double) i->block_bytes / i->block_pixels : 0;
}
int get_pf_block_bytes(codec_t codec)
{
        const info_t *i = find(codec);
        return i ? i->block_bytes : 0;
}
bool is_codec_opaque(codec_t codec)
{
        const info_t *i = find(codec);
        return i && i->opaque;
}
bool codec_is_planar(codec_t codec) { return codec == I420; }
const char *get_codec_name(codec_t codec)
{
        const info_t *i = find(codec);
        return i ? i->name : "(unknown)";
}
struct pixfmt_desc get_pixfmt_desc(codec_t pixfmt)
{
        const info_t *i = find(pixfmt);
        assert(i != nullptr);
        return pixfmt_desc{ i->bits, i->subs, i->rgb };
}

int compare_pixdesc(const pixfmt_desc *a, const pixfmt_desc *b, const pixfmt_desc *src)
{
        for (const char *f = pixfmt_conv_pref; *f; ++f) {  // first pass: anything worse than the source sorts last
                switch (*f) {
                case 'd':
                        if (a->depth != b->depth && (a->depth < src->depth || b->depth < src->depth)) {
                                return b->depth - a->depth;
                        }
                        break;
                case 's':
                        if (a->subsampling != b->subsampling && (a->subsampling < src->subsampling || b->subsampling < src->subsampling)) {
                                return b->subsampling - a->subsampling;
                        }
                        break;
                case 'c':
                        if (a->rgb != b->rgb) {
                                return a->rgb == src->rgb ? -1 : 1;
                        }
                        break;
                }
        }
        for (const char *f = pixfmt_conv_pref; *f; ++f) {  // both at least as good as the source: the closer one wins
                if (*f == 'd' && a->depth != b->depth) {
                        return a->depth - b->depth;
                }
                if (*f == 's' && a->subsampling != b->subsampling) {
                        return a->subsampling - b->subsampling;
                }
        }
        return 0;
}

decoder_t get_decoder_from_to(codec_t in, codec_t out)
{
        return ugb200_pixfmt_supported(in, out) ? decoder_t{ in, out } : decoder_t{ VIDEO_CODEC_NONE, VIDEO_CODEC_NONE };
}

decoder_t get_best_decoder_from(codec_t in, const codec_t *out_candidates, codec_t *out)
{
        for (const codec_t *it = out_candidates; *it != VIDEO_CODEC_NONE; ++it) {
                if (*it == in && in != RGBA && in != RGB) {  // pixfmt_conv.c:3150-3153
                        *out = in;
                        return decoder_t{ in, in };
                }
        }
        std::vector<codec_t> cand;
        for (const codec_t *it = out_candidates; *it != VIDEO_CODEC_NONE; ++it) {
                if (get_decoder_from_to(in, *it)) {
                        cand.push_back(*it);
                }
        }
        if (cand.empty()) {
                return decoder_t{ VIDEO_CODEC_NONE, VIDEO_CODEC_NONE };
        }
        const pixfmt_desc src = get_pixfmt_desc(in);
        std::sort(cand.begin(), cand.end(), [&](codec_t x, codec_t y) {  // best_decoder_cmp, pixfmt_conv.c:3128-3141
                const pixfmt_desc dx = get_pixfmt_desc(x), dy = get_pixfmt_desc(y);
                const int r = compare_pixdesc(&dx, &dy, &src);
                return r != 0 ? r < 0 : (int) x < (int) y;
        });
        *out = cand[0];
        return get_decoder_from_to(in, *out);
}
