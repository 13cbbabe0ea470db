#include "video_codec.h"

#include <algorithm>
#include <cassert>
#include <cstring>
#include <strings.h>
#include <vector>

namespace {
struct info_t {
        codec_t codec;
        const char *name;
        int block_bytes, block_pixels, h_align, bits;
        bool rgb;
        enum subsampling subs;
};
// codec_info[], src/video_codec.c:120-206 (pixel formats + the compressed formats this path emits)
const info_t infos[] = {
        { RGBA, "RGBA", 4, 1, 1, 8, true, SUBS_4444 }, { UYVY, "UYVY", 4, 2, 2, 8, false, SUBS_422 },  { YUYV, "YUYV", 4, 2, 2, 8, false, SUBS_422 },
        { VUYA, "VUYA", 4, 1, 1, 8, false, SUBS_4444 }, { R10k, "R10k", 4, 1, 64, 10, true, SUBS_444 }, { R12L, "R12L", 36, 8, 8, 12, true, SUBS_444 },
        { v210, "v210", 16, 6, 48, 10, false, SUBS_422 }, { UGB_DVS10, "DVS10", 16, 6, 48, 10, false, SUBS_422 }, { DXT1, "DXT1", 1, 2, 0, 2, true, SUBS_UNKNOWN }, { DXT5, "DXT5", 1, 1, 0, 4, false, SUBS_UNKNOWN },
        { RGB, "RGB", 3, 1, 1, 8, true, SUBS_444 },      { JPEG, "JPEG", 1, 1, 0, 8, false, SUBS_UNKNOWN }, { BGR, "BGR", 3, 1, 1, 8, true, SUBS_444 },
        { RG48, "RG48", 6, 1, 1, 16, true, SUBS_444 },   { I420, "I420", 3, 2, 2, 8, false, SUBS_420 },     { Y216, "Y216", 8, 2, 2, 16, false, SUBS_422 },
        { Y416, "Y416", 8, 1, 1, 16, false, SUBS_4444 },
};
const info_t *find(codec_t c)
{
        for (const info_t &i : infos) {
                if (i.codec == c) {
                        return &i;
                }
        }
        return nullptr;
}
const char pixfmt_conv_pref[] = "dsc";  // video_codec.c:80
}  // namespace

int vc_get_linesize(unsigned int width, codec_t codec)
{
        const info_t *i = find(codec);
        if (!i) {
                return 0;
        }
        if (i->h_align) {
                width = (width + i->h_align - 1) / i->h_align * i->h_align;
        }
        return (width + i->block_pixels - 1) / i->block_pixels * i->block_bytes;
}
int vc_get_size(unsigned int width, codec_t codec)
{
        const info_t *i = find(codec);
        return i ? (width + i->block_pixels - 1) / i->block_pixels * i->block_bytes : 0;
}
size_t vc_get_datalen(unsigned int width, unsigned int height, codec_t codec)
{
        if (codec == I420) {
                return (size_t) width * height + 2 * (size_t) ((width + 1) / 2) * ((height + 1) / 2);
        }
        return (size_t) vc_get_linesize(width, codec) * height;
}
int get_bits_per_component(codec_t codec)
{
        const info_t *i = find(codec);
        return i ? i->bits : 0;
}
bool codec_is_a_rgb(codec_t codec)
{
        const info_t *i = find(codec);
        return i && i->rgb;
}
const char *get_codec_name(codec_t codec)
{
        const info_t *i = find(codec);
        return i ? i->name : "(unknown)";
}
codec_t get_codec_from_name(const char *name)
{
        for (const info_t &i : infos) {
                if (strcasecmp(i.name, name) == 0) {
                        return i.codec;
                }
        }
        return VIDEO_CODEC_NONE;
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
