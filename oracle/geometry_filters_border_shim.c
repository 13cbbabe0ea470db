// TEST INFRASTRUCTURE: the UNMODIFIED src/vo_postprocess/border.c, included where it lies under $(REF), with its
// static functions exposed to tests/test_geometry_filters.py.
#include "vo_postprocess/border.c"

/// border_init: 0 with the state's colour bytes and width / height, or -2 where it refuses cfg
int ref_border_init(const char *cfg, unsigned char *color, unsigned *wh)
{
        struct state_border *s = border_init(cfg);
        if (s == NULL) {
                return -2;
        }
        memcpy(color, s->color, 4);
        wh[0] = s->width;
        wh[1] = s->height;
        border_done(s);
        return 0;
}

/// init + reconfigure + border_postprocess from the harness's input into its output at pitch vc_get_linesize(width):
/// 0, -1 (postprocess failed) or -2 (init refused cfg)
int ref_border(const char *cfg, int codec, int width, int height, char *in, char *out)
{
        struct state_border *s = border_init(cfg);
        if (s == NULL) {
                return -2;
        }
        struct video_desc desc = { .width = width, .height = height, .color_spec = (codec_t) codec, .interlacing = PROGRESSIVE,
                                   .fps = 30, .tile_count = 1 };
        border_postprocess_reconfigure(s, desc);
        struct video_frame *f = vf_alloc_desc(desc);
        f->tiles[0].data = in;
        struct video_frame *o = vf_alloc_desc(desc);
        o->tiles[0].data = out;
        const bool ok = border_postprocess(s, f, o, vc_get_linesize(width, (codec_t) codec));
        vf_free(o);
        vf_free(f);
        border_done(s);
        return ok ? 0 : -1;
}
