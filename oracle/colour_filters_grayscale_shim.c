// TEST INFRASTRUCTURE: the UNMODIFIED src/capture_filter/grayscale.c, included where it lies under $(REF), with its
// static functions exposed to tests/test_colour_filters.py.
#include "capture_filter/grayscale.c"

static struct video_frame *frame_on(int codec, int width, int height, void *data)
{
        struct video_frame *f = vf_alloc(1);
        f->color_spec = (codec_t) codec;
        f->interlacing = PROGRESSIVE;
        f->fps = 30;
        f->tiles[0].width = width;
        f->tiles[0].height = height;
        f->tiles[0].data = data;
        f->tiles[0].data_len = vc_get_linesize(width, (codec_t) codec) * height;
        return f;
}

/// filter() with the output through the vo_pp_out_buffer hook: 0, or 1 where filter returns its input
int ref_grayscale_filter(int codec, int width, int height, char *in, char *out)
{
        struct state_grayscale s = { 0 };
        vo_pp_set_out_buffer(&s, out);
        struct video_frame *f = frame_on(codec, width, height, in);
        struct video_frame *o = filter(&s, f);
        const int rc = o == f ? 1 : 0;
        if (o != f) {
                VIDEO_FRAME_DISPOSE(o);
        }
        vf_free(f);
        return rc;
}

/// the vo_pp wrapper over one UYVY frame
int ref_grayscale_vopp(const char *cfg, int width, int height, const char *in, char *out)
{
        void *s = vo_pp_grayscale.init(cfg);
        if (s == NULL) {
                return -2;
        }
        struct video_desc desc = { .width = width, .height = height, .color_spec = UYVY, .interlacing = PROGRESSIVE, .fps = 30, .tile_count = 1 };
        vo_pp_grayscale.reconfigure(s, desc);
        struct video_frame *f = vo_pp_grayscale.getf(s);
        memcpy(f->tiles[0].data, in, f->tiles[0].data_len);
        struct video_frame *o = frame_on(UYVY, width, height, out);
        const bool ok = vo_pp_grayscale.vo_postprocess(s, f, o, vc_get_linesize(width, UYVY));
        vf_free(o);
        vo_pp_grayscale.done(s);
        return ok ? 0 : -1;
}
