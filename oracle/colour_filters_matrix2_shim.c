// TEST INFRASTRUCTURE: the UNMODIFIED src/capture_filter/matrix2.c, included where it lies under $(REF), with its
// static functions exposed to tests/test_colour_filters.py.  The harness owns the state, the output and the Y416
// scratch: on v210 the reference reads 3 x tmp_len from the scratch and writes w * h * 8 bytes into the v210 frame.
#include "capture_filter/matrix2.c"

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

/// filter() on a harness-owned state: y416_tmp_buffer = tmp (tmp_sz bytes, more than w * h * 8, so it is kept)
void ref_matrix2_filter(const double *m, int codec, int width, int height, char *in, char *out, char *tmp, size_t tmp_sz)
{
        struct state_capture_filter_matrix2 s = { 0 };
        memcpy(s.transform_matrix, m, sizeof s.transform_matrix);
        s.y416_tmp_buffer = tmp;
        s.y416_tmp_buffer_sz = tmp_sz;
        vo_pp_set_out_buffer(&s, out);
        struct video_frame *f = frame_on(codec, width, height, in);
        struct video_frame *o = filter(&s, f);
        VIDEO_FRAME_DISPOSE(o);
        vf_free(f);
}

/// init(): its return value; on 0 the parsed matrix is copied out
int ref_matrix2_init(const char *cfg, double *m)
{
        void *st = NULL;
        const int rc = init(NULL, cfg, &st);
        if (rc == 0) {
                struct state_capture_filter_matrix2 *s = st;
                memcpy(m, s->transform_matrix, sizeof s->transform_matrix);
                done(st);
        }
        return rc;
}

/// the vo_pp wrapper over one frame (UYVY and Y416 only: on v210 the module's own scratch would overflow)
int ref_matrix2_vopp(const char *cfg, int codec, int width, int height, const char *in, char *out)
{
        void *s = vo_pp_matrix2.init(cfg);
        if (s == NULL) {
                return -2;
        }
        struct video_desc desc = { .width = width, .height = height, .color_spec = (codec_t) codec, .interlacing = PROGRESSIVE,
                                   .fps = 30, .tile_count = 1 };
        vo_pp_matrix2.reconfigure(s, desc);
        struct video_frame *f = vo_pp_matrix2.getf(s);
        memcpy(f->tiles[0].data, in, f->tiles[0].data_len);
        struct video_frame *o = frame_on(codec, width, height, out);
        const bool ok = vo_pp_matrix2.vo_postprocess(s, f, o, vc_get_linesize(width, (codec_t) codec));
        vf_free(o);
        vo_pp_matrix2.done(s);
        return ok ? 0 : -1;
}
