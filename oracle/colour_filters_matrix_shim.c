// TEST INFRASTRUCTURE: the UNMODIFIED src/capture_filter/matrix.c, included where it lies under $(REF), with its
// static functions exposed to tests/test_colour_filters.py.  The harness owns every buffer: at odd widths the UYVY
// branch writes 3 * h bytes past the RGB frame.
#include "capture_filter/matrix.c"

// module registration constructors (of all four shims): nothing to register with here
void register_library(const char *name, const void *info, enum library_class cls, int abi, enum mod_visibility_flag flag)
{
        (void) name, (void) info, (void) cls, (void) abi, (void) flag;
}

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

/// filter() on a harness-built state, output through the vo_pp_out_buffer hook; 0, or -1 where filter returns NULL
int ref_matrix_filter(const double *m, int check_bounds, int codec, int width, int height, char *in, char *out)
{
        struct state_capture_filter_matrix s = { 0 };
        memcpy(s.transform_matrix, m, sizeof s.transform_matrix);
        s.check_bounds = check_bounds != 0;
        vo_pp_set_out_buffer(&s, out);
        struct video_frame *f = frame_on(codec, width, height, in);
        struct video_frame *o = filter(&s, f);
        const int rc = o != NULL ? 0 : -1;
        VIDEO_FRAME_DISPOSE(o);
        vf_free(f);
        return rc;
}

/// init(): its return value; on 0 the parsed matrix and check_bounds are copied out
int ref_matrix_init(const char *cfg, double *m, int *check_bounds)
{
        void *st = NULL;
        const int rc = init(NULL, cfg, &st);
        if (rc == 0) {
                struct state_capture_filter_matrix *s = st;
                memcpy(m, s->transform_matrix, sizeof s->transform_matrix);
                *check_bounds = s->check_bounds;
                done(st);
        }
        return rc;
}

/// the vo_pp wrapper's own init / reconfigure / getf / postprocess / done over one frame: 0, -1 (postprocess
/// failed) or -2 (init refused cfg)
int ref_matrix_vopp(const char *cfg, int codec, int width, int height, const char *in, int out_codec, char *out)
{
        void *s = vo_pp_matrix.init(cfg);
        if (s == NULL) {
                return -2;
        }
        struct video_desc desc = { .width = width, .height = height, .color_spec = (codec_t) codec, .interlacing = PROGRESSIVE,
                                   .fps = 30, .tile_count = 1 };
        vo_pp_matrix.reconfigure(s, desc);
        struct video_frame *f = vo_pp_matrix.getf(s);
        memcpy(f->tiles[0].data, in, f->tiles[0].data_len);
        struct video_frame *o = frame_on(out_codec, width, height, out);
        const bool ok = vo_pp_matrix.vo_postprocess(s, f, o, vc_get_linesize(width, (codec_t) out_codec));
        vf_free(o);
        vo_pp_matrix.done(s);
        return ok ? 0 : -1;
}
