// TEST INFRASTRUCTURE: the UNMODIFIED src/vo_postprocess/3d-interlaced.c, included where it lies under $(REF), with
// its static functions exposed to tests/test_geometry_filters.py.  The harness owns both eye tiles (with slack after
// them: rows are read past their end) and the output (the drifted rows are written past the frame).
#include "vo_postprocess/3d-interlaced.c"

/// init + reconfigure + interlaced_3d_postprocess from the harness's tiles: 0, -1 (postprocess failed) or -2 (init)
int ref_interlaced_3d(int codec, int width, int height, char *left, char *right, char *out)
{
        struct state_interlaced_3d *s = interlaced_3d_init("");
        if (s == NULL) {
                return -2;
        }
        struct video_desc desc = { .width = width, .height = height, .color_spec = (codec_t) codec, .interlacing = PROGRESSIVE,
                                   .fps = 30, .tile_count = 2 };
        interlaced_3d_postprocess_reconfigure(s, desc);
        struct video_frame *f = interlaced_3d_getf(s);
        char *own[2] = { f->tiles[0].data, f->tiles[1].data };
        f->tiles[0].data = left;
        f->tiles[1].data = right;
        struct video_desc od;
        int mode;
        interlaced_3d_get_out_desc(s, &od, &mode);
        struct video_frame *o = vf_alloc_desc(od);
        o->tiles[0].data = out;
        const bool ok = interlaced_3d_postprocess(s, f, o, vc_get_linesize(width, (codec_t) codec));
        vf_free(o);
        f->tiles[0].data = own[0];
        f->tiles[1].data = own[1];
        interlaced_3d_done(s);
        return ok ? 0 : -1;
}
