// TEST INFRASTRUCTURE: the UNMODIFIED src/vo_postprocess/split.c, included where it lies under $(REF), with its static
// functions exposed to tests/test_geometry_filters.py.  The harness owns the input and every output tile.
#include "vo_postprocess/split.c"

/// split_init + reconfigure + split_postprocess into the harness's tiles: 0, -1 (postprocess failed) or -2 (init
/// refused cfg); xy = the grid the module parsed
int ref_split_vopp(const char *cfg, int codec, int width, int height, char *in, char **tiles, int *xy)
{
        struct state_split *s = split_init(cfg);
        if (s == NULL) {
                return -2;
        }
        xy[0] = s->grid_width;
        xy[1] = s->grid_height;
        struct video_desc desc = { .width = width, .height = height, .color_spec = (codec_t) codec, .interlacing = PROGRESSIVE,
                                   .fps = 30, .tile_count = 1 };
        split_postprocess_reconfigure(s, desc);
        struct video_frame *f = split_getf(s);
        char *own = f->tiles[0].data;
        f->tiles[0].data = in;
        struct video_desc od;
        int mode;
        split_get_out_desc(s, &od, &mode);
        struct video_frame *o = vf_alloc(od.tile_count);
        for (unsigned i = 0; i < od.tile_count; ++i) {
                o->tiles[i].data = tiles[i];
        }
        const bool ok = split_postprocess(s, f, o, 0);
        f->tiles[0].data = own;
        vf_free(o);
        split_done(s);
        return ok ? 0 : -1;
}
