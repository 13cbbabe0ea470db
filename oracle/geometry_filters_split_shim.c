// TEST INFRASTRUCTURE: the UNMODIFIED src/capture_filter/split.c and src/vo_postprocess/split.c, each included where
// it lies under $(REF) by a shim of its own (this one and geometry_filters_vo_split_shim.c), with their static
// functions exposed to tests/test_geometry_filters.py.  vf_split comes from the shim of src/utils/vf_split.cpp.
#include "capture_filter/split.c"

/// the capture filter's init: 0 with x, y parsed, or its return value
int ref_split_init(const char *cfg, int *x, int *y)
{
        void *st = NULL;
        const int rc = init(NULL, cfg, &st);
        if (rc == 0) {
                struct state_split *s = st;
                *x = s->x;
                *y = s->y;
                done(st);
        }
        return rc;
}

/// init + filter(): each output tile's data_len bytes are copied to tiles[i] (only the bytes vf_split writes are
/// meaningful: the tiles come from malloc)
int ref_split_filter(const char *cfg, int codec, int width, int height, char *in, char **tiles)
{
        void *st = NULL;
        if (init(NULL, cfg, &st) != 0) {
                return -2;
        }
        struct video_frame *f = vf_alloc(1);
        f->color_spec = (codec_t) codec;
        f->interlacing = PROGRESSIVE;
        f->fps = 30;
        f->tiles[0].width = width;
        f->tiles[0].height = height;
        f->tiles[0].data = in;
        f->tiles[0].data_len = vc_get_linesize(width, (codec_t) codec) * height;
        struct video_frame *o = filter(st, f);
        for (unsigned i = 0; i < o->tile_count; ++i) {
                memcpy(tiles[i], o->tiles[i].data, o->tiles[i].data_len);
        }
        VIDEO_FRAME_DISPOSE(o);
        vf_free(f);
        done(st);
        return 0;
}
