// TEST INFRASTRUCTURE: the UNMODIFIED src/capture_filter/flip.c, included where it lies under $(REF), with its
// static functions exposed to tests/test_geometry_filters.py.
#include "capture_filter/flip.c"

// module registration constructors (of all the geometry shims): nothing to register with here
void register_library(const char *name, const void *info, enum library_class cls, int abi, enum mod_visibility_flag flag)
{
        (void) name, (void) info, (void) cls, (void) abi, (void) flag;
}

/// filter() with the output through the vo_pp_out_buffer hook, on a frame of the harness's buffer
int ref_flip_filter(int codec, int width, int height, char *in, char *out)
{
        void *st = NULL;
        if (init(NULL, "", &st) != 0) {
                return -2;
        }
        vo_pp_set_out_buffer(st, out);
        struct video_frame *f = vf_alloc(1);
        f->color_spec = (codec_t) codec;
        f->interlacing = PROGRESSIVE;
        f->fps = 30;
        f->tiles[0].width = width;
        f->tiles[0].height = height;
        f->tiles[0].data = in;
        f->tiles[0].data_len = vc_get_linesize(width, (codec_t) codec) * height;
        struct video_frame *o = filter(st, f);
        VIDEO_FRAME_DISPOSE(o);
        vf_free(f);
        done(st);
        return 0;
}
