// TEST INFRASTRUCTURE: the UNMODIFIED src/vo_postprocess/crop.c, included where it lies under $(REF), with its
// static functions exposed to tests/test_geometry_filters.py.  The harness owns the input (with slack before and
// after it: rows may start before the frame and read past it) and the output.
#include "vo_postprocess/crop.c"

/// crop_init + crop_postprocess_reconfigure: 0 with geom = {out width, out height, xoff, yoff} as crop_postprocess
/// computes the offsets, -2 where init refuses cfg
int ref_crop_geometry(const char *cfg, int codec, int width, int height, int *geom)
{
        struct state_crop *s = crop_init(cfg);
        if (s == NULL) {
                return -2;
        }
        struct video_desc desc = { .width = width, .height = height, .color_spec = (codec_t) codec, .interlacing = PROGRESSIVE,
                                   .fps = 30, .tile_count = 1 };
        crop_postprocess_reconfigure(s, desc);
        geom[0] = (int) s->out_desc.width;
        geom[1] = (int) s->out_desc.height;
        geom[2] = s->xoff + s->out_desc.width > desc.width ? desc.width - s->out_desc.width : (unsigned) s->xoff;
        geom[3] = s->yoff + s->out_desc.height > desc.height ? desc.height - s->out_desc.height : (unsigned) s->yoff;
        crop_done(s);
        return 0;
}

/// init, reconfigure, then crop_postprocess into `out` at req_pitch (< 0: the capture filter's vc_get_linesize(out
/// width), as cf_crop_filter passes it): 0, -1 (postprocess failed) or -2 (init refused cfg)
int ref_crop(const char *cfg, int codec, int width, int height, char *in, char *out, int req_pitch)
{
        struct state_crop *s = crop_init(cfg);
        if (s == NULL) {
                return -2;
        }
        struct video_desc desc = { .width = width, .height = height, .color_spec = (codec_t) codec, .interlacing = PROGRESSIVE,
                                   .fps = 30, .tile_count = 1 };
        crop_postprocess_reconfigure(s, desc);
        struct video_frame *f = vf_alloc_desc(desc);
        f->tiles[0].data = in;
        struct video_frame *o = vf_alloc_desc(s->out_desc);
        o->tiles[0].data = out;
        if (req_pitch < 0) {
                req_pitch = vc_get_linesize(s->out_desc.width, (codec_t) codec);
        }
        const bool ok = crop_postprocess(s, f, o, req_pitch);
        vf_free(o);
        vf_free(f);
        crop_done(s);
        return ok ? 0 : -1;
}
