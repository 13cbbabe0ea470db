// TEST INFRASTRUCTURE: the UNMODIFIED src/vo_postprocess/interlace.c, included where it lies under $(REF), with its
// static functions exposed to tests/test_field_rate.py.  A translation unit of its own: temporal-deint.c defines a
// static copy_data_to_int_buf_if_cf too.
#include "vo_postprocess/interlace.c"

static struct video_frame *frame_on(int codec, int width, int height, void *data)
{
        struct video_frame *f = vf_alloc(1);
        f->color_spec = (codec_t) codec;
        f->interlacing = PROGRESSIVE;
        f->fps = 50;
        f->tiles[0].width = width;
        f->tiles[0].height = height;
        f->tiles[0].data = data;
        f->tiles[0].data_len = vc_get_linesize(width, (codec_t) codec) * height;
        return f;
}

/// interlace_postprocess once both frames are in: out row i from `first` (the module's s->odd) for even i, from
/// `second` (s->even) for odd i
int ref_interlace_weave(int codec, int width, int height, char *first, char *second, char *out, int pitch)
{
        struct state_interlace s;
        s.odd = frame_on(codec, width, height, first);
        s.even = frame_on(codec, width, height, second);
        s.last = EVEN;
        struct video_frame *o = frame_on(codec, width, height, out);
        const bool ok = interlace_postprocess(&s, s.even, o, pitch);
        vf_free(o);
        vf_free(s.odd);
        vf_free(s.even);
        return ok ? 0 : -1;
}

/// the module's own init / reconfigure / getf / postprocess over n progressive frames: out gets one merged frame
/// for every second input (n / 2 frames at pitch `pitch`); returns how many it emitted
int ref_interlace_sequence(int codec, int width, int height, const char *frames, int n, char *out, int pitch)
{
        void *s = vo_pp_interlace_info.init("");
        struct video_desc desc = { .width = width, .height = height, .color_spec = (codec_t) codec, .interlacing = PROGRESSIVE,
                                   .fps = 50, .tile_count = 1 };
        vo_pp_interlace_info.reconfigure(s, desc);
        const size_t fsz = (size_t) vc_get_linesize(width, (codec_t) codec) * height;
        int emitted = 0;
        for (int i = 0; i < n; ++i) {
                struct video_frame *in = vo_pp_interlace_info.getf(s);
                memcpy(in->tiles[0].data, frames + i * fsz, fsz);
                struct video_frame *o = frame_on(codec, width, height, out + (size_t) emitted * pitch * height);
                if (vo_pp_interlace_info.vo_postprocess(s, in, o, pitch)) {
                        ++emitted;
                }
                vf_free(o);
        }
        vo_pp_interlace_info.done(s);
        return emitted;
}
