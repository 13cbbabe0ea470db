// TEST INFRASTRUCTURE: the UNMODIFIED src/capture_filter/gamma.cpp, included where it lies under $(REF), with its
// state and static functions exposed to tests/test_colour_filters.py.  apply_lut splits a frame among
// hardware_concurrency() tasks of len / cpus samples each, so the harness needs that count to know the tail it skips.
#include "capture_filter/gamma.cpp"

static struct video_frame *frame_on(int codec, int width, int height, void *data)
{
        struct video_frame *f = vf_alloc(1);
        f->color_spec = (codec_t) codec;
        f->interlacing = PROGRESSIVE;
        f->fps = 30;
        f->tiles[0].width = width;
        f->tiles[0].height = height;
        f->tiles[0].data = (char *) data;
        f->tiles[0].data_len = vc_get_linesize(width, (codec_t) codec) * height;
        return f;
}

extern "C" {

unsigned ref_gamma_cpus()
{
        return thread::hardware_concurrency();
}

void *ref_gamma_create(double gamma, int out_depth)
{
        return new state_capture_filter_gamma(gamma, out_depth);
}

void ref_gamma_destroy(void *s)
{
        delete static_cast<state_capture_filter_gamma *>(s);
}

/// apply_gamma over in_len bytes: 0, or -1 where it throws
int ref_gamma_apply(void *s, int in_depth, int out_depth, size_t in_len, const void *in, void *out)
{
        try {
                static_cast<state_capture_filter_gamma *>(s)->apply_gamma(in_depth, out_depth, in_len, in, out);
        } catch (...) {
                return -1;
        }
        return 0;
}

/// filter() on a state made by ref_gamma_create, output through the vo_pp_out_buffer hook; -1 where it returns NULL
int ref_gamma_filter(void *st, int codec, int width, int height, char *in, char *out)
{
        auto *s = static_cast<state_capture_filter_gamma *>(st);
        vo_pp_set_out_buffer(s, out);
        struct video_frame *f = frame_on(codec, width, height, in);
        struct video_frame *o = filter(s, f);
        const int rc = o != nullptr ? 0 : -1;
        VIDEO_FRAME_DISPOSE(o);
        vf_free(f);
        return rc;
}

/// init(): its return value; on 0 the parsed out_depth is copied out
int ref_gamma_init(const char *cfg, int *out_depth)
{
        void *st = nullptr;
        const int rc = init(nullptr, cfg, &st);
        if (rc == 0) {
                *out_depth = static_cast<state_capture_filter_gamma *>(st)->out_depth;
                done(st);
        }
        return rc;
}

/// the vo_pp wrapper over one frame
int ref_gamma_vopp(const char *cfg, int codec, int width, int height, const char *in, int out_codec, char *out)
{
        void *s = vo_pp_gamma.init(cfg);
        if (s == nullptr) {
                return -2;
        }
        struct video_desc desc{};
        desc.width = width;
        desc.height = height;
        desc.color_spec = (codec_t) codec;
        desc.interlacing = PROGRESSIVE;
        desc.fps = 30;
        desc.tile_count = 1;
        vo_pp_gamma.reconfigure(s, desc);
        struct video_frame *f = vo_pp_gamma.getf(s);
        memcpy(f->tiles[0].data, in, f->tiles[0].data_len);
        struct video_frame *o = frame_on(out_codec, width, height, out);
        const bool ok = vo_pp_gamma.vo_postprocess(s, f, o, vc_get_linesize(width, (codec_t) out_codec));
        vf_free(o);
        vo_pp_gamma.done(s);
        return ok ? 0 : -1;
}

}  // extern "C"
