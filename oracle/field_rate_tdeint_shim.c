// TEST INFRASTRUCTURE: the UNMODIFIED src/vo_postprocess/temporal-deint.c, included where it lies under $(REF), with
// its static functions exposed to tests/test_field_rate.py (double_framerate, deinterlace_bob, deinterlace_linear).
// The harness owns every buffer: perform_* and avg_lines write past the frame for some codecs (R10k: 4 x linesize).
#include "vo_postprocess/temporal-deint.c"

// tools/ug_stub.c has get_commandline_param only; init_common sets the drop policy for `nodelay`
void set_commandline_param(const char *key, const char *val)
{
        (void) key, (void) val;
}

// module registration constructors (of both shims): nothing to register with here
void register_library(const char *name, const void *info, enum library_class cls, int abi, enum mod_visibility_flag flag)
{
        (void) name, (void) info, (void) cls, (void) abi, (void) flag;
}

static struct video_frame *frame_on(int codec, int width, int height, void *data)
{
        struct video_frame *f = vf_alloc(1);
        f->color_spec = (codec_t) codec;
        f->interlacing = INTERLACED_MERGED;
        f->fps = 50;
        f->tiles[0].width = width;
        f->tiles[0].height = height;
        f->tiles[0].data = data;
        f->tiles[0].data_len = vc_get_linesize(width, (codec_t) codec) * height;
        return f;
}

/// one perform_df / perform_bob / perform_linear call: algo 0 DF, 1 bob, 2 linear; call 0 is postprocess(in = frame),
/// call 1 postprocess(in = NULL); cur is the frame just received, prev the one before
void ref_tdi_perform(int algo, int codec, int width, int height, char *prev, char *cur, int call, int deinterlace, char *out, int pitch)
{
        struct state_df s = { 0 };
        s.algo = (enum algo) algo;
        s.in = frame_on(codec, width, height, cur);
        s.buffers[0] = cur;
        s.buffers[1] = prev;
        s.buffer_current = 0;
        s.deinterlace = deinterlace != 0;
        struct video_frame *o = frame_on(codec, width, height, out);
        struct video_frame *in = call == 0 ? s.in : NULL;
        switch (s.algo) {
        case DF: perform_df(&s, in, o, pitch); break;
        case BOB: perform_bob(&s, in, o, pitch); break;
        case LINEAR: perform_linear(&s, in, o, pitch); break;
        }
        vf_free(o);
        vf_free(s.in);
}

/// avg_lines at a raw line size; returns whether it averaged (false: the caller copies)
int ref_tdi_avg_lines(int codec, size_t linesize, char *src1, char *src2, char *dst)
{
        return avg_lines((codec_t) codec, linesize, src1, src2, dst);
}

/// the module's own init / reconfigure / getf / postprocess over n merged frames, both calls each: out holds 2n frames
/// at pitch `pitch`.  cfg is the module option (`nodelay`, so postprocess does not wait half a frame time).
int ref_tdi_sequence(int algo, const char *cfg, int codec, int width, int height, const char *frames, int n, char *out, int pitch)
{
        const struct vo_postprocess_info *info = algo == DF ? &vo_pp_df_info : algo == BOB ? &vo_pp_bob_info : &vo_pp_linear_info;
        void *s = info->init(cfg);
        if (s == NULL) {
                return -1;
        }
        struct video_desc desc = { .width = width, .height = height, .color_spec = (codec_t) codec, .interlacing = INTERLACED_MERGED,
                                   .fps = 50, .tile_count = 1 };
        info->reconfigure(s, desc);
        const size_t fsz = (size_t) vc_get_linesize(width, (codec_t) codec) * height;
        const size_t osz = (size_t) pitch * height;
        int rc = 0;
        for (int i = 0; i < n; ++i) {
                struct video_frame *in = info->getf(s);
                memcpy(in->tiles[0].data, frames + i * fsz, fsz);
                for (int call = 0; call < 2; ++call) {
                        struct video_frame *o = frame_on(codec, width, height, out + (2 * i + call) * osz);
                        if (!info->vo_postprocess(s, call == 0 ? in : NULL, o, pitch)) {
                                rc = -1;
                        }
                        vf_free(o);
                }
        }
        info->done(s);
        return rc;
}
