// TEST INFRASTRUCTURE: the UNMODIFIED src/vo_postprocess/y416_to_r12l_fake.c, included where it lies under $(REF),
// with its static functions exposed to tests/test_logo_filters.py.
#include "vo_postprocess/y416_to_r12l_fake.c"

// tv.c and text.c are not in _ref/libugref.so.  The two pass-through filters (both shims) only time themselves for a
// debug message and print wrapped help text: a clock of 0 and no help text change none of their bytes.
time_ns_t get_time_in_ns(void) { return 0; }
void color_printf_wrapped(const char *text) { (void) text; }

/// one task over the whole frame: row y at y * pitch of the harness's `dst`
void ref_y416_to_r12l_task(int full_range, int width, int height, const unsigned char *src, unsigned char *dst, int pitch)
{
        struct task_data d = { width, height, (const uint16_t *) src, dst, pitch };
        if (full_range) {
                y416_to_r12l_full(&d);
        } else {
                y416_to_r12l_limited(&d);
        }
}

/// init() on cfg, reconfigure, then postprocess() of a tight Y416 frame into `dst` at req_pitch.  0, -1 (postprocess
/// failed) or -2 (init refused cfg)
int ref_y416_to_r12l_postprocess(const char *cfg, int width, int height, char *src, char *dst, int req_pitch)
{
        void *st = init(cfg);
        if (st == NULL || st == INIT_NOERR) {
                return -2;
        }
        ((struct state_vopp_y416_to_r12l_fake *) st)->f = NULL;  // init leaves it unset; reconfigure frees it
        struct video_desc desc = { .width = width, .height = height, .color_spec = Y416, .interlacing = PROGRESSIVE,
                                   .fps = 30, .tile_count = 1 };
        reconfigure(st, desc);
        struct video_frame *f = vf_alloc_desc(desc);
        f->tiles[0].data = src;
        desc.color_spec = R12L;
        struct video_frame *o = vf_alloc_desc(desc);
        o->tiles[0].data = dst;
        const bool ok = postprocess(st, f, o, req_pitch);
        vf_free(o);
        vf_free(f);
        done(st);
        return ok ? 0 : -1;
}
