// TEST INFRASTRUCTURE: the UNMODIFIED src/capture_filter/r12l_to_y416_fake.c, included where it lies under $(REF),
// with its static functions exposed to tests/test_logo_filters.py.
#include "capture_filter/r12l_to_y416_fake.c"

/// one task of the filter's thread pool over the whole frame, into the harness's `dst`
void ref_r12l_to_y416_task(int full_range, int width, int height, const unsigned char *src, unsigned char *dst)
{
        struct task_data d = { width, height, src, (uint16_t *) dst };
        if (full_range) {
                r12l_to_y416_full(&d);
        } else {
                r12l_to_y416_limited(&d);
        }
}

/// init() on cfg, then filter() on a tight R12L frame; the Y416 frame it returns is copied to `dst`.  0, or -2 where
/// init refuses cfg
int ref_r12l_to_y416_filter(const char *cfg, int width, int height, char *src, unsigned char *dst)
{
        void *st = NULL;
        if (init(NULL, cfg, &st) != 0) {
                return -2;
        }
        struct video_frame *f = vf_alloc(1);
        f->color_spec = R12L;
        f->interlacing = PROGRESSIVE;
        f->fps = 30;
        f->tiles[0].width = width;
        f->tiles[0].height = height;
        f->tiles[0].data = src;
        f->tiles[0].data_len = vc_get_linesize(width, R12L) * height;
        struct video_frame *o = filter(st, f);  // f has no dispose callback, so the harness keeps it and src
        memcpy(dst, o->tiles[0].data, o->tiles[0].data_len);
        VIDEO_FRAME_DISPOSE(o);
        vf_free(f);
        done(st);
        return 0;
}
