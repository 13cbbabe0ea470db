// TEST INFRASTRUCTURE: the UNMODIFIED src/capture_filter/logo.c, included where it lies under $(REF), with its
// static functions exposed to tests/test_logo_filters.py.  The harness owns the frame (with slack after it: the
// decoder reads past the logo's span, past the frame on its last row).
#include "capture_filter/logo.c"

// module registration constructors (of all the logo shims): nothing to register with here
void register_library(const char *name, const void *info, enum library_class cls, int abi, enum mod_visibility_flag flag)
{
        (void) name, (void) info, (void) cls, (void) abi, (void) flag;
}

/// init() on "<file>[:<x>[:<y>]]": the state, or NULL where init refuses cfg
void *ref_logo_init(const char *cfg)
{
        void *st = NULL;
        return init(NULL, cfg, &st) == 0 ? st : NULL;
}

/// the state init() left: {width, height, x, y}; the logo's RGBA bytes into `rgba` when it is not NULL
void ref_logo_state(void *state, int *geom, unsigned char *rgba)
{
        struct state_capture_filter_logo *s = state;
        geom[0] = (int) s->width;
        geom[1] = (int) s->height;
        geom[2] = s->x;
        geom[3] = s->y;
        if (rgba != NULL) {
                memcpy(rgba, s->logo, 4 * (size_t) s->width * s->height);
        }
}

/// a state as init() makes it, from a logo already in memory (copied)
void *ref_logo_make(const unsigned char *rgba, unsigned width, unsigned height, int x, int y)
{
        struct state_capture_filter_logo *s = calloc(1, sizeof *s);
        s->logo = malloc(4 * (size_t) width * height);
        memcpy(s->logo, rgba, 4 * (size_t) width * height);
        s->width = width;
        s->height = height;
        s->x = x;
        s->y = y;
        return s;
}

void ref_logo_done(void *state) { done(state); }

/// filter() in place on a codec frame of width x height at `data`: 0, or 1 where it finds no decoder or coder
int ref_logo_filter(void *state, int codec, int width, int height, char *data)
{
        struct video_frame *f = vf_alloc(1);
        f->color_spec = (codec_t) codec;
        f->interlacing = PROGRESSIVE;
        f->fps = 30;
        f->tiles[0].width = width;
        f->tiles[0].height = height;
        f->tiles[0].data = data;
        f->tiles[0].data_len = vc_get_linesize(width, (codec_t) codec) * height;
        const int rc = get_decoder_from_to((codec_t) codec, RGB) != NULL && get_decoder_from_to(RGB, (codec_t) codec) != NULL ? 0 : 1;
        struct video_frame *o = filter(state, f);
        assert(o == f);
        vf_free(f);
        return rc;
}
