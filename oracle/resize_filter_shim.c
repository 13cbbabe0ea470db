// TEST INFRASTRUCTURE: the UNMODIFIED src/capture_filter/resize.c, included where it lies under $(REF), with its static
// functions exposed to tests/test_resize_filter.py.  resize_utils.cpp needs OpenCV, so this file defines the two
// functions resize.c takes from it: resize_frame records what the filter hands it, and resize_algo_from_string maps
// the five names of its interp_map (and `help`) to their cv::INTER_* values.
#include "capture_filter/resize.c"

// module registration constructors (the filter and its postprocessor wrapper): nothing to register with here
void register_library(const char *name, const void *info, enum library_class cls, int abi, enum mod_visibility_flag flag)
{
        (void) name, (void) info, (void) cls, (void) abi, (void) flag;
}

int resize_algo_from_string(const char *str)
{
        static const char *const names[] = { "nearest", "linear", "cubic", "area", "lanczos4" };
        static const int vals[] = { 0, 1, 2, 3, 4 };  // cv::INTER_NEAREST, _LINEAR, _CUBIC, _AREA, _LANCZOS4
        if (strcmp(str, "help") == 0) {
                return RESIZE_ALGO_HELP_SHOWN;
        }
        for (int i = 0; i < 5; ++i) {
                if (strcmp(names[i], str) == 0) {
                        return vals[i];
                }
        }
        return RESIZE_ALGO_UNKN;
}

// the last resize_frame call: in_color, width, height, mode, target_width, target_height, algo; factor; its input
static int last_i[7];
static double last_factor;
static unsigned char *last_bytes;
static size_t last_len;

void resize_frame(char *indata, codec_t in_color, char *outdata, int width, int height, struct resize_param *p)
{
        (void) outdata;
        const int v[7] = { in_color, width, height, p->mode, p->mode == USE_DIMENSIONS ? p->target_width : 0,
                           p->mode == USE_DIMENSIONS ? p->target_height : 0, p->algo };
        memcpy(last_i, v, sizeof v);
        last_factor = p->mode == USE_FRACTION ? p->factor : 0.;
        // the Mat ug_to_rgb_mat wraps: height * 3 / 2 rows of width bytes for I420, tight rows otherwise
        last_len = in_color == I420 ? (size_t) width * (height * 3 / 2) : (size_t) vc_get_linesize(width, in_color) * height;
        free(last_bytes);
        last_bytes = malloc(last_len);
        memcpy(last_bytes, indata, last_len);
}

/// init() on cfg: its return value; on 0, the state's resize_param as {mode, target_width, target_height, algo} and
/// factor, and the state itself in *state
int ref_resize_init(const char *cfg, void **state, int *param, double *factor)
{
        void *st = NULL;
        const int rc = init(NULL, cfg, &st);
        if (rc == 0) {
                const struct resize_param *p = &((struct state_resize *) st)->param;
                param[0] = p->mode;
                param[1] = p->mode == USE_DIMENSIONS ? p->target_width : 0;
                param[2] = p->mode == USE_DIMENSIONS ? p->target_height : 0;
                param[3] = p->algo;
                *factor = p->mode == USE_FRACTION ? p->factor : 0.;
                *state = st;
        }
        return rc;
}

void ref_resize_done(void *state) { done(state); }

/// filter() on a codec frame of width x height at `data` (the harness's, with slack after it).  1 where it drops the
/// frame; 0 otherwise, with out = {out codec, out width, out height, data_len, in_color, width, height, mode,
/// target_width, target_height, algo} (the last seven as resize_frame received them)
int ref_resize_filter(void *state, int codec, int width, int height, char *data, long *out)
{
        struct video_frame *f = vf_alloc(1);
        f->color_spec = (codec_t) codec;
        f->interlacing = PROGRESSIVE;
        f->fps = 30;
        f->tiles[0].width = width;
        f->tiles[0].height = height;
        f->tiles[0].data = data;
        f->tiles[0].data_len = vc_get_linesize(width, (codec_t) codec) * height;
        last_len = 0;
        struct video_frame *o = filter(state, f);  // f has no dispose callback: the harness keeps it
        vf_free(f);
        if (o == NULL) {
                return 1;
        }
        const long v[4] = { o->color_spec, o->tiles[0].width, o->tiles[0].height, o->tiles[0].data_len };
        for (int i = 0; i < 4; ++i) {
                out[i] = v[i];
        }
        for (int i = 0; i < 7; ++i) {
                out[4 + i] = last_i[i];
        }
        VIDEO_FRAME_DISPOSE(o);
        return 0;
}

/// the factor and input bytes of the last resize_frame call; returns their length
long ref_resize_last(double *factor, unsigned char *bytes, long cap)
{
        *factor = last_factor;
        if (bytes != NULL) {
                memcpy(bytes, last_bytes, (size_t) cap < last_len ? (size_t) cap : last_len);
        }
        return (long) last_len;
}
