/* TEST INFRASTRUCTURE: the host functions the reference's tools/ug_stub.c supplies, for an UltraGrid started with `--param color-601`.
 * Linked in place of ug_stub.c into _ref/libugref601.so (color601.mk): get_default_cs() (src/color_space.c:186-191) then returns CS_601, so
 * every get_color_coeffs(CS_DFL, depth) of the unmodified objects gives the BT.601 set. */
#include <stdbool.h>
#include <stddef.h>
#include <string.h>

char *uv_argv[] = { "ug_stub", NULL };

const char *get_commandline_param(const char *key)
{
        return strcmp(key, "color-601") == 0 ? "" : NULL;  /* `--param color-601` has no value: the reference tests for non-NULL */
}

void register_param(const char *param, const char *doc)
{
        (void) param;
        (void) doc;
}

bool tok_in_argv(char **argv, const char *tok)
{
        (void) argv, (void) tok;
        return false;
}
