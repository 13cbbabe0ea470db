// Resampling tables of the resize filter; see resize_tables.h.  Built with -ffp-contract=off (csrc/Makefile).
#include "resize_tables.h"

#include <cfloat>
#include <cmath>
#include <cstring>

namespace ugb_resize {

static int32_t float_bits(float f)
{
        int32_t i;
        std::memcpy(&i, &f, sizeof i);
        return i;
}

static int clampi(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

void nearest_table(int n_src, int n_dst, double inv_scale, Tap2 *t)
{
        const double ifs = 1. / inv_scale;
        for (int d = 0; d < n_dst; ++d) {
                const int s = (int) std::floor(d * ifs);
                t[d] = Tap2{ s < n_src - 1 ? s : n_src - 1, 0, 0, 0 };
        }
}

void linear_table(int n_src, int n_dst, double inv_scale, bool zero_frac, bool float_weights, Tap2 *t)
{
        const double scale = 1. / inv_scale;
        for (int d = 0; d < n_dst; ++d) {
                float f = (float) ((d + 0.5) * scale - 0.5);
                int s = (int) std::floor(f);
                f -= (float) s;
                int s1 = s + 1;
                if (zero_frac) {
                        if (s < 0) {
                                s = 0, f = 0.f;
                        }
                        if (s >= n_src - 1) {
                                s = n_src - 1, f = 0.f;
                        }
                        s1 = s + 1 < n_src ? s + 1 : n_src - 1;
                } else {
                        s1 = clampi(s1, 0, n_src - 1);
                        s = clampi(s, 0, n_src - 1);
                }
                const float c0 = 1.0f - f, c1 = f;
                if (float_weights) {
                        t[d] = Tap2{ s, s1, float_bits(c0), float_bits(c1) };
                } else {  // cvRound: nearest, ties to even (the default rounding mode)
                        t[d] = Tap2{ s, s1, (int32_t) std::nearbyint(c0 * 2048.0f), (int32_t) std::nearbyint(c1 * 2048.0f) };
                }
        }
}

int area_factor(int n_src, int n_dst, double inv_scale)
{
        const double scale = 1. / inv_scale;
        const int k = (int) std::round(scale);
        if (k < 1 || !(std::fabs(scale - k) < DBL_EPSILON) || (long) n_dst * k > n_src) {
                return 0;
        }
        return k;
}

}  // namespace ugb_resize
