// Resampling tables of the resize filter; see resize_tables.h.  Built with -ffp-contract=off (csrc/Makefile).
#include "resize_tables.h"

#include <cfloat>
#include <cmath>
#include <cstring>

#include <algorithm>

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

// one linear entry from the source position s and the fraction f (DESIGN.md §2 "Resize")
static Tap2 linear_entry(int n_src, int s, float f, bool zero_frac, bool float_weights)
{
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
                return Tap2{ s, s1, float_bits(c0), float_bits(c1) };
        }  // cvRound: nearest, ties to even (the default rounding mode)
        return Tap2{ s, s1, (int32_t) std::nearbyint(c0 * 2048.0f), (int32_t) std::nearbyint(c1 * 2048.0f) };
}

void linear_table(int n_src, int n_dst, double inv_scale, bool zero_frac, bool float_weights, Tap2 *t)
{
        const double scale = 1. / inv_scale;
        for (int d = 0; d < n_dst; ++d) {
                float f = (float) ((d + 0.5) * scale - 0.5);
                const int s = (int) std::floor(f);
                f -= (float) s;
                t[d] = linear_entry(n_src, s, f, zero_frac, float_weights);
        }
}

void linear_area_table(int n_src, int n_dst, double inv_scale, bool zero_frac, bool float_weights, Tap2 *t)
{
        const double scale = 1. / inv_scale;
        for (int d = 0; d < n_dst; ++d) {
                const int s = (int) std::floor(d * scale);
                float f = (float) ((d + 1) - (s + 1) * inv_scale);
                f = f <= 0 ? 0.f : f - (float) (int) std::floor(f);
                t[d] = linear_entry(n_src, s, f, zero_frac, float_weights);
        }
}

// interpolateCubic's weights, A = -0.75, each step one float operation
static void cubic_weights(float x, float *c)
{
        const float A = -0.75f;
        c[0] = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A;
        c[1] = ((A + 2) * x - (A + 3)) * x * x + 1;
        c[2] = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1;
        c[3] = 1.f - c[0] - c[1] - c[2];
}

// interpolateLanczos4's weights: the C library's sin and cos, normalised in float
static void lanczos4_weights(float x, float *c)
{
        static const double s45 = 0.70710678118654752440084436210485;
        static const double cs[8][2] = { { 1, 0 }, { -s45, -s45 }, { 0, 1 }, { s45, -s45 }, { -1, 0 }, { s45, s45 }, { 0, -1 }, { -s45, s45 } };
        const double y0 = -(x + 3) * M_PI * 0.25, s0 = std::sin(y0), c0 = std::cos(y0);
        float sum = 0;
        for (int i = 0; i < 8; ++i) {
                const float t = x + 3 - i;
                if (std::fabs(t) >= 1e-6f) {
                        const double y = -t * M_PI * 0.25;
                        c[i] = (float) ((cs[i][0] * s0 + cs[i][1] * c0) / (y * y));
                } else {
                        c[i] = 1e30f;
                }
                sum += c[i];
        }
        sum = 1.f / sum;
        for (int i = 0; i < 8; ++i) {
                c[i] *= sum;
        }
}

template <int K>
static void multitap_table(int n_dst, double inv_scale, bool float_weights, void (*weights)(float, float *), int32_t *t)
{
        const double scale = 1. / inv_scale;
        for (int d = 0; d < n_dst; ++d, t += K + 1) {
                float f = (float) ((d + 0.5) * scale - 0.5);
                const int s = (int) std::floor(f);
                f -= (float) s;
                float w[K];
                weights(f, w);
                t[0] = s - K / 2 + 1;
                for (int j = 0; j < K; ++j) {  // saturate_cast<short>(w * 2048): cvRound, then saturation
                        const float q = std::nearbyint(w[j] * 2048.0f);
                        t[1 + j] = float_weights ? float_bits(w[j]) : (int32_t) (q < -32768.f ? -32768.f : q > 32767.f ? 32767.f : q);
                }
        }
}

void cubic_table(int n_dst, double inv_scale, bool float_weights, int32_t *t)
{
        multitap_table<4>(n_dst, inv_scale, float_weights, cubic_weights, t);
}

void lanczos4_table(int n_dst, double inv_scale, bool float_weights, int32_t *t)
{
        multitap_table<8>(n_dst, inv_scale, float_weights, lanczos4_weights, t);
}

void area_tab(int n_src, int n_dst, double scale, std::vector<int32_t> &head, std::vector<int32_t> &ent)
{
        head.clear(), ent.clear();
        const auto add = [&](int s, float alpha) { ent.push_back(s), ent.push_back(float_bits(alpha)); };
        for (int d = 0; d < n_dst; ++d) {
                const double fs1 = d * scale, fs2 = fs1 + scale, cw = std::min(scale, n_src - fs1);
                int s1 = (int) std::ceil(fs1), s2 = (int) std::floor(fs2);
                s2 = std::min(s2, n_src - 1);
                s1 = std::min(s1, s2);
                head.push_back((int32_t) (ent.size() / 2));
                if (s1 - fs1 > 1e-3) {
                        add(s1 - 1, (float) ((s1 - fs1) / cw));
                }
                for (int s = s1; s < s2; ++s) {
                        add(s, (float) (1.0 / cw));
                }
                if (fs2 - s2 > 1e-3) {
                        add(s2, (float) (std::min(std::min(fs2 - s2, 1.), cw) / cw));
                }
                head.push_back((int32_t) (ent.size() / 2) - head.back());
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
