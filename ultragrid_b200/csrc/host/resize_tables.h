// Per-geometry tables of the resize filter's resampling (DESIGN.md §2 "Resize"), computed once per input descriptor on
// the host and read by resize_kernels.cu.  resize_tables.cpp is compiled with -ffp-contract=off: every float / double
// operation below is one IEEE operation, as the contract states it.
#pragma once
#include <stdint.h>

namespace ugb_resize {

// one destination column or row: source positions s0, s1 and their weights w0, w1 (Q11 ints for 8-bit frames, float
// bits for RG48); nearest uses s0 only
struct Tap2 {
        int32_t s0, s1, w0, w1;
};

// nearest: s0 = min(floor(d * (1 / inv_scale)), n_src - 1), in double
void nearest_table(int n_src, int n_dst, double inv_scale, Tap2 *t);
// linear: f = (float) ((d + 0.5) * scale - 0.5), s = floor(f), f -= s (float), scale = 1 / inv_scale.  Columns
// (zero_frac) set s = 0, f = 0 where s < 0 and s = n_src - 1, f = 0 where s >= n_src - 1; rows keep f and clamp both
// positions into [0, n_src - 1].  Weights cvRound((1.0f - f) * 2048), cvRound(f * 2048), or the floats 1.0f - f, f.
void linear_table(int n_src, int n_dst, double inv_scale, bool zero_frac, bool float_weights, Tap2 *t);
// area: k when scale = 1 / inv_scale is within DBL_EPSILON of an integer k >= 1 and n_dst * k <= n_src, else 0
int area_factor(int n_src, int n_dst, double inv_scale);

}  // namespace ugb_resize
