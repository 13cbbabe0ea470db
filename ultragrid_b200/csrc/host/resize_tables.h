// Per-geometry tables of the resize filter's resampling (DESIGN.md §2 "Resize"), computed once per input descriptor on
// the host and read by resize_kernels.cu.  resize_tables.cpp is compiled with -ffp-contract=off: every float / double
// operation below is one IEEE operation, as the contract states it.
#pragma once
#include <stdint.h>

#include <vector>

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
// linear with area-mode positions (area upscaling): s = floor(d * scale), f = (float) ((d + 1) - (s + 1) * inv_scale),
// f = f <= 0 ? 0 : f - floor(f); then clamps and weights as linear_table
void linear_area_table(int n_src, int n_dst, double inv_scale, bool zero_frac, bool float_weights, Tap2 *t);
// cubic (K = 4) and lanczos4 (K = 8): per destination K + 1 int32, the first tap s - K / 2 + 1 (unclamped; tap j is
// clamp(first + j)) and K weights, saturate_cast<short>(w * 2048) or float bits.  f as linear_table, never zeroed.
void cubic_table(int n_dst, double inv_scale, bool float_weights, int32_t *t);
void lanczos4_table(int n_dst, double inv_scale, bool float_weights, int32_t *t);
// computeResizeAreaTab: head holds (offset, count) per destination into ent, which holds (source index, float bits
// of alpha) per entry
void area_tab(int n_src, int n_dst, double scale, std::vector<int32_t> &head, std::vector<int32_t> &ent);
// area: k when scale = 1 / inv_scale is within DBL_EPSILON of an integer k >= 1 and n_dst * k <= n_src, else 0
int area_factor(int n_src, int n_dst, double inv_scale);

}  // namespace ugb_resize
