// Baseline JPEG decoder (include/ugb200_jpeg.h, decode part): the stage libgpujpeg performs for UltraGrid's
// src/video_decompress/gpujpeg.c:268-330 and gpujpeg_to_dxt.cpp:117-166 (SURVEY.md section 8f rank 1).
//
//   host   parse_stream     markers up to each SOS (tables, frame, scans) and ONE pass over the entropy-coded bytes that records
//                           where every restart segment starts (what GPUJPEG's reader does when the stream carries no segment info)
//   K0     jpeg_marker_*_kernel   the same segment table built on the device for the two regular stream shapes (one interleaved scan, or one scan
//                           per component): the host then only reads the headers in front of the first SOS
//   K1     jpeg_decode_huffman_kernel   one thread per restart segment: T.81 F.2.2 Huffman decoding with a 9-bit look-ahead
//                           table per Huffman table in shared memory (longer codes: min/max-code walk), DC prediction; every block is
//                           built in shared memory and written as 128 bytes into the int16 [block][64] buffer (or, when the scans do
//                           not cover every block, scattered into a cleared buffer)
//   K1'    jpeg_sync_table_kernel, jpeg_sync_kernel, jpeg_sync_write_kernel   instead of K1 for restart segments of at least kSyncMinMcus MCUs
//                           (every scan without DRI): self-synchronising decoding, one thread per kSyncBytes of entropy-coded data, the same
//                           coefficients as K1 for any bytes (both use jpeg_huffman_step.cuh; see the comment above jpeg_sync_kernel)
//   K2     jpeg_idct_kernel one thread per 8x8 block: dequantise, float AAN inverse DCT (fixed operation order = bit-exact with
//                           oracle/jpeg_decode_oracle.c), level shift, clamp, 8 x 8-byte stores into the component plane
//   K2'    jpeg_idct_packed_kernel  instead of K2 for 4:2:2 and 4:2:0 YCbCr: the IDCT of an MCU row's blocks into a shared tile, chroma replicated
//                           from its pair or quad, and the UYVY words stored as UYVY or handed to a line converter functor (yuv_rgb_conv.cuh):
//                           UltraGrid's UYVY -> RGB / RGBA, or the integer YCbCr -> RGB of a colour space (ugb200_jpeg_decode_cs); no planes.
//                           With ugb200_jpeg_decoder_set_upsampling(FANCY), RGB / RGBA in a colour space: libjpeg's interpolated chroma instead
//                           (epi_fancy; the halo of neighbouring chroma blocks is IDCT'd in the kernel)
//   pack   the component planes of K2 go through the from_planar kernels that already exist (planar_conv_kernels.cu): 4:4:4 YCbCr -> VUYA
//                           (yuv444p_to_vuya), RGB -> RGB (rgbpXX_to_rgb), R G B A (gbrap_to_rgba); then ugb200_pixfmt_convert when another
//                           output codec was asked for (also from K2's UYVY to VUYA / I420).  4:4:4 YCbCr in a colour space: jpeg_planes_cs_kernel.
// Restart intervals are the unit of parallelism of K1; K1' does not depend on them.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <emmintrin.h>

#include <algorithm>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <chrono>
#include <cstdio>
#include <new>
#include <thread>
#include <type_traits>
#include <vector>

#include "../../include/ugb200.h"
#include "../../include/ugb200_jpeg.h"
#include "jpeg_marker_bounds.cuh"
#include "jpeg_huffman_step.cuh"
#include "yuv_rgb_conv.cuh"
#include "../../include/cuda_wrapper.h"

#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace ugb {

static const uint8_t kZigzag[64] = { 0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 };

struct bit_reader {  // MSB-first, removes stuffed zero bytes, feeds zeros beyond `end`
        const uint8_t *p, *end;
        uint64_t acc;
        int nbits;
        // the two aligned words that hold bytes p .. p + 3, fetched one refill AHEAD of their use: the thread's next four bytes are already in registers when
        // it needs them (ncu of the byte-wise reader: `long_scoreboard` on top of the stall list - every refill waited for its own loads with ~13 warps per SM)
        const uint32_t *wa;
        uint32_t w0, w1;
        /// the stream buffer is 16 bytes longer than the stream: the aligned loads around any p <= end stay inside the allocation
        __device__ __forceinline__ void prime()
        {
                wa = (const uint32_t *) ((size_t) p & ~(size_t) 3);
                w0 = __ldg(wa), w1 = __ldg(wa + 1);
        }
        /// after the call at least 33 bits are valid (code of up to 16 bits + up to 15 value bits), zeros beyond `end`.
        /// Fast path: four stream bytes at once when none of them is 0xFF (entropy-coded data holds one 0xFF in ~256 bytes).
        __device__ __forceinline__ void refill()
        {
                if (nbits > 32) {
                        return;
                }
                if (p + 4 <= end) {
                        const uint32_t le = __funnelshift_r(w0, w1, 8 * (unsigned) ((size_t) p & 3));  // bytes p[0..3], p[0] lowest
                        if (__vcmpeq4(le, 0xffffffffu) == 0) {
                                acc |= (uint64_t) __byte_perm(le, 0, 0x0123) << (32 - nbits);
                                nbits += 32, p += 4;
                                ++wa, w0 = w1, w1 = __ldg(wa + 1);  // for the next refill
                                return;
                        }
                }
                while (nbits <= 56) {
                        uint32_t b = 0;
                        if (p < end) {
                                b = __ldg(p++);
                                if (b == 0xFF && p < end && __ldg(p) == 0) {
                                        ++p;
                                }
                        }
                        acc |= (uint64_t) b << (56 - nbits);
                        nbits += 8;
                }
                prime();
        }
        __device__ __forceinline__ uint32_t peek(int n) const { return (uint32_t) (acc >> (64 - n)); }
        __device__ __forceinline__ void skip(int n) { acc <<= n, nbits -= n; }
};

/// FULL: every block of the coefficient array is decoded by exactly one thread (the host checks: every component in a scan, the scans' MCU grids equal to the
/// padded planes) - the thread then builds its block in shared memory ([word][thread]: conflict-free, dynamically indexable) and writes all 128 bytes of it,
/// so the array needs no clearing beforehand (133 MB at 8K) and the scattered 2-byte stores become whole-line stores.  !FULL: sparse stores into a cleared array.
/// kHuffThreads: an 8K UYVY frame has 64 800 restart segments = threads, all resident at once; with 128-thread CTAs that is 3.4 CTAs per SM (some SMs run four, the
/// kernel lasts as long as those), with 64-thread CTAs 6.8 (seven against six)
constexpr int kHuffThreads = 64;
/// block-wide copy of `bytes` (a multiple of 4) between 4-byte aligned addresses
__device__ __forceinline__ void copy_words(void *dst, const void *src, int bytes)
{
        for (int i = threadIdx.x; i < bytes / 4; i += blockDim.x) {
                ((uint32_t *) dst)[i] = ((const uint32_t *) src)[i];
        }
}
/// what the Huffman kernels read of the tables: the slots in use and the zig-zag order (not the dequantisation multipliers)
__device__ __forceinline__ void copy_tables(dec_tables *t, const dec_tables *tables, int ntables)
{
        copy_words(t->lut, tables->lut, ntables * (int) sizeof t->lut[0]);
        copy_words(t->maxcode, tables->maxcode, ntables * (int) sizeof t->maxcode[0]);
        copy_words(t->valoff, tables->valoff, ntables * (int) sizeof t->valoff[0]);
        copy_words(t->vals, tables->vals, ntables * (int) sizeof t->vals[0]);
        copy_words(t->zz, tables->zz, (int) sizeof t->zz);
}
constexpr size_t kTablesSmem = (sizeof(dec_tables) + 15) & ~(size_t) 15;

/// where decode_block puts a block: FULL - the thread's column of shared memory, written out as 128 bytes by finish(); !FULL - the non-zero coefficients
/// straight into the cleared array.  Padding blocks of an MCU (`inside` false) are decoded and not stored.
template <bool FULL>
struct block_sink {
        uint32_t *col;
        int16_t *blk;
        const uint8_t *zz;
        bool inside;
        __device__ __forceinline__ void begin()
        {
                if (FULL) {
#pragma unroll
                        for (int w = 0; w < 32; ++w) {
                                col[w * kHuffThreads] = 0;
                        }
                }
        }
        __device__ __forceinline__ void dc(uint32_t pred)
        {
                if (FULL) {
                        col[0] = pred & 0xffffu;
                } else if (inside && pred != 0) {
                        blk[0] = (int16_t) pred;
                }
        }
        __device__ __forceinline__ void operator()(int i, int v)
        {
                const int n = zz[i];
                if (FULL) {
                        ((int16_t *) (col + (n >> 1) * kHuffThreads))[n & 1] = (int16_t) v;
                } else if (inside) {
                        blk[n] = (int16_t) v;
                }
        }
        __device__ __forceinline__ void finish()
        {
                if (FULL && inside) {
#pragma unroll
                        for (int q = 0; q < 8; ++q) {
                                ((uint4 *) blk)[q] = make_uint4(col[(4 * q) * kHuffThreads], col[(4 * q + 1) * kHuffThreads], col[(4 * q + 2) * kHuffThreads], col[(4 * q + 3) * kHuffThreads]);
                        }
                }
        }
};

/// the scan of restart segment `s` (with the table selectors the device read for the later scans of a multi-scan stream) and its MCUs [m0, m1)
__device__ __forceinline__ bool segment_scan(const dec_geom &g, int s, const uint32_t *__restrict__ dev_scans, dec_scan &S, int &m0, int &m1)
{
        int sc = 0;
        while (sc < g.nscans && s >= g.s[sc].seg0 + g.s[sc].nseg) {
                ++sc;
        }
        if (sc >= g.nscans) {
                return false;
        }
        S = g.s[sc];
        if (dev_scans != nullptr && sc > 0) {  // multi-scan stream with the marker scan on the device: the SOS headers of the later scans were read there
                S.td[0] = (int) dev_scans[kMetaBounds + 6 * sc + 4], S.ta[0] = 2 + (int) dev_scans[kMetaBounds + 6 * sc + 5];  // no DHT between the scans
        }
        const int ls = s - S.seg0;
        m0 = g.ri ? ls * g.ri : 0, m1 = g.ri ? min(m0 + g.ri, S.nmcu) : S.nmcu;
        return true;
}

template <bool FULL>
__global__ void __launch_bounds__(kHuffThreads) jpeg_decode_huffman_kernel(const uint8_t *__restrict__ stream, const uint32_t *__restrict__ seg_begin,
                                                                  const uint32_t *__restrict__ seg_end, const dec_tables *__restrict__ tables,
                                                                  dec_geom g, int16_t *__restrict__ coef, const uint32_t *__restrict__ dev_scans)
{
        extern __shared__ uint8_t smem_raw[];
        dec_tables *t = (dec_tables *) smem_raw;
        uint32_t *const col = (uint32_t *) (smem_raw + kTablesSmem) + threadIdx.x;  // FULL: word w of my block at col[w * kHuffThreads]
        copy_tables(t, tables, g.ntables);
        __syncthreads();
        const int s = blockIdx.x * blockDim.x + threadIdx.x;
        dec_scan S;
        int m0, m1;
        if (!segment_scan(g, s, dev_scans, S, m0, m1)) {
                return;
        }
        bit_reader r = { stream + seg_begin[s], stream + seg_end[s], 0, 0, nullptr, 0, 0 };
        r.prime();
        uint32_t pred[4] = { 0, 0, 0, 0 };
        for (int m = m0; m < m1; ++m) {
                const int mx = m % S.mcux, my = m / S.mcux;
                for (int k = 0; k < S.ns; ++k) {
                        const dec_comp &c = g.c[S.comp[k]];
                        const int nh = S.ns == 1 ? 1 : c.h, nv = S.ns == 1 ? 1 : c.v;
                        for (int by = 0; by < nv; ++by) {
                                for (int bx = 0; bx < nh; ++bx) {
                                        const int X = mx * nh + bx, Y = my * nv + by;
                                        block_sink<FULL> sink = { col, coef + ((long) c.blk_off + (long) Y * c.bw + X) * 64, t->zz, X < c.bw && Y < c.bh };
                                        sink.begin();
                                        decode_block(r, t, S.td[k], S.ta[k], pred[k], sink);
                                        sink.finish();
                                }
                        }
                }
        }
}

// ---- the self-synchronising route (segments of many MCUs; every scan without DRI) -------------------------------------------------------------------
// A segment's bytes are cut into subsequences of `sub` bytes, one thread each (Weißenberger & Schmidt, ICPP 2018).  A subsequence's entry is the decoder
// state (bit address, block of the MCU, zig-zag position) at the first symbol boundary at or after its start.  The first subsequence of a segment knows its
// entry; the others start from a guess.
//   jpeg_sync_table_kernel  subsequences per segment (from the segment table, so the device marker scan needs no host round trip) and their prefix sum
//   jpeg_sync_kernel        cooperative grid.  Round r: every subsequence whose entry changed decodes from it to its exit - the first symbol boundary at or
//                           after the next subsequence's start - counting the blocks whose DC symbol starts inside and their DC differences per component
//                           (walk_count); an exit that differs from the next entry replaces it.  A round without a change ends the loop: then every
//                           entry is the exit of its predecessor, proved from the segment's start (after round r the first r + 1 are proved, so at most
//                           one round per subsequence).  Then an exclusive scan of the counts and sums over all subsequences (uint32, wrapping).
//   jpeg_sync_write_kernel  one thread per subsequence: from its proved entry, the rest of a block begun before (not stored), then every block whose DC
//                           symbol starts inside, each decoded whole (read past the end as far as it needs) with decode_block and stored as the
//                           restart-segment kernel stores it; block index and DC predictors = the scan minus the value at the segment's first subsequence.
//                           Blocks past the segment's MCUs are dropped; the last subsequence goes on into the zero tail until they are all there.
constexpr int kSyncThreads = 128;
/// subsequence length in bytes (the default; UGB200_JPEG_SYNC=on:<bytes> sets another at decoder creation): 64 B give an 8K q90 frame ~80 000
/// threads, about 60 % of what the cooperative grid holds at once; it is the only length timed so far (DESIGN.md section 4.1)
constexpr int kSyncBytes = 64;
constexpr int kSyncVals = 5;
/// restart intervals of at least this many MCUs take the self-synchronising route (chosen from tools/jpeg_nodri_bench.py, DESIGN.md section 4)
constexpr int kSyncMinMcus = 64;  // per subsequence: blocks, DC sums of the scan components 0..3

struct sync_bufs {
        uint32_t *sub_first;  // [nseg + 1]: first subsequence of each segment, total at [nseg]
        sync_point *entry, *exitp;
        uint32_t *res, *scan;  // [kSyncVals][nsub]
        uint32_t *dirty;       // entry changed in the last round
        uint32_t *cta;         // [kSyncVals][grid] CTA totals
        uint32_t *ctr;         // [3] changes per round (rotating), [3] rounds, [4] subsequences
};

__global__ void __launch_bounds__(1024) jpeg_sync_table_kernel(const uint32_t *__restrict__ seg_begin, const uint32_t *__restrict__ seg_end, int nseg, int sub,
                                                                 uint32_t *__restrict__ sub_first)
{
        __shared__ uint32_t s_w[32];
        __shared__ uint32_t s_carry;
        if (threadIdx.x == 0) {
                s_carry = 0;
        }
        __syncthreads();
        for (int base = 0; base < nseg; base += 1024) {
                const int i = base + (int) threadIdx.x;
                const uint32_t v = i < nseg ? (uint32_t) sub_count(seg_end[i] - seg_begin[i], sub) : 0;
                uint32_t incl = v;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                        const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
                        if ((threadIdx.x & 31) >= (unsigned) d) {
                                incl += o;
                        }
                }
                if ((threadIdx.x & 31) == 31) {
                        s_w[threadIdx.x >> 5] = incl;
                }
                __syncthreads();
                uint32_t before = s_carry;
                for (int w = 0; w < (int) (threadIdx.x >> 5); ++w) {
                        before += s_w[w];
                }
                if (i < nseg) {
                        sub_first[i] = before + incl - v;
                }
                __syncthreads();
                if (threadIdx.x == 1023) {
                        s_carry = before + incl;
                }
                __syncthreads();
        }
        if (threadIdx.x == 0) {
                sub_first[nseg] = s_carry;
        }
}

/// the segment of subsequence j: the last one whose first subsequence is <= j
__device__ __forceinline__ int sub_segment(const uint32_t *__restrict__ sub_first, int nseg, uint32_t j)
{
        int lo = 0, hi = nseg - 1;
        while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (sub_first[mid] <= j) {
                        lo = mid;
                } else {
                        hi = mid - 1;
                }
        }
        return lo;
}

__device__ __forceinline__ bool same_point(sync_point a, sync_point b) { return a.byte == b.byte && a.tag == b.tag; }

__global__ void __launch_bounds__(kSyncThreads, 8) jpeg_sync_kernel(const uint8_t *__restrict__ stream, const uint32_t *__restrict__ seg_begin,
                                                                 const uint32_t *__restrict__ seg_end, int nseg, int sub, const dec_tables *__restrict__ tables,
                                                                 dec_geom g, const uint32_t *__restrict__ dev_scans, sync_bufs B, uint32_t cap)
{
        extern __shared__ uint8_t smem_raw[];
        dec_tables *t = (dec_tables *) smem_raw;
        __shared__ uint32_t s_w[kSyncThreads / 32][kSyncVals];
        __shared__ uint32_t s_pre[kSyncVals];
        copy_tables(t, tables, g.ntables);
        if (threadIdx.x < kSyncVals) {
                s_pre[threadIdx.x] = 0;
        }
        __syncthreads();
        cg::grid_group grid = cg::this_grid();
        const uint32_t nsub = min(B.sub_first[nseg], cap);
        const uint32_t nthreads = gridDim.x * blockDim.x, gt = blockIdx.x * blockDim.x + threadIdx.x;
        const uint32_t per = (nsub + nthreads - 1) / nthreads, j0 = min(nsub, gt * per), j1 = min(nsub, j0 + per);
        // contiguous subsequences per thread: the same ones in every round and in the scan
        for (uint32_t j = j0; j < j1; ++j) {
                const int s = sub_segment(B.sub_first, nseg, j);
                const uint32_t f = B.sub_first[s];
                B.entry[j] = make_point(sub_start(stream, seg_begin[s], seg_end[s], (int) (j - f), sub), 0, 0);
                B.dirty[j] = 1;
                for (int v = 0; v < kSyncVals; ++v) {
                        B.res[v * cap + j] = 0;
                }
        }
        int round = 0;
        for (;; ++round) {
                if (gt == 0) {
                        B.ctr[(round + 1) % 3] = 0;
                }
                for (uint32_t j = j0; j < j1; ++j) {
                        const int s = sub_segment(B.sub_first, nseg, j);
                        if (!B.dirty[j] || j + 1 == B.sub_first[s + 1]) {
                                continue;  // the entry is unchanged, or the last subsequence of its segment (it proves nothing)
                        }
                        dec_scan S;
                        int m0, m1;
                        segment_scan(g, s, dev_scans, S, m0, m1);
                        const mcu_layout L = layout_of(g, S);
                        const sync_point e = B.entry[j];
                        pos_reader r;
                        r.s = stream, r.end = seg_end[s];
                        r.start(e.byte, (int) (e.tag >> 16));
                        int blk = (e.tag >> 8) & 0xff, zz = e.tag & 0xff;
                        uint32_t count = 0, sum[4] = { 0, 0, 0, 0 };
                        const uint64_t limit = sub_start(stream, seg_begin[s], seg_end[s], (int) (j + 1 - B.sub_first[s]), sub);
                        walk_count(r, t, S.td, S.ta, L, limit, blk, zz, count, sum);
                        B.exitp[j] = make_point(r.pos(), blk, zz);
                        B.res[j] = count;
                        for (int v = 0; v < 4; ++v) {
                                B.res[(v + 1) * cap + j] = sum[v];
                        }
                }
                grid.sync();
                uint32_t changed = 0;
                for (uint32_t j = j0; j < j1; ++j) {
                        const int s = sub_segment(B.sub_first, nseg, j);
                        if (j == B.sub_first[s]) {
                                B.dirty[j] = 0;  // its entry is the segment's start
                        }
                        if (j + 1 == B.sub_first[s + 1]) {
                                continue;
                        }
                        // an exit not recomputed this round equals the next entry already: the owner of j + 1 reads dirty[j + 1] only after the grid sync
                        const bool moved = !same_point(B.exitp[j], B.entry[j + 1]);
                        if (moved) {
                                B.entry[j + 1] = B.exitp[j];
                        }
                        B.dirty[j + 1] = moved;
                        changed += moved;
                }
                if (changed) {
                        atomicAdd(B.ctr + round % 3, changed);
                }
                grid.sync();
                if (B.ctr[round % 3] == 0) {
                        break;
                }
        }
        // exclusive scan of res over all subsequences: thread totals -> CTA -> grid
        uint32_t tot[kSyncVals] = { 0, 0, 0, 0, 0 };
        for (uint32_t j = j0; j < j1; ++j) {
                for (int v = 0; v < kSyncVals; ++v) {
                        tot[v] += B.res[v * cap + j];
                }
        }
        uint32_t incl[kSyncVals];
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
        for (int v = 0; v < kSyncVals; ++v) {
                incl[v] = tot[v];
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                        const uint32_t o = __shfl_up_sync(0xffffffffu, incl[v], d);
                        if (lane >= d) {
                                incl[v] += o;
                        }
                }
                if (lane == 31) {
                        s_w[warp][v] = incl[v];
                }
        }
        __syncthreads();
        if (threadIdx.x < kSyncVals) {
                uint32_t c = 0;
                for (int w = 0; w < kSyncThreads / 32; ++w) {
                        c += s_w[w][threadIdx.x];
                }
                B.cta[threadIdx.x * gridDim.x + blockIdx.x] = c;
        }
        grid.sync();
        for (int v = 0; v < kSyncVals; ++v) {
                uint32_t c = 0;
                for (uint32_t b = threadIdx.x; b < blockIdx.x; b += blockDim.x) {
                        c += B.cta[v * gridDim.x + b];
                }
                if (c) {
                        atomicAdd(s_pre + v, c);
                }
        }
        __syncthreads();
        uint32_t run[kSyncVals];
#pragma unroll
        for (int v = 0; v < kSyncVals; ++v) {
                run[v] = s_pre[v] + incl[v] - tot[v];
                for (int w = 0; w < warp; ++w) {
                        run[v] += s_w[w][v];
                }
        }
        for (uint32_t j = j0; j < j1; ++j) {
                for (int v = 0; v < kSyncVals; ++v) {
                        B.scan[v * cap + j] = run[v];
                        run[v] += B.res[v * cap + j];
                }
        }
        if (gt == 0) {
                B.ctr[3] = (uint32_t) round + 1, B.ctr[4] = nsub;
        }
}

template <bool FULL>
__global__ void __launch_bounds__(kHuffThreads, 16) jpeg_sync_write_kernel(const uint8_t *__restrict__ stream, const uint32_t *__restrict__ seg_begin,
                                                                     const uint32_t *__restrict__ seg_end, int nseg, int sub, const dec_tables *__restrict__ tables,
                                                                     dec_geom g, int16_t *__restrict__ coef, const uint32_t *__restrict__ dev_scans, sync_bufs B,
                                                                     uint32_t cap)
{
        extern __shared__ uint8_t smem_raw[];
        dec_tables *t = (dec_tables *) smem_raw;
        uint32_t *const col = (uint32_t *) (smem_raw + kTablesSmem) + threadIdx.x;
        copy_tables(t, tables, g.ntables);
        __syncthreads();
        const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
        if (j >= min(B.sub_first[nseg], cap)) {
                return;
        }
        const int s = sub_segment(B.sub_first, nseg, j);
        dec_scan S;
        int m0, m1;
        if (!segment_scan(g, s, dev_scans, S, m0, m1)) {
                return;
        }
        const mcu_layout L = layout_of(g, S);
        const uint32_t f = B.sub_first[s], nblk = (uint32_t) (m1 - m0) * (uint32_t) L.bpm;
        uint32_t idx = B.scan[j] - B.scan[f], pred[4];
        for (int v = 0; v < 4; ++v) {
                pred[v] = B.scan[(v + 1) * cap + j] - B.scan[(v + 1) * cap + f];
        }
        if (idx >= nblk) {
                return;
        }
        const sync_point e = B.entry[j];
        pos_reader r;
        r.s = stream, r.end = seg_end[s];
        r.start(e.byte, (int) (e.tag >> 16));
        const int zz = e.tag & 0xff;
        if (zz) {
                finish_block(r, t, S.ta[L.k[(e.tag >> 8) & 0xff]], zz);
        }
        const bool last = j + 1 == B.sub_first[s + 1];
        const uint64_t limit = last ? ~(uint64_t) 0 : sub_start(stream, seg_begin[s], seg_end[s], (int) (j + 1 - f), sub);
        while (idx < nblk && r.pos() < limit) {
                const int m = m0 + (int) (idx / (uint32_t) L.bpm), b = (int) (idx % (uint32_t) L.bpm), k = L.k[b];
                const int mx = m % S.mcux, my = m / S.mcux;
                const dec_comp &c = g.c[S.comp[k]];
                const int nh = S.ns == 1 ? 1 : c.h, nv = S.ns == 1 ? 1 : c.v;
                const int X = mx * nh + L.bx[b], Y = my * nv + L.by[b];
                block_sink<FULL> sink = { col, coef + ((long) c.blk_off + (long) Y * c.bw + X) * 64, t->zz, X < c.bw && Y < c.bh };
                sink.begin();
                decode_block(r, t, S.td[k], S.ta[k], pred[k], sink);
                sink.finish();
                ++idx;
        }
}

__device__ __forceinline__ void idct8(float &d0, float &d1, float &d2, float &d3, float &d4, float &d5, float &d6, float &d7)
{
        const float e0 = __fadd_rn(d0, d4), e1 = __fadd_rn(d0, -d4);
        const float e3 = __fadd_rn(d2, d6), e2 = __fadd_rn(__fmul_rn(__fadd_rn(d2, -d6), 1.414213562f), -e3);
        const float a0 = __fadd_rn(e0, e3), a3 = __fadd_rn(e0, -e3), a1 = __fadd_rn(e1, e2), a2 = __fadd_rn(e1, -e2);
        const float z13 = __fadd_rn(d5, d3), z10 = __fadd_rn(d5, -d3), z11 = __fadd_rn(d1, d7), z12 = __fadd_rn(d1, -d7);
        const float b7 = __fadd_rn(z11, z13);
        const float b11 = __fmul_rn(__fadd_rn(z11, -z13), 1.414213562f);
        const float z5 = __fmul_rn(__fadd_rn(z10, z12), 1.847759065f);
        const float b10 = __fmaf_rn(1.082392200f, z12, -z5);
        const float b12 = __fmaf_rn(-2.613125930f, z10, z5);
        const float b6 = __fadd_rn(b12, -b7), b5 = __fadd_rn(b11, -b6), b4 = __fadd_rn(b10, b5);
        d0 = __fadd_rn(a0, b7), d7 = __fadd_rn(a0, -b7);
        d1 = __fadd_rn(a1, b6), d6 = __fadd_rn(a1, -b6);
        d2 = __fadd_rn(a2, b5), d5 = __fadd_rn(a2, -b5);
        d4 = __fadd_rn(a3, b4), d3 = __fadd_rn(a3, -b4);
}

__global__ void __launch_bounds__(128) jpeg_idct_kernel(const int16_t *__restrict__ coef, const dec_tables *__restrict__ tables, dec_geom g,
                                                        uint8_t *__restrict__ planes)
{
        __shared__ float s_m[4][64];
        for (int i = threadIdx.x; i < 256; i += blockDim.x) {
                s_m[i >> 6][i & 63] = tables->m[i >> 6][i & 63];
        }
        __syncthreads();
        const int b = blockIdx.x * blockDim.x + threadIdx.x;
        if (b >= g.nblocks) {
                return;
        }
        int ci = 0;
        while (ci + 1 < g.ncomp && b >= g.c[ci + 1].blk_off) {
                ++ci;
        }
        const dec_comp &c = g.c[ci];
        const int lb = b - c.blk_off, X = lb % c.bw, Y = lb / c.bw;
        const float *m = s_m[c.tq];
        float f[64];
        const uint4 *src = (const uint4 *) (coef + (long) b * 64);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
                const uint4 v = __ldg(src + q);
                const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
                for (int j = 0; j < 4; ++j) {  // int16 -> float without I2F: 1.5 * 2^23 + c is exact
                        const int lo = (int) (short) (w[j] & 0xffffu), hi = (int) w[j] >> 16;
                        f[8 * q + 2 * j] = __fmul_rn(__fadd_rn(__uint_as_float(0x4B400000u + (uint32_t) lo), -12582912.0f), m[8 * q + 2 * j]);
                        f[8 * q + 2 * j + 1] = __fmul_rn(__fadd_rn(__uint_as_float(0x4B400000u + (uint32_t) hi), -12582912.0f), m[8 * q + 2 * j + 1]);
                }
        }
#pragma unroll
        for (int col = 0; col < 8; ++col) {
                idct8(f[col], f[8 + col], f[16 + col], f[24 + col], f[32 + col], f[40 + col], f[48 + col], f[56 + col]);
        }
#pragma unroll
        for (int r = 0; r < 8; ++r) {
                idct8(f[8 * r], f[8 * r + 1], f[8 * r + 2], f[8 * r + 3], f[8 * r + 4], f[8 * r + 5], f[8 * r + 6], f[8 * r + 7]);
        }
        uint8_t *dst = planes + c.plane_off + ((long) Y * 8) * (c.bw * 8) + X * 8;
#pragma unroll
        for (int r = 0; r < 8; ++r) {
                uint32_t o[8];
#pragma unroll
                for (int x = 0; x < 8; ++x) {  // rintf(v + 128) through the 1.5 * 2^23 magic, clamp 0..255
                        const int v = (int) __float_as_uint(__fadd_rn(__fadd_rn(f[8 * r + x], 128.0f), 12582912.0f)) - 0x4B400000;
                        o[x] = (uint32_t) min(max(v, 0), 255);
                }
                *(uint2 *) (dst + (long) r * (c.bw * 8)) = make_uint2(o[0] | o[1] << 8 | o[2] << 16 | o[3] << 24, o[4] | o[5] << 8 | o[6] << 16 | o[7] << 24);
        }
}

/// UYVY output: the pixel pair words as they are, 16 bytes (8 pixels) per piece
struct epi_uyvy {
        static constexpr int PX = 8, OUT = 16, BPP = 2;
        static __device__ __forceinline__ void run(const uint32_t *w, uint32_t *o, const conv_params &) { o[0] = w[0], o[1] = w[1], o[2] = w[2], o[3] = w[3]; }
};
/// I420 output: the kernel writes the three planes from its tile (its planar epilogue); the constants only size the unused packed path
struct epi_i420 : epi_uyvy {};
/// RGB / RGBA output: a line converter functor (yuv_rgb_conv.cuh) applied to the UYVY words of 16 pixels, as ugb200_pixfmt_convert would apply it
/// to the UYVY frame
template <class C>
struct epi_conv {
        static constexpr int PX = 16, OUT = C::OUT * 32 / C::IN, BPP = OUT / 16;
        static __device__ __forceinline__ void run(const uint32_t *w, uint32_t *o, const conv_params &p)
        {
#pragma unroll
                for (int k = 0; k < 32 / C::IN; ++k) {
                        C::run(w + k * (C::IN / 4), o + k * (C::OUT / 4), p, row_ctx{});
                }
        }
};
using epi_rgb = epi_conv<conv_yuv422_rgb<1, 3, 0, 2>>;  // vc_copylineUYVYtoRGB = BT.709 limited range
using epi_rgba = epi_conv<conv_uyvy_rgba>;             // vc_copylineUYVYtoRGBA
template <class CS>
using epi_cs_rgb = epi_conv<conv_yuv422_rgb<1, 3, 0, 2, CS>>;
template <class CS>
using epi_cs_rgba = epi_conv<conv_yuv422_rgb<1, 3, 0, 2, CS, true>>;

/// RGB / RGBA output in a colour space with libjpeg's interpolated chroma (UGB200_JPEG_UPSAMPLE_FANCY): every pixel of the row, 16 per thread,
/// YCBCR_TO_R/G/B of its own luma and its own upsampled Cb, Cr (the integers of jpeg_planes_cs_kernel); staged like epi_conv
template <class CS, bool RGBA>
struct epi_fancy {
        static constexpr int PX = 16, BPP = RGBA ? 4 : 3, OUT = 16 * BPP;
        using cs = CS;
        static constexpr bool rgba = RGBA;
};
template <class E>
constexpr bool is_fancy = false;
template <class CS, bool RGBA>
constexpr bool is_fancy<epi_fancy<CS, RGBA>> = true;

/// FANCY: both chroma tiles of the CTA with their halo, rows -1..8 of the MCU row (4:2:2: rows 0..7 only) x columns -1..256 (byte 7 = column -1,
/// bytes 8..263 = the CTA's 256 columns, byte 264 = column 256; 16-byte rows)
constexpr int kFancyRow = 272;
__device__ __forceinline__ uint8_t (*fancy_chroma())[10][kFancyRow]
{
        __shared__ __align__(16) uint8_t s[2][10][kFancyRow];
        return s;
}

/// dequantisation and column pass of one block, the arithmetic of jpeg_idct_packed_kernel
__device__ __forceinline__ void idct_columns(const int16_t *__restrict__ blk, const float *mq, float *f)
{
        const uint4 *src = (const uint4 *) blk;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
                const uint4 v = __ldg(src + q);
                const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                        const int lo = (int) (short) (w[j] & 0xffffu), hi = (int) w[j] >> 16;
                        f[8 * q + 2 * j] = __fmul_rn(__fadd_rn(__uint_as_float(0x4B400000u + (uint32_t) lo), -12582912.0f), mq[8 * q + 2 * j]);
                        f[8 * q + 2 * j + 1] = __fmul_rn(__fadd_rn(__uint_as_float(0x4B400000u + (uint32_t) hi), -12582912.0f), mq[8 * q + 2 * j + 1]);
                }
        }
#pragma unroll
        for (int col = 0; col < 8; ++col) {
                idct8(f[col], f[8 + col], f[16 + col], f[24 + col], f[32 + col], f[40 + col], f[48 + col], f[56 + col]);
        }
}

/// row pass of row r after idct_columns: the 8 samples as jpeg_idct_packed_kernel stores them in its tile
__device__ __forceinline__ uint2 idct_row(const float *f, int r)
{
        float v[8];
#pragma unroll
        for (int x = 0; x < 8; ++x) {
                v[x] = f[8 * r + x];
        }
        idct8(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]);
        uint32_t o[8];
#pragma unroll
        for (int x = 0; x < 8; ++x) {
                const int s = (int) __float_as_uint(__fadd_rn(__fadd_rn(v[x], 128.0f), 12582912.0f)) - 0x4B400000;
                o[x] = (uint32_t) min(max(s, 0), 255);
        }
        return make_uint2(o[0] | o[1] << 8 | o[2] << 16 | o[3] << 24, o[4] | o[5] << 8 | o[6] << 16 | o[7] << 24);
}

/// FANCY: fill fancy_chroma() from the CTA's chroma tiles and the halo.  The halo is the IDCT of the neighbouring chroma blocks, computed here with
/// the same operations as the CTA that owns them, so a halo sample equals that CTA's sample bit for bit: the last column of block mx0 - 1 and the
/// first of block mx0 + 32 (full IDCT, one thread per block), and for 4:2:0 the last row of the 34 blocks mx0 - 1 .. mx0 + 32 of the MCU row above and
/// the first row of those below (column pass and one row pass).  Blocks outside the grid are skipped: the clamp of fancy_rgb never reads them.
template <int V>
__device__ __forceinline__ void fancy_fill(const int16_t *__restrict__ coef, const float (*s_m)[64], const uint2 (*s_tile)[8][32], const dec_geom &g, int tid, int nt)
{
        uint8_t(*s_c)[10][kFancyRow] = fancy_chroma();
        for (int i = tid; i < 512; i += nt) {
                const int comp = i >> 8, r = (i >> 5) & 7, m = i & 31;
                *(uint2 *) &s_c[comp][r + 1][8 + 8 * m] = s_tile[2 * V + comp][r][m];
        }
        const int mcux = g.c[1].bw, mcuy = g.c[1].bh, mx0 = blockIdx.x * 32, my = blockIdx.y;
        constexpr int NROW = V == 2 ? 2 * 2 * 34 : 0;  // (component, above / below, block) tasks of the vertical halo
        float f[64];
        if (tid < NROW) {
                const int comp = tid / 68, below = (tid / 34) & 1, X = mx0 - 1 + tid % 34, Y = below ? my + 1 : my - 1;
                if (X >= 0 && X < mcux && Y >= 0 && Y < mcuy) {
                        const dec_comp &c = g.c[1 + comp];
                        idct_columns(coef + ((long) c.blk_off + (long) Y * c.bw + X) * 64, s_m[c.tq], f);
                        *(uint2 *) &s_c[comp][below ? 9 : 0][8 * (X - mx0 + 1)] = below ? idct_row(f, 0) : idct_row(f, 7);  // f stays in registers
                }
        } else if (tid < NROW + 4) {
                const int t = tid - NROW, comp = t >> 1, right = t & 1, X = right ? mx0 + 32 : mx0 - 1;
                if (X >= 0 && X < mcux) {
                        const dec_comp &c = g.c[1 + comp];
                        idct_columns(coef + ((long) c.blk_off + (long) my * c.bw + X) * 64, s_m[c.tq], f);
#pragma unroll
                        for (int r = 0; r < 8; ++r) {
                                const uint2 v = idct_row(f, r);
                                s_c[comp][r + 1][right ? 264 : 7] = (uint8_t) (right ? v.x : v.y >> 24);
                        }
                }
        }
}

/// FANCY: the RGB / RGBA bytes of the 16 pixels of MCU `mcu` in pixel row `row` of the CTA.  Chroma is upsampled as libjpeg-turbo does it
/// (jdsample.c h2v1 / h2v2 fancy upsampling): a neighbour outside [0, cw - 1] x [0, ch - 1] takes the nearest edge sample, and chroma rows of at most
/// two samples are replicated, as libjpeg-turbo replicates them.
template <int V, class CS, bool RGBA>
__device__ __forceinline__ void fancy_rgb(const uint2 (*s_tile)[8][32], const dec_geom &g, int row, int mcu, uint32_t *o, const conv_params &p)
{
        const uint8_t(*s_c)[10][kFancyRow] = fancy_chroma();
        const int cw = (g.w + 1) / 2, ch = V == 2 ? (g.h + 1) / 2 : g.h;
        const int x0 = (blockIdx.x * 32 + mcu) * 8, base = 8 - (int) blockIdx.x * 256;  // byte of global chroma column x: base + x
        const int cr = V == 2 ? row >> 1 : row;
        // 4:2:0: the tile row of the neighbouring chroma row (above for an even pixel row, below for an odd one)
        const int nr = V == 2 ? min(max((int) blockIdx.y * 8 + cr + (row & 1 ? 1 : -1), 0), ch - 1) - (int) blockIdx.y * 8 + 1 : 0;
        int up[2][16];
#pragma unroll
        for (int comp = 0; comp < 2; ++comp) {
                if (cw <= 2) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                                up[comp][2 * j] = up[comp][2 * j + 1] = s_c[comp][cr + 1][base + x0 + j];
                        }
                        continue;
                }
                int s[10];  // columns x0 - 1 .. x0 + 8, each clamped to [0, cw - 1]: c (4:2:2) or 3 c + n (4:2:0)
#pragma unroll
                for (int k = 0; k < 10; ++k) {
                        const int x = base + min(max(x0 + k - 1, 0), cw - 1);
                        const int c = s_c[comp][cr + 1][x];
                        s[k] = V == 2 ? 3 * c + s_c[comp][nr][x] : c;
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                        if (V == 2) {
                                up[comp][2 * j] = (3 * s[j + 1] + s[j] + 8) >> 4, up[comp][2 * j + 1] = (3 * s[j + 1] + s[j + 2] + 7) >> 4;
                        } else {
                                up[comp][2 * j] = (3 * s[j + 1] + s[j] + 1) >> 2, up[comp][2 * j + 1] = (3 * s[j + 1] + s[j + 2] + 2) >> 2;
                        }
                }
        }
        constexpr color_coeffs c = CS::coeffs();
        const uint2 ya = s_tile[(V == 2 ? 2 * (row >> 3) : 0)][row & 7][mcu], yb = s_tile[(V == 2 ? 2 * (row >> 3) : 0) + 1][row & 7][mcu];
        const uint32_t amask = 0xFFFFFFFFu ^ (0xFFu << p.rshift) ^ (0xFFu << p.gshift) ^ (0xFFu << p.bshift);
        if (!RGBA) {
#pragma unroll
                for (int q = 0; q < 12; ++q) {
                        o[q] = 0;
                }
        }
#pragma unroll
        for (int i = 0; i < 16; ++i) {
                const uint32_t yw = i < 4 ? ya.x : i < 8 ? ya.y : i < 12 ? yb.x : yb.y;
                const int ys = c.y_scale * ((int) ((yw >> (8 * (i & 3))) & 0xffu) - CS::y_off), cb = up[0][i] - 128, cr2 = up[1][i] - 128;
                const uint32_t r = (uint32_t) min(max((ys + c.r_cr * cr2) >> COMP_BASE, 0), 255),
                               gg = (uint32_t) min(max((ys + c.g_cb * cb + c.g_cr * cr2) >> COMP_BASE, 0), 255),
                               b = (uint32_t) min(max((ys + c.b_cb * cb) >> COMP_BASE, 0), 255);
                if (RGBA) {
                        o[i] = amask | r << p.rshift | gg << p.gshift | b << p.bshift;
                } else {
                        o[(3 * i) >> 2] |= r << (8 * ((3 * i) & 3));
                        o[(3 * i + 1) >> 2] |= gg << (8 * ((3 * i + 1) & 3));
                        o[(3 * i + 2) >> 2] |= b << (8 * ((3 * i + 2) & 3));
                }
        }
}

/// the UYVY words of 8 pixels: 8 luma samples, the 4 Cb and 4 Cr samples of their pairs
__device__ __forceinline__ void uyvy_words(uint2 Y, uint32_t C, uint32_t R, uint32_t *w)
{
        w[0] = __byte_perm(__byte_perm(C, R, 0x0040), Y.x, 0x5140), w[1] = __byte_perm(__byte_perm(C, R, 0x0051), Y.x, 0x7160);
        w[2] = __byte_perm(__byte_perm(C, R, 0x0062), Y.y, 0x5140), w[3] = __byte_perm(__byte_perm(C, R, 0x0073), Y.y, 0x7160);
}

/// 4:2:2 (V = 1) and 4:2:0 (V = 2) YCbCr streams: IDCT, chroma replication and packing in one kernel, no component planes.  CTA = 32 MCUs of one
/// MCU row x the MCU's blocks (4:2:2: Y0 Y1 Cb Cr; 4:2:0: Y0 Y1 Y2 Y3 Cb Cr), warp k = block kind k (component-uniform dequantisation), lane = MCU.
/// The 8 x 8 samples of each block go to a shared tile as 8-byte rows.  The tile then leaves as UYVY words, the chroma of a pair row shared by both luma
/// rows of a 4:2:0 MCU (what yuv420p_to_uyvy does), through the epilogue E: as UYVY in 16-byte pieces, consecutive threads consecutive in memory; or
/// converted to RGB / RGBA, 16 pixels per thread, staged per warp in shared memory so that each warp stores its row's run as consecutive 16-byte
/// pieces.  Same IDCT arithmetic as jpeg_idct_kernel.  A row holds ((w + 1) / 2) * 4 bytes of UYVY (the last pair of an odd width takes the padded
/// plane's luma) but only whole pixel pairs of RGB / RGBA (the line converters' out_len), and rows but the last stop at the pitch, as there.
/// MX: the samples are taken from one YCbCr colour space to another (ycc_matrix, color_space.h) in the shared tile before they are packed - luma
/// first, with the source chroma of its pair / quad, then each chroma sample once - so the epilogue and its stores are those of the plain kernel.
/// E = epi_i420: `out` is a tight I420 frame (Y plane of w x h, then Cb and Cr of (w + 1) / 2 x (h + 1) / 2).  Luma rows leave the tile as 8-byte pieces,
/// consecutive threads consecutive in memory.  A 4:2:0 stream's chroma tiles ARE the I420 chroma (uyvy_to_i420(yuv420p_to_uyvy(x)) = x); a 4:2:2 stream's
/// chroma rows are averaged in pairs, (a + b + 1) / 2, as uyvy_to_i420 does (to_planar.c:364-367) - an MCU row is 8 pixel rows, so a pair never straddles
/// CTAs - and the last row of an odd height is taken as it is.  With MX the averaged samples are the converted ones ("convert, then pack").
/// GRAY: a one-component stream (V = 1): the CTA is 32 pairs of luma blocks of a block row, two warps, and the epilogues are fed Cb = Cr = 128.
template <int V, class E, bool MX = false, bool GRAY = false>
__global__ void __launch_bounds__(32 * (GRAY ? 2 : 2 * V + 2)) jpeg_idct_packed_kernel(const int16_t *__restrict__ coef, const dec_tables *__restrict__ tables, dec_geom g,
                                                                                       uint8_t *__restrict__ out, long pitch, bool vec_ok, conv_params p, ycc_matrix ym)
{
        static_assert(!GRAY || V == 1, "a one-component scan is not interleaved: its MCU is one block");
        constexpr int NB = GRAY ? 2 : 2 * V + 2, NT = 32 * NB, ROWS = 8 * V, PPR = 32 * 16 / E::PX;  // blocks per MCU, threads, pixel rows, pieces per row
        constexpr bool STAGED = E::PX == 16;
        __shared__ float s_m[4][64];
        __shared__ uint2 s_tile[NB][8][32];
        __shared__ uint4 s_out[STAGED ? NB : 1][STAGED ? 32 * E::OUT / 16 : 1];
        const int tid = threadIdx.x;
        for (int i = tid; i < 256; i += NT) {
                s_m[i >> 6][i & 63] = tables->m[i >> 6][i & 63];
        }
        __syncthreads();
        const int mcux = GRAY ? (g.c[0].bw + 1) / 2 : g.c[1].bw, my = blockIdx.y, mx0 = blockIdx.x * 32;
        const int k = tid >> 5, lane = tid & 31, mx = mx0 + lane;
        if (mx < mcux && (!GRAY || 2 * mx + k < g.c[0].bw)) {  // GRAY: an odd block count leaves the last pair's second block out (it lies past the width)
                const int ci = k < 2 * V ? 0 : k - 2 * V + 1;
                const dec_comp &c = g.c[ci];
                const int X = ci == 0 ? 2 * mx + (k & 1) : mx, Y = ci == 0 ? V * my + (k >> 1) : my;
                const long b = (long) c.blk_off + (long) Y * c.bw + X;
                const float *mq = s_m[c.tq];
                float f[64];
                const uint4 *src = (const uint4 *) (coef + b * 64);
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                        const uint4 v = __ldg(src + q);
                        const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                                const int lo = (int) (short) (w[j] & 0xffffu), hi = (int) w[j] >> 16;
                                f[8 * q + 2 * j] = __fmul_rn(__fadd_rn(__uint_as_float(0x4B400000u + (uint32_t) lo), -12582912.0f), mq[8 * q + 2 * j]);
                                f[8 * q + 2 * j + 1] = __fmul_rn(__fadd_rn(__uint_as_float(0x4B400000u + (uint32_t) hi), -12582912.0f), mq[8 * q + 2 * j + 1]);
                        }
                }
#pragma unroll
                for (int col = 0; col < 8; ++col) {
                        idct8(f[col], f[8 + col], f[16 + col], f[24 + col], f[32 + col], f[40 + col], f[48 + col], f[56 + col]);
                }
#pragma unroll
                for (int r = 0; r < 8; ++r) {
                        idct8(f[8 * r], f[8 * r + 1], f[8 * r + 2], f[8 * r + 3], f[8 * r + 4], f[8 * r + 5], f[8 * r + 6], f[8 * r + 7]);
                        uint32_t o[8];
#pragma unroll
                        for (int x = 0; x < 8; ++x) {
                                const int v = (int) __float_as_uint(__fadd_rn(__fadd_rn(f[8 * r + x], 128.0f), 12582912.0f)) - 0x4B400000;
                                o[x] = (uint32_t) min(max(v, 0), 255);
                        }
                        s_tile[k][r][lane] = make_uint2(o[0] | o[1] << 8 | o[2] << 16 | o[3] << 24, o[4] | o[5] << 8 | o[6] << 16 | o[7] << 24);
                }
        }
        __syncthreads();
        if constexpr (is_fancy<E>) {
                fancy_fill<V>(coef, s_m, s_tile, g, tid, NT);
                __syncthreads();
        }
        if constexpr (MX) {
                const int ybias = 8192 - ym.yy * ym.o_in;
                auto conv4 = [&](uint32_t y, int t0, int t1) {  // four luma samples, two pairs
                        uint32_t r = 0;
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                                const int v = ((ym.yy * (int) ((y >> (8 * i)) & 0xffu) + (i < 2 ? t0 : t1)) >> 14) + ym.o_out;
                                r |= (uint32_t) min(max(v, 0), 255) << (8 * i);
                        }
                        return r;
                };
                for (int i = tid; i < 2 * V * 256; i += NT) {  // luma: 8 samples of a block row with the 4 chroma pairs above them
                        const int mcu = i & 31, r = (i >> 5) & 7, kb = i >> 8;
                        int t[4] = { ybias, ybias, ybias, ybias };
                        if constexpr (!GRAY) {
                                const int crow = V == 2 ? 4 * (kb >> 1) + (r >> 1) : r;
                                const uint2 CB = s_tile[2 * V][crow][mcu], CR = s_tile[2 * V + 1][crow][mcu];
                                const uint32_t cb = kb & 1 ? CB.y : CB.x, cr = kb & 1 ? CR.y : CR.x;
#pragma unroll
                                for (int j = 0; j < 4; ++j) {
                                        t[j] += ym.yb * ((int) ((cb >> (8 * j)) & 0xffu) - 128) + ym.yr * ((int) ((cr >> (8 * j)) & 0xffu) - 128);
                                }
                        }
                        const uint2 y = s_tile[kb][r][mcu];
                        s_tile[kb][r][mcu] = make_uint2(conv4(y.x, t[0], t[1]), conv4(y.y, t[2], t[3]));
                }
                if constexpr (!GRAY) {
                        __syncthreads();  // every luma sample has read its source chroma
                        for (int i = tid; i < 512; i += NT) {  // chroma: four samples of Cb and of Cr at the same place
                                const int mcu = i & 31, r = (i >> 5) & 7, half = i >> 8;
                                uint32_t *pb = (uint32_t *) &s_tile[2 * V][r][mcu] + half, *pr = (uint32_t *) &s_tile[2 * V + 1][r][mcu] + half;
                                const uint32_t cb = *pb, cr = *pr;
                                uint32_t ob = 0, orr = 0;
#pragma unroll
                                for (int j = 0; j < 4; ++j) {
                                        const int b = (int) ((cb >> (8 * j)) & 0xffu) - 128, r2 = (int) ((cr >> (8 * j)) & 0xffu) - 128;
                                        ob |= (uint32_t) min(max(((ym.bb * b + ym.br * r2 + 8192) >> 14) + 128, 0), 255) << (8 * j);
                                        orr |= (uint32_t) min(max(((ym.rb * b + ym.rr * r2 + 8192) >> 14) + 128, 0), 255) << (8 * j);
                                }
                                *pb = ob, *pr = orr;
                        }
                }
                __syncthreads();
        }
        if constexpr (std::is_same<E, epi_i420>::value) {
                const int cw = (g.w + 1) / 2, chh = (g.h + 1) / 2;
                auto store8 = [&](uint8_t *row, int x, int width, uint2 v) {  // 8 samples at row[x], cut at the plane's width
                        if (x >= width) {
                                return;
                        }
                        if (vec_ok && x + 8 <= width) {
                                *(uint2 *) (row + x) = v;
                        } else {
                                for (int b = 0; b < 8 && x + b < width; ++b) {
                                        row[x + b] = (uint8_t) ((b < 4 ? v.x : v.y) >> (8 * (b & 3)));
                                }
                        }
                };
                for (int i = tid; i < ROWS * 64; i += NT) {  // luma: 64 pieces of 8 pixels per row
                        const int row = i >> 6, piece = i & 63, mcu = piece >> 1, y = my * ROWS + row;
                        if (y < g.h && mx0 + mcu < mcux) {
                                store8(out + (long) y * g.w, (mx0 + mcu) * 16 + (piece & 1) * 8, g.w, s_tile[(V == 2 ? 2 * (row >> 3) : 0) + (piece & 1)][row & 7][mcu]);
                        }
                }
                constexpr int CROWS = V == 2 ? 8 : 4;  // chroma rows of the MCU row
                uint8_t *const cplane = out + (long) g.w * g.h;
                for (int i = tid; i < 2 * CROWS * 32; i += NT) {
                        const int mcu = i & 31, r = (i >> 5) % CROWS, comp = i / (32 * CROWS), cy = my * CROWS + r;
                        if (cy >= chh || mx0 + mcu >= mcux) {
                                continue;
                        }
                        uint2 v = make_uint2(0x80808080u, 0x80808080u);
                        if constexpr (!GRAY) {
                                if (V == 2) {
                                        v = s_tile[4 + comp][r][mcu];
                                } else {
                                        v = s_tile[2 + comp][2 * r][mcu];
                                        if (my * 8 + 2 * r + 1 < g.h) {
                                                const uint2 b = s_tile[2 + comp][2 * r + 1][mcu];
                                                v = make_uint2(__vavgu4(v.x, b.x), __vavgu4(v.y, b.y));
                                        }
                                }
                        }
                        store8(cplane + (long) comp * cw * chh + (long) cy * cw, (mx0 + mcu) * 8, cw, v);
                }
                return;
        }
        const int row_full = is_fancy<E> ? g.w * E::BPP : E::BPP == 2 ? ((g.w + 1) / 2) * 4 : (g.w / 2) * 2 * E::BPP;
        for (int cidx = tid; cidx < ROWS * PPR; cidx += NT) {
                const int row = cidx / PPR, piece = cidx % PPR, mcu = piece / (16 / E::PX), half = piece % (16 / E::PX);
                const int y = my * ROWS + row;
                if (y >= g.h) {  // uniform over the warp
                        break;
                }
                const int lim = E::BPP == 2 || y == g.h - 1 || row_full <= pitch ? row_full : (int) pitch;
                uint32_t o[E::OUT / 4];
                if constexpr (is_fancy<E>) {
                        fancy_rgb<V, typename E::cs, E::rgba>(s_tile, g, row, mcu, o, p);
                } else {
                        const int cb = 2 * V, crow = V == 2 ? row >> 1 : row, yb = V == 2 ? 2 * (row >> 3) : 0, yrow = row & 7;
                        uint2 CB, CR;
                        if constexpr (GRAY) {
                                CB = CR = make_uint2(0x80808080u, 0x80808080u);
                        } else {
                                CB = s_tile[cb][crow][mcu], CR = s_tile[cb + 1][crow][mcu];
                        }
                        uint32_t w[E::PX / 2];
                        if (E::PX == 8) {
                                uyvy_words(s_tile[yb + half][yrow][mcu], half ? CB.y : CB.x, half ? CR.y : CR.x, w);
                        } else {
                                uyvy_words(s_tile[yb][yrow][mcu], CB.x, CR.x, w);
                                uyvy_words(s_tile[yb + 1][yrow][mcu], CB.y, CR.y, w + 4);
                        }
                        E::run(w, o, p);
                }
                uint8_t *d = out + (long) y * pitch;
                if constexpr (!STAGED) {
                        const int xoff = (mx0 + mcu) * 32 + half * 16;
                        if (mx0 + mcu >= mcux || xoff >= lim) {
                                continue;
                        }
                        if (vec_ok && xoff + 16 <= lim) {
                                *(uint4 *) (d + xoff) = make_uint4(o[0], o[1], o[2], o[3]);
                        } else {
                                for (int bq = 0; bq < 16 && xoff + bq < lim; ++bq) {
                                        d[xoff + bq] = (uint8_t) (o[bq >> 2] >> (8 * (bq & 3)));
                                }
                        }
                } else {  // the warp holds one row's 32 pieces: stage them, then store the run as consecutive 16-byte pieces
                        constexpr int NQ = E::OUT / 16;
                        uint4 *sw = s_out[k];
#pragma unroll
                        for (int q = 0; q < NQ; ++q) {
                                sw[lane * NQ + q] = make_uint4(o[4 * q], o[4 * q + 1], o[4 * q + 2], o[4 * q + 3]);
                        }
                        __syncwarp();
                        const int x0 = mx0 * 16 * E::BPP, run = min(lim - x0, 32 * E::OUT);
#pragma unroll
                        for (int q = 0; q < NQ; ++q) {
                                const int off = (q * 32 + lane) * 16;
                                if (off >= run) {
                                        continue;
                                }
                                const uint4 v = sw[q * 32 + lane];
                                if (vec_ok && off + 16 <= run) {
                                        *(uint4 *) (d + x0 + off) = v;
                                } else {
                                        const uint32_t vw[4] = { v.x, v.y, v.z, v.w };
                                        for (int bq = 0; bq < 16 && off + bq < run; ++bq) {
                                                d[x0 + off + bq] = (uint8_t) (vw[bq >> 2] >> (8 * (bq & 3)));
                                        }
                                }
                        }
                        __syncwarp();
                }
        }
}

/// 4:4:4 YCbCr streams to RGB / RGBA in a colour space: one thread per pixel over the component planes of jpeg_idct_kernel (same formula as
/// conv_yuv422_rgb<..., CS>, in integers)
template <class CS, bool RGBA>
__global__ void __launch_bounds__(256) jpeg_planes_cs_kernel(const uint8_t *__restrict__ planes, dec_geom g, uint8_t *__restrict__ out, long pitch, conv_params p)
{
        const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
        if (x >= g.w) {
                return;
        }
        constexpr color_coeffs c = CS::coeffs();
        const long ls = (long) g.c[0].bw * 8;  // 1x1 sampling: the three planes have the same line size
        const int Y = planes[g.c[0].plane_off + y * ls + x] - CS::y_off, cb = planes[g.c[1].plane_off + y * ls + x] - 128,
                  cr = planes[g.c[2].plane_off + y * ls + x] - 128;
        const int ys = c.y_scale * Y;
        const uint32_t r = (uint32_t) min(max((ys + c.r_cr * cr) >> COMP_BASE, 0), 255), gg = (uint32_t) min(max((ys + c.g_cb * cb + c.g_cr * cr) >> COMP_BASE, 0), 255),
                       b = (uint32_t) min(max((ys + c.b_cb * cb) >> COMP_BASE, 0), 255);
        uint8_t *d = out + (long) y * pitch;
        if (RGBA) {
                const uint32_t v = (0xFFFFFFFFu ^ (0xFFu << p.rshift) ^ (0xFFu << p.gshift) ^ (0xFFu << p.bshift)) | r << p.rshift | gg << p.gshift | b << p.bshift;
                d[4 * x] = (uint8_t) v, d[4 * x + 1] = (uint8_t) (v >> 8), d[4 * x + 2] = (uint8_t) (v >> 16), d[4 * x + 3] = (uint8_t) (v >> 24);
        } else {
                d[3 * x] = (uint8_t) r, d[3 * x + 1] = (uint8_t) gg, d[3 * x + 2] = (uint8_t) b;
        }
}

/// 4:4:4 YCbCr streams from one YCbCr colour space to another (ycc_matrix): the three component planes of jpeg_idct_kernel in place, four samples
/// per thread, before the packers read them (same integers as the MX phase of jpeg_idct_packed_kernel)
__global__ void __launch_bounds__(256) jpeg_planes_ycc_kernel(uint8_t *__restrict__ planes, dec_geom g, ycc_matrix ym)
{
        const long i = (long) blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= (long) g.c[0].bw * g.c[0].bh * 16) {  // 1x1 sampling: the three padded planes have the same size, a multiple of 64
                return;
        }
        uint32_t *py = (uint32_t *) (planes + g.c[0].plane_off) + i, *pb = (uint32_t *) (planes + g.c[1].plane_off) + i, *pr = (uint32_t *) (planes + g.c[2].plane_off) + i;
        const uint32_t y = *py, cb = *pb, cr = *pr;
        uint32_t oy = 0, ob = 0, orr = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
                const int Y = (int) ((y >> (8 * j)) & 0xffu) - ym.o_in, b = (int) ((cb >> (8 * j)) & 0xffu) - 128, r = (int) ((cr >> (8 * j)) & 0xffu) - 128;
                oy |= (uint32_t) min(max(((ym.yy * Y + ym.yb * b + ym.yr * r + 8192) >> 14) + ym.o_out, 0), 255) << (8 * j);
                ob |= (uint32_t) min(max(((ym.bb * b + ym.br * r + 8192) >> 14) + 128, 0), 255) << (8 * j);
                orr |= (uint32_t) min(max(((ym.rb * b + ym.rr * r + 8192) >> 14) + 128, 0), 255) << (8 * j);
        }
        *py = oy, *pb = ob, *pr = orr;
}

// ---- marker scan on the device (streams with one interleaved scan: what UltraGrid sends for UYVY; or one scan per component: RGB) ---------------
// The host's part shrinks to the header segments in front of the SOS and a plain copy of the stream into pinned memory; the RSTn markers that
// split the entropy-coded data are found here: K-a counts the marker candidates of every 4 KB piece, K-b is a one-CTA exclusive scan, K-c writes
// their positions in stream order and notes the first one that is not an RSTn (it ends the scan), K-d turns the list into the segment table the
// Huffman kernel reads - the same rules as parse_stream (excess RSTn are ignored, missing segments decode as nothing).
constexpr int kMarkThreads = 256;  // x 16 bytes

/// bit k: byte base + k is 0xFF, its follower neither a stuffed 0x00 nor a fill 0xFF, and the pair lies inside [from, len)
__device__ __forceinline__ unsigned marker_mask16(const uint8_t *__restrict__ s, size_t len, size_t base, size_t from)
{
        if (base + 1 >= len) {
                return 0;
        }
        const uint4 v = *(const uint4 *) (s + base);       // the buffer is 16 bytes longer than the stream
        const uint32_t nxt = s[base + 16];
        const uint32_t w[5] = { v.x, v.y, v.z, v.w, nxt };
        unsigned mask = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
                const uint32_t follower = __funnelshift_r(w[i], w[i + 1], 8);
                const uint32_t cand = __vcmpeq4(w[i], 0xffffffffu) & ~(__vcmpeq4(follower, 0u) | __vcmpeq4(follower, 0xffffffffu));
                mask |= (((cand & 0x01010101u) * 0x01020408u) >> 24) << (4 * i);
        }
        const size_t last = len - 1;  // candidates need p + 1 < len
        if (base + 16 > last) {
                mask &= (1u << (unsigned) (last - base)) - 1u;
        }
        if (from > base) {
                mask &= from - base >= 16 ? 0u : ~((1u << (unsigned) (from - base)) - 1u);
        }
        return mask;
}

__global__ void __launch_bounds__(kMarkThreads) jpeg_marker_count_kernel(const uint8_t *__restrict__ s, size_t len, size_t from, uint32_t *__restrict__ cnt)
{
        __shared__ uint32_t s_w[kMarkThreads / 32];
        const size_t base = ((size_t) blockIdx.x * kMarkThreads + threadIdx.x) * 16;
        uint32_t n = __popc(marker_mask16(s, len, base, from));
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
                n += __shfl_xor_sync(0xffffffffu, n, d);
        }
        if ((threadIdx.x & 31) == 0) {
                s_w[threadIdx.x >> 5] = n;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
                uint32_t t = 0;
                for (int i = 0; i < kMarkThreads / 32; ++i) {
                        t += s_w[i];
                }
                cnt[blockIdx.x] = t;
        }
}

/// exclusive scan of cnt[0..n) in place; meta[0] = total, meta[1] = 0xFFFFFFFF (index of the first non-RSTn candidate, filled by K-c)
__global__ void __launch_bounds__(1024) jpeg_marker_scan_kernel(uint32_t *__restrict__ cnt, int n, uint32_t *__restrict__ meta)
{
        __shared__ uint32_t s_w[32];
        __shared__ uint32_t s_carry;
        if (threadIdx.x == 0) {
                s_carry = 0;
        }
        __syncthreads();
        for (int base = 0; base < n; base += 1024) {
                const int i = base + (int) threadIdx.x;
                const uint32_t v = i < n ? cnt[i] : 0;
                uint32_t incl = v;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                        const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
                        if ((threadIdx.x & 31) >= (unsigned) d) {
                                incl += o;
                        }
                }
                if ((threadIdx.x & 31) == 31) {
                        s_w[threadIdx.x >> 5] = incl;
                }
                __syncthreads();
                uint32_t before = s_carry;
                for (int w = 0; w < (int) (threadIdx.x >> 5); ++w) {
                        before += s_w[w];
                }
                if (i < n) {
                        cnt[i] = before + incl - v;
                }
                __syncthreads();
                if (threadIdx.x == 1023) {
                        s_carry = before + incl;
                }
                __syncthreads();
        }
        if (threadIdx.x == 0) {
                meta[kMetaTotal] = s_carry, meta[kMetaFirstOther] = 0xffffffffu, meta[kMetaOtherCount] = 0, meta[kMetaError] = 0;
        }
}

__global__ void __launch_bounds__(kMarkThreads) jpeg_marker_write_kernel(const uint8_t *__restrict__ s, size_t len, size_t from, const uint32_t *__restrict__ off,
                                                                         uint32_t *__restrict__ list, uint32_t *__restrict__ meta)
{
        __shared__ uint32_t s_w[kMarkThreads / 32];
        const size_t base = ((size_t) blockIdx.x * kMarkThreads + threadIdx.x) * 16;
        unsigned mask = marker_mask16(s, len, base, from);
        const uint32_t n = __popc(mask);
        uint32_t incl = n;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
                const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
                if ((threadIdx.x & 31) >= (unsigned) d) {
                        incl += o;
                }
        }
        if ((threadIdx.x & 31) == 31) {
                s_w[threadIdx.x >> 5] = incl;
        }
        __syncthreads();
        uint32_t idx = off[blockIdx.x] + incl - n;
        for (int w = 0; w < (int) (threadIdx.x >> 5); ++w) {
                idx += s_w[w];
        }
        while (mask) {
                const size_t p = base + (size_t) (__ffs((int) mask) - 1);
                mask &= mask - 1;
                list[idx] = (uint32_t) p;
                const int code = s[p + 1];
                if (code < 0xD0 || code > 0xD7) {
                        atomicMin(meta + kMetaFirstOther, idx);
                        const uint32_t k = atomicAdd(meta + kMetaOtherCount, 1u);  // the handful of markers that are not RSTn: SOS of later scans, EOI
                        if (k < (uint32_t) kMaxOther) {
                                meta[kMetaOther + k] = idx;
                        }
                }
                ++idx;
        }
}

/// segment table of ONE scan that starts at `begin0`: the rules of parse_stream's SOS branch
__global__ void __launch_bounds__(256) jpeg_marker_segments_kernel(const uint32_t *__restrict__ list, const uint32_t *__restrict__ meta, uint32_t begin0, uint32_t len,
                                                                   int nseg, uint32_t *__restrict__ seg_begin, uint32_t *__restrict__ seg_end)
{
        const int i = blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= nseg) {
                return;
        }
        const uint32_t total = meta[0], stop = min(meta[1], total);  // `stop` RSTn candidates precede the marker that ends the scan
        const uint32_t term = stop < total ? list[stop] : len;
        const uint32_t pushed = min(stop, (uint32_t) (nseg - 1));
        uint32_t b, e;
        if ((uint32_t) i < pushed) {
                b = i == 0 ? begin0 : list[i - 1] + 2, e = list[i];
        } else if ((uint32_t) i == pushed) {
                b = stop == 0 ? begin0 : list[stop - 1] + 2, e = term;
        } else {
                b = e = term;
        }
        seg_begin[i] = b, seg_end[i] = e;
}

/// multi-scan streams: see jpeg_marker_bounds.cuh (the same code is checked against the host parser on the CPU)
__global__ void jpeg_marker_bounds_kernel(const uint8_t *__restrict__ s, uint32_t len, const uint32_t *__restrict__ list, uint32_t *__restrict__ meta, uint32_t begin0,
                                          int nscans, uint32_t comp_ids)
{
        if (threadIdx.x == 0 && blockIdx.x == 0) {
                marker_bounds(s, len, list, meta, begin0, nscans, comp_ids);
        }
}

/// segment table of a multi-scan stream from the bounds above: the rules of jpeg_marker_segments_kernel per scan
__global__ void __launch_bounds__(256) jpeg_marker_segments_multi_kernel(const uint32_t *__restrict__ list, const uint32_t *__restrict__ meta, int nscans, int seg1, int seg2,
                                                                         int nseg, uint32_t *__restrict__ seg_begin, uint32_t *__restrict__ seg_end)
{
        const int i = blockIdx.x * blockDim.x + threadIdx.x;
        if (i < nseg) {
                marker_segment_multi(list, meta, nscans, seg1, seg2, nseg, i, seg_begin + i, seg_end + i);
        }
}

}  // namespace ugb

using namespace ugb;

/// A handful of persistent host threads for the marker scan (creating threads per frame costs more than the scan of an 8K stream).
class scan_pool {
public:
        explicit scan_pool(int n)
        {
                for (int i = 0; i < n; ++i) {
                        workers.emplace_back([this, i] { run(i); });
                }
        }
        ~scan_pool()
        {
                {
                        std::lock_guard<std::mutex> lk(m);
                        quit = true;
                }
                cv.notify_all();
                for (auto &t : workers) {
                        t.join();
                }
        }
        int size() const { return (int) workers.size(); }
        /// runs job(i) for i in 0..n-1 on the workers (n <= size()) while the caller does its own share; returns when all are done
        void parallel(int n, const std::function<void(int)> &job_, const std::function<void()> &own)
        {
                {
                        std::lock_guard<std::mutex> lk(m);
                        job = &job_, todo = n, left = n, ++generation;
                }
                cv.notify_all();
                own();
                std::unique_lock<std::mutex> lk(m);
                done.wait(lk, [this] { return left == 0; });
                job = nullptr;
        }

private:
        void run(int i)
        {
                unsigned seen = 0;
                for (;;) {
                        const std::function<void(int)> *j;
                        {
                                std::unique_lock<std::mutex> lk(m);
                                cv.wait(lk, [&] { return quit || (generation != seen && i < todo); });
                                if (quit) {
                                        return;
                                }
                                seen = generation, j = job;
                        }
                        (*j)(i);
                        std::lock_guard<std::mutex> lk(m);
                        if (--left == 0) {
                                done.notify_one();
                        }
                }
        }
        std::vector<std::thread> workers;
        std::mutex m;
        std::condition_variable cv, done;
        const std::function<void(int)> *job = nullptr;
        int todo = 0, left = 0;
        unsigned generation = 0;
        bool quit = false;
};

struct ugb200_jpeg_decoder {
        cudaStream_t stream = nullptr;
        scan_pool pool{ 7 };
        cudaStream_t copy = nullptr;  // the stream upload of frame n + 1 runs here, under the kernels of frame n (its device copy is double-buffered with the host slots)
        uint8_t *planes = nullptr, *native = nullptr, *staging = nullptr;
        int16_t *coef = nullptr;
        uint32_t *d_seg = nullptr, *d_marks = nullptr, *d_mark_cnt = nullptr;  // d_mark_cnt: per-piece counts / offsets, then meta[kMetaWords]
        dec_tables *d_tables = nullptr;
        size_t planes_cap = 0, native_cap = 0, staging_cap = 0, coef_cap = 0, seg_cap = 0, marks_cap = 0, mark_cnt_cap = 0;
        int scan_mode = 0;      // 0: device scan for large streams (one interleaved scan, or one scan per component), 1: always the host scan, 2: device scan at any size
        bool host_once = false; // the device found a multi-scan stream irregular: this frame is repeated with the host parser
        uint32_t *h_flag = nullptr;  // pinned: the device's verdict on a multi-scan stream
        size_t last_nseg = 0;   // segments of the last decode (ugb200_jpeg_decoder_last_segments)
        // the self-synchronising route: 0 = for segments of at least kSyncMinMcus MCUs (every scan without DRI), 1 = never, 2 = always (UGB200_JPEG_SYNC)
        int sync_mode = 0, sync_bytes = kSyncBytes;
        uint32_t *d_sync = nullptr;
        size_t sync_cap = 0;
        int sync_grid = 0;       // co-resident CTAs of jpeg_sync_kernel
        uint32_t *last_sync_ctr = nullptr;  // rounds and subsequences of the last decode on the device (nullptr: the route did not run)
        int last_sync_scans = 0;
        // pinned staging (the caller's stream buffer is pageable and freed right after the call), two slots: the host side of frame
        // i + 1 (scan, parse, staging copy) runs while the device still works on frame i
        struct host_slot {
                uint8_t *stream = nullptr;
                uint32_t *seg = nullptr;
                dec_tables *tables = nullptr;
                uint8_t *d_stream = nullptr;  // this slot's copy of the stream on the device (16 bytes longer than the stream)
                size_t stream_cap = 0, seg_cap = 0, d_stream_cap = 0;
                cudaEvent_t uploaded = nullptr;   // segment table + Huffman / quantisation tables left the pinned slot (decoder's stream)
                cudaEvent_t stream_up = nullptr;  // the stream left the pinned slot and is on the device (copy stream)
                cudaEvent_t consumed = nullptr;   // the last kernel that reads d_stream is done (decoder's stream)
                bool pending = false, consumed_pending = false;
        } hs[2];
        unsigned frame_no = 0;
        int expect_w = 0, expect_h = 0;  // ugb200_jpeg_decoder_expect: the destination was sized for these; 0 = unchecked
        int upsampling = UGB200_JPEG_UPSAMPLE_REPLICATE;  // ugb200_jpeg_decoder_set_upsampling
        // host scratch that keeps its capacity from frame to frame
        std::vector<uint64_t> scan_part[8], markers;
        std::vector<uint32_t> seg_begin, seg_end;
};

namespace {

template <class T>
bool dgrow(T *&ptr, size_t &cap, size_t need)
{
        if (need <= cap) {
                return true;
        }
        if (ptr) {
                cudaFree(ptr);
        }
        ptr = nullptr, cap = 0;
        if (cudaMalloc((void **) &ptr, need * sizeof(T)) != cudaSuccess) {
                return false;
        }
        cap = need;
        return true;
}
template <class T>
bool hgrow(T *&ptr, size_t &cap, size_t need)
{
        if (need <= cap) {
                return true;
        }
        if (ptr) {
                cudaFreeHost(ptr);
        }
        ptr = nullptr, cap = 0;
        if (cudaMallocHost((void **) &ptr, need * sizeof(T)) != cudaSuccess) {
                return false;
        }
        cap = need;
        return true;
}

int be16(const uint8_t *p) { return p[0] << 8 | p[1]; }

template <class T>
struct type_tag {  // carries an epilogue type into a generic lambda
        using type = T;
};

constexpr long kMaxPixels = 16384L * 16384L;  // four 8K frames side by side; larger SOF dimensions are refused before anything is allocated

struct huff_defs {  // the current DHT definition of each table id, built into a slot of dec_tables when a scan first uses it
        uint8_t bits[4][16], vals[4][256];
        int n[4] = { 0, 0, 0, 0 };
        bool defined[4] = { false, false, false, false };
        int slot[4] = { -1, -1, -1, -1 };  // slot holding the current definition, -1 = not built yet
        bool taken[kTables] = {};          // built: a scan reads it
};

struct parsed {
        dec_geom g{};
        int adobe = -1, comp_id[4] = { 0, 0, 0, 0 };
        int spiff = -1;  // colour space field of the first SPIFF APP8, -2 when that segment is too short to hold it
        bool jfif = false;
        bool have_sof = false, have_q[4] = { false, false, false, false };
        huff_defs hd;
        uint8_t q[4][64];
        std::vector<uint32_t> seg_begin, seg_end;
};

/// @returns false for an over-subscribed code-length histogram (the Kraft check behind libjpeg's JERR_BAD_HUFF_TABLE): after the codes of
/// length l are assigned the next code must still fit in l bits, otherwise the look-up fill of build_table would run past the table
bool kraft_ok(const uint8_t *bits)
{
        for (int l = 1, code = 0; l <= 16; ++l) {
                code += bits[l - 1];
                if (code > (1 << l)) {
                        return false;
                }
                code <<= 1;
        }
        return true;
}

/// the table slot of the current definition of table id `id`, built on first use (see kTables); -1: the table is undefined or no slot is left
int table_slot(huff_defs &H, dec_tables *T, int id)
{
        if (!H.defined[id]) {
                return -1;
        }
        if (H.slot[id] < 0) {
                int k = id;
                if (H.taken[k]) {
                        for (k = 0; k < kTables && H.taken[k]; ++k) {
                        }
                        if (k == kTables) {
                                return -1;
                        }
                }
                H.taken[k] = true, H.slot[id] = k;
                if (T) {
                        build_table(*T, k, H.bits[id], H.vals[id], H.n[id]);
                }
        }
        return H.slot[id];
}

const bool g_stream_stores = [] {
        const char *e = getenv("UGB200_JPEG_STAGE");  // "plain": ordinary stores into the pinned staging buffer (A/B timing)
        return !(e && e[0] == 'p');
}();

const float kAan[8] = { 1.0f, 1.387039845f, 1.306562965f, 1.175875602f, 1.0f, 0.785694958f, 0.541196100f, 0.275899379f };

/// marker candidates of [lo, hi): positions p with s[p] == 0xFF and s[p + 1] neither a stuffed 0x00 nor a fill 0xFF.  One SSE2 compare per
/// 16 bytes, then only the 0xFF positions are looked at.  Optionally copies the range to `copy_to` in the same pass (staging for the upload).
void scan_markers(const uint8_t *s, size_t lo, size_t hi, size_t len, std::vector<uint64_t> &out, uint8_t *copy_to)
{
        const __m128i ff16 = _mm_set1_epi8((char) 0xFF), zero = _mm_setzero_si128();
        size_t i = lo;
        // the staging buffer is read next by the copy engine, not by a CPU: non-temporal stores keep it out of the caches (an upload of a stream
        // that several cores had just written through their caches was slow on an earlier machine)
        const bool stream_stores = copy_to != nullptr && g_stream_stores && ((uintptr_t) (copy_to + lo) & 15) == 0;
        // 0xFF is frequent in Huffman-coded data (runs of 1-bits), a marker is not: the follower byte is tested in the vector domain too
        for (; i + 17 <= len && i + 16 <= hi; i += 16) {
                const __m128i v = _mm_loadu_si128((const __m128i *) (s + i)), nx = _mm_loadu_si128((const __m128i *) (s + i + 1));
                if (copy_to) {
                        if (stream_stores) {
                                _mm_stream_si128((__m128i *) (copy_to + i), v);
                        } else {
                                _mm_storeu_si128((__m128i *) (copy_to + i), v);
                        }
                }
                const __m128i stuffed = _mm_or_si128(_mm_cmpeq_epi8(nx, zero), _mm_cmpeq_epi8(nx, ff16));
                unsigned mask = (unsigned) _mm_movemask_epi8(_mm_andnot_si128(stuffed, _mm_cmpeq_epi8(v, ff16)));
                while (mask) {  // entry = marker code << 32 | position: the parser never has to touch the stream again (one cache miss per marker)
                        const size_t p = i + (size_t) __builtin_ctz(mask);
                        out.push_back((uint64_t) s[p + 1] << 32 | p);
                        mask &= mask - 1;
                }
        }
        for (; i < hi; ++i) {
                if (copy_to) {
                        copy_to[i] = s[i];
                }
                if (s[i] == 0xFF && i + 1 < len && s[i + 1] != 0 && s[i + 1] != 0xFF) {
                        out.push_back((uint64_t) s[i + 1] << 32 | i);
                }
        }
        if (stream_stores) {
                _mm_sfence();
        }
}

/// plain staging copy (device marker scan): non-temporal stores when the destination allows it
void stage_copy(uint8_t *dst, const uint8_t *src, size_t n)
{
        if (!g_stream_stores || ((uintptr_t) dst & 15) != 0) {
                memcpy(dst, src, n);
                return;
        }
        size_t i = 0;
        for (; i + 64 <= n; i += 64) {
                const __m128i a = _mm_loadu_si128((const __m128i *) (src + i)), b = _mm_loadu_si128((const __m128i *) (src + i + 16));
                const __m128i c = _mm_loadu_si128((const __m128i *) (src + i + 32)), e = _mm_loadu_si128((const __m128i *) (src + i + 48));
                _mm_stream_si128((__m128i *) (dst + i), a), _mm_stream_si128((__m128i *) (dst + i + 16), b);
                _mm_stream_si128((__m128i *) (dst + i + 32), c), _mm_stream_si128((__m128i *) (dst + i + 48), e);
        }
        memcpy(dst + i, src + i, n - i);
        _mm_sfence();
}

/// header markers up to and including every SOS; `full` also finds the restart segments of the entropy-coded data, from the marker
/// candidates in `markers` (sorted; scanned here when the caller has none)
int parse_stream(const uint8_t *s, size_t len, parsed &P, dec_tables *T, bool full, const std::vector<uint64_t> *markers = nullptr,
                 size_t *first_scan_data = nullptr)
{
        std::vector<uint64_t> own;
        if (full && markers == nullptr) {
                scan_markers(s, 0, len, len, own, nullptr);
                markers = &own;
        }
        const uint8_t *p = s, *end = s + len;
        if (len < 4 || p[0] != 0xFF || p[1] != 0xD8) {
                return -1;
        }
        p += 2;
        dec_geom &g = P.g;
        while (p + 4 <= end) {
                if (p[0] != 0xFF) {
                        return -3;
                }
                const int mk = p[1];
                if (mk == 0xD9) {
                        break;
                }
                if (mk == 0xFF) {  // fill byte
                        ++p;
                        continue;
                }
                const int L = be16(p + 2);
                const uint8_t *d = p + 4, *dend = p + 2 + L;
                if (L < 2 || dend > end) {
                        return -3;
                }
                if (mk == 0xDB) {
                        while (d + 65 <= dend) {
                                const int pq = d[0] >> 4, tq = d[0] & 15;
                                if (pq != 0 || tq > 3) {
                                        return -4;
                                }
                                for (int k = 0; k < 64; ++k) {
                                        P.q[tq][kZigzag[k]] = d[1 + k];
                                }
                                P.have_q[tq] = true;
                                if (T) {
                                        for (int n = 0; n < 64; ++n) {
                                                T->m[tq][n] = ((float) P.q[tq][n] * kAan[n >> 3]) * kAan[n & 7] * 0.125f;
                                        }
                                }
                                d += 65;
                        }
                } else if (mk == 0xC4) {
                        while (d + 17 <= dend) {
                                const int tc = d[0] >> 4, th = d[0] & 15;
                                int n = 0;
                                for (int i = 0; i < 16; ++i) {
                                        n += d[1 + i];
                                }
                                if (tc > 1 || th > 1 || n > 256 || d + 17 + n > dend) {
                                        return -4;  // baseline: two tables per class
                                }
                                if (!kraft_ok(d + 1)) {
                                        return -4;  // over-subscribed Huffman table
                                }
                                const int id = tc * 2 + th;  // a new definition: the slot of the old one stays with the scans that used it
                                memcpy(P.hd.bits[id], d + 1, 16), memcpy(P.hd.vals[id], d + 17, n);
                                P.hd.n[id] = n, P.hd.defined[id] = true, P.hd.slot[id] = -1;
                                d += 17 + n;
                        }
                } else if (mk == 0xC0) {
                        if (L < 8 || L < 8 + 3 * d[5] || d[0] != 8) {  // L first: d[5] lies inside the segment only then
                                return -4;
                        }
                        g.h = be16(d + 1), g.w = be16(d + 3), g.ncomp = d[5];
                        if ((g.ncomp != 1 && g.ncomp != 3 && g.ncomp != 4) || g.w == 0 || g.h == 0) {
                                return -4;
                        }
                        if ((long) g.w * g.h > kMaxPixels) {  // header fields are untrusted: they size every host and device allocation below
                                return -4;
                        }
                        g.hmax = g.vmax = 1;
                        for (int i = 0; i < g.ncomp; ++i) {
                                P.comp_id[i] = d[6 + 3 * i];
                                g.c[i].h = d[7 + 3 * i] >> 4, g.c[i].v = d[7 + 3 * i] & 15, g.c[i].tq = d[8 + 3 * i];
                                if (g.ncomp == 1) {  // T.81 A.2.2: a single-component scan is never interleaved, its sampling factors have no effect
                                        g.c[i].h = g.c[i].v = 1;
                                }
                                g.hmax = g.c[i].h > g.hmax ? g.c[i].h : g.hmax, g.vmax = g.c[i].v > g.vmax ? g.c[i].v : g.vmax;
                        }
                        int blk = 0;
                        long off = 0;
                        for (int i = 0; i < g.ncomp; ++i) {  // four components: every one sampled 1x1 (no subsampled alpha)
                                dec_comp &c = g.c[i];
                                if (c.h < 1 || c.h > 2 || c.v < 1 || c.v > 2 || ((i > 0 || g.ncomp == 4) && (c.h != 1 || c.v != 1)) || c.tq > 3) {
                                        return -4;
                                }
                                if (c.v > c.h) {  // luma 1x2 (4:4:0): no output layout packs it (UYVY and the 4:4:4 packers would read chroma rows that do not exist)
                                        return -4;
                                }
                                c.bw = (g.w + 8 * g.hmax - 1) / (8 * g.hmax) * c.h, c.bh = (g.h + 8 * g.vmax - 1) / (8 * g.vmax) * c.v;
                                c.blk_off = blk, c.plane_off = off;
                                blk += c.bw * c.bh, off += (long) c.bw * c.bh * 64;
                        }
                        g.nblocks = blk;
                        P.have_sof = true;
                } else if (mk >= 0xC1 && mk <= 0xCF && mk != 0xC4 && mk != 0xC8 && mk != 0xCC) {
                        return -4;  // not baseline sequential Huffman
                } else if (mk == 0xDD) {
                        if (L < 4) {
                                return -3;
                        }
                        g.ri = be16(d);
                } else if (mk == 0xEE && L >= 14 && memcmp(d, "Adobe", 5) == 0) {
                        P.adobe = d[11];
                } else if (mk == 0xE8 && L >= 8 && memcmp(d, "SPIFF", 6) == 0 && P.spiff == -1) {
                        P.spiff = L >= 21 ? d[18] : -2;  // identifier 6, version 2, profile 1, components 1, height 4, width 4, colour space 1
                } else if (mk == 0xE0 && L >= 7 && memcmp(d, "JFIF", 5) == 0) {
                        P.jfif = true;
                } else if (mk == 0xDA) {
                        if (!P.have_sof || g.nscans >= g.ncomp) {
                                return -3;
                        }
                        if (g.ncomp == 4 && P.adobe != -1 && P.adobe != 0) {
                                return -4;  // Adobe transform 2 (YCCK) or 1: samples are not R G B A as stored
                        }
                        dec_scan &S = g.s[g.nscans];
                        if (L < 3) {
                                return -3;
                        }
                        S.ns = d[0];
                        if (S.ns < 1 || S.ns > g.ncomp || L < 6 + 2 * S.ns) {
                                return -4;
                        }
                        for (int i = 0; i < S.ns; ++i) {
                                S.comp[i] = -1;
                                for (int j = 0; j < g.ncomp; ++j) {
                                        if (P.comp_id[j] == d[1 + 2 * i]) {
                                                S.comp[i] = j;
                                        }
                                }
                                const int td = d[2 + 2 * i] >> 4, ta = d[2 + 2 * i] & 15;
                                if (S.comp[i] < 0 || td > 1 || ta > 1 || !P.have_q[g.c[S.comp[i]].tq]) {
                                        return -4;
                                }
                                S.td[i] = table_slot(P.hd, T, td), S.ta[i] = table_slot(P.hd, T, 2 + ta);
                                if (S.td[i] < 0 || S.ta[i] < 0) {
                                        return -4;  // an undefined table, or more table definitions in use than a valid stream has
                                }
                        }
                        int mcuy;
                        if (S.ns == 1) {
                                const dec_comp &c = g.c[S.comp[0]];
                                S.mcux = ((g.w * c.h + g.hmax - 1) / g.hmax + 7) / 8, mcuy = ((g.h * c.v + g.vmax - 1) / g.vmax + 7) / 8;
                        } else {
                                S.mcux = (g.w + 8 * g.hmax - 1) / (8 * g.hmax), mcuy = (g.h + 8 * g.vmax - 1) / (8 * g.vmax);
                        }
                        S.nmcu = S.mcux * mcuy;
                        S.seg0 = (int) P.seg_begin.size();
                        S.nseg = g.ri ? (S.nmcu + g.ri - 1) / g.ri : 1;
                        // every segment but the last ends in a 2-byte RSTn: a stream of `len` bytes cannot hold more than len / 2 + 1 of them (the
                        // rest of a truncated stream is filled in below, bounded by kMaxPixels)
                        P.seg_begin.reserve(P.seg_begin.size() + std::min((size_t) S.nseg, len / 2 + 1)), P.seg_end.reserve(P.seg_begin.capacity());
                        ++g.nscans;
                        p = dend;
                        if (!full) {
                                if (first_scan_data) {
                                        *first_scan_data = (size_t) (p - s);
                                }
                                return 0;  // enough for the image info
                        }
                        // entropy-coded segment(s): RSTn candidates split it, the first other marker ends it
                        uint32_t begin = (uint32_t) (p - s);
                        int found = 0;
                        auto it = std::lower_bound(markers->begin(), markers->end(), (uint64_t) begin,
                                                   [](uint64_t e, uint64_t pos) { return (uint32_t) e < pos; });
                        for (; it != markers->end(); ++it) {
                                const int c2 = (int) (*it >> 32);
                                const uint32_t pos = (uint32_t) *it;
                                if (c2 < 0xD0 || c2 > 0xD7) {
                                        break;
                                }
                                if (found + 1 < S.nseg) {
                                        P.seg_begin.push_back(begin), P.seg_end.push_back(pos);
                                        ++found;
                                }
                                begin = pos + 2;
                        }
                        p = it != markers->end() ? s + (uint32_t) *it : end;
                        P.seg_begin.push_back(begin), P.seg_end.push_back((uint32_t) (p - s));
                        ++found;
                        while (found < S.nseg) {  // truncated stream: the missing segments decode as nothing (zero coefficients)
                                P.seg_begin.push_back((uint32_t) (p - s)), P.seg_end.push_back((uint32_t) (p - s));
                                ++found;
                        }
                        continue;
                }
                p = dend;
        }
        return P.have_sof && g.nscans > 0 ? 0 : -3;
}

/// all marker candidates of the stream, in order; large streams are split over the pool (piece 0 on the calling thread)
constexpr int kMaxScanThreads = 8;
/// `scratch`: kMaxScanThreads vectors that keep their capacity between frames (a decoder's frames have the same ~65 000 markers each time:
/// growing eight fresh vectors and the merged list per frame was a visible share of the host time), or nullptr
void collect_markers(const uint8_t *stream, size_t len, scan_pool *pool, uint8_t *copy_to, std::vector<uint64_t> &markers, std::vector<uint64_t> *scratch = nullptr)
{
        constexpr int kMaxThreads = kMaxScanThreads;
        int nt = len > (4u << 20) ? kMaxThreads : len > (1u << 20) ? 4 : 1;
        if (pool == nullptr || pool->size() + 1 < nt) {
                nt = pool ? pool->size() + 1 : 1;
        }
        std::vector<uint64_t> own[kMaxThreads];
        std::vector<uint64_t> *part = scratch ? scratch : own;
        for (int i = 0; i < kMaxThreads; ++i) {
                part[i].clear();
        }
        const size_t chunk = (len / nt + 15) & ~(size_t) 15;
        auto range = [&](int i) {
                const size_t lo = std::min(len, chunk * i), hi = i == nt - 1 ? len : std::min(len, chunk * (i + 1));
                scan_markers(stream, lo, hi, len, part[i], copy_to);
        };
        if (nt == 1) {
                range(0);
        } else {
                pool->parallel(nt - 1, [&](int w) { range(w + 1); }, [&] { range(0); });
        }
        for (int i = 0; i < nt; ++i) {
                markers.insert(markers.end(), part[i].begin(), part[i].end());
        }
}

int native_codec(const parsed &P)
{
        const dec_geom &g = P.g;
        if (g.ncomp == 4) {
                return UGB_RGBA;  // R G B A as stored (the parser refuses subsampled and YCCK four-component streams)
        }
        if (g.c[0].h == 2 || g.ncomp == 1) {
                return UGB_UYVY;  // 4:2:2 and 4:2:0 land in UYVY; so does grayscale, with Cb = Cr = 128
        }
        const bool rgb = P.adobe == 0 || (P.comp_id[0] == 'R' && P.comp_id[1] == 'G' && P.comp_id[2] == 'B');
        return rgb ? UGB_RGB : UGB_VUYA;
}

/// the colour space the stream declares (ugb200_jpeg_stream_color_space): UGB200_JPEG_CS_*, or -3 / -4
int declared_color_space(const parsed &P)
{
        const int nc = native_codec(P);
        if (nc == UGB_RGB || nc == UGB_RGBA) {
                return UGB200_JPEG_CS_RGB;
        }
        if (P.spiff != -1) {  // SPIFF colour space codes (ITU-T T.84 Annex F)
                if (P.g.ncomp == 1 && (P.spiff == 8 || P.spiff == 10)) {  // grayscale is full-range luma; a one-component stream is never RGB
                        return P.spiff == 8 ? UGB200_JPEG_CS_Y601FULL : -4;
                }
                switch (P.spiff) {
                case -2: return -3;
                case 1: return UGB200_JPEG_CS_Y709;
                case 3: return UGB200_JPEG_CS_Y601FULL;
                case 4: return UGB200_JPEG_CS_Y601;
                case 10: return UGB200_JPEG_CS_RGB;
                default: return -4;
                }
        }
        if (P.adobe == 1 || P.jfif) {  // Adobe APP14 transform 1, JFIF (T.871): full-range BT.601
                return UGB200_JPEG_CS_Y601FULL;
        }
        return UGB200_JPEG_CS_Y709;  // no marker: what UltraGrid tells GPUJPEG to assume (src/video_decompress/gpujpeg.c:103-112)
}

}  // namespace

extern "C" {

UGB_API int ugb200_jpeg_get_image_info(const uint8_t *stream, size_t len, struct ugb200_jpeg_image_info *info)
{
        if (!stream || !info) {
                return -1;
        }
        parsed P;
        const int rc = parse_stream(stream, len, P, nullptr, false);
        if (rc != 0) {
                return rc;
        }
        info->width = P.g.w, info->height = P.g.h, info->components = P.g.ncomp;
        info->h_samp = P.g.c[0].h, info->v_samp = P.g.c[0].v;
        info->adobe_transform = P.adobe, info->restart_interval = P.g.ri;
        info->native_codec = native_codec(P);
        return 0;
}

UGB_API int ugb200_jpeg_stream_color_space(const uint8_t *stream, size_t len)
{
        if (!stream) {
                return -1;
        }
        parsed P;
        const int rc = parse_stream(stream, len, P, nullptr, false);
        return rc != 0 ? rc : declared_color_space(P);
}

UGB_API long ugb200_jpeg_debug_segments(const uint8_t *stream, size_t len, uint32_t *begin, uint32_t *end, long cap)
{
        if (!stream) {
                return -1;
        }
        parsed P;
        dec_tables T;
        std::vector<uint64_t> markers;
        if (len > (1u << 20)) {  // the same threaded scan the decoder uses
                scan_pool pool(7);
                collect_markers(stream, len, &pool, nullptr, markers);
        } else {
                collect_markers(stream, len, nullptr, nullptr, markers);
        }
        const int rc = parse_stream(stream, len, P, &T, true, &markers);
        if (rc != 0) {
                return rc;
        }
        const long n = (long) P.seg_begin.size();
        for (long i = 0; i < n && i < cap; ++i) {
                begin[i] = P.seg_begin[i], end[i] = P.seg_end[i];
        }
        return n;
}

UGB_API ugb200_jpeg_decoder *ugb200_jpeg_decoder_create(cuda_wrapper_stream_t stream)
{
        ugb200_jpeg_decoder *d = new (std::nothrow) ugb200_jpeg_decoder;
        if (!d) {
                return nullptr;
        }
        d->stream = (cudaStream_t) stream;
        if (cudaMalloc((void **) &d->d_tables, sizeof(dec_tables)) != cudaSuccess || cudaMallocHost((void **) &d->hs[0].tables, sizeof(dec_tables)) != cudaSuccess ||
            cudaMallocHost((void **) &d->hs[1].tables, sizeof(dec_tables)) != cudaSuccess || cudaMallocHost((void **) &d->h_flag, 64) != cudaSuccess ||
            cudaEventCreateWithFlags(&d->hs[0].uploaded, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&d->hs[1].uploaded, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&d->hs[0].stream_up, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&d->hs[1].stream_up, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&d->hs[0].consumed, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&d->hs[1].consumed, cudaEventDisableTiming) != cudaSuccess ||
            cudaStreamCreateWithFlags(&d->copy, cudaStreamNonBlocking) != cudaSuccess) {
                ugb200_jpeg_decoder_destroy(d);
                return nullptr;
        }
        const char *m = getenv("UGB200_JPEG_MARKER_SCAN");  // "host" / "device": force one of the two marker scans (tests, A/B timing)
        d->scan_mode = !m ? 0 : m[0] == 'h' ? 1 : m[0] == 'd' ? 2 : 0;
        const char *y = getenv("UGB200_JPEG_SYNC");  // test hook: "off" / "on[:<subsequence bytes>]" forces the Huffman route (include/ugb200_jpeg.h)
        if (y && strncmp(y, "off", 3) == 0) {
                d->sync_mode = 1;
        } else if (y && strncmp(y, "on", 2) == 0) {
                d->sync_mode = 2;
                if (y[2] == ':' && atoi(y + 3) >= 1) {
                        d->sync_bytes = atoi(y + 3);
                }
        }
        return d;
}

UGB_API void ugb200_jpeg_decoder_destroy(ugb200_jpeg_decoder *d)
{
        if (!d) {
                return;
        }
        cudaStreamSynchronize(d->stream);
        if (d->copy) {
                cudaStreamSynchronize(d->copy);
                cudaStreamDestroy(d->copy);
        }
        cudaFree(d->planes), cudaFree(d->native), cudaFree(d->staging), cudaFree(d->coef), cudaFree(d->d_seg), cudaFree(d->d_tables);
        cudaFree(d->d_marks), cudaFree(d->d_mark_cnt), cudaFree(d->d_sync);
        cudaFreeHost(d->h_flag);
        for (auto &h : d->hs) {
                if (h.stream) {
                        cuda_wrapper_free_host(h.stream);
                }
                cudaFreeHost(h.seg), cudaFreeHost(h.tables);
                cudaFree(h.d_stream);
                for (cudaEvent_t e : { h.stream_up, h.consumed }) {
                        if (e) {
                                cudaEventDestroy(e);
                        }
                }
                if (h.uploaded) {
                        cudaEventDestroy(h.uploaded);
                }
        }
        delete d;
}

/// the segment table of the last decode as the device holds it (tests: the device marker scan against the host's)
UGB_API long ugb200_jpeg_decoder_last_segments(ugb200_jpeg_decoder *d, uint32_t *begin, uint32_t *end, long cap)
{
        if (!d || !begin || !end) {
                return -1;
        }
        const long n = (long) d->last_nseg;
        if (cudaStreamSynchronize(d->stream) != cudaSuccess) {
                return -2;
        }
        const long m = n < cap ? n : cap;
        if (m > 0 && (cudaMemcpy(begin, d->d_seg, (size_t) m * 4, cudaMemcpyDeviceToHost) != cudaSuccess ||
                      cudaMemcpy(end, d->d_seg + n, (size_t) m * 4, cudaMemcpyDeviceToHost) != cudaSuccess)) {
                return -2;
        }
        return n;
}

UGB_API int ugb200_jpeg_decoder_last_sync(ugb200_jpeg_decoder *d, struct ugb200_jpeg_sync_stats *st)
{
        if (!d || !st) {
                return -1;
        }
        if (cudaStreamSynchronize(d->stream) != cudaSuccess) {
                return -2;
        }
        uint32_t c[2] = { 0, 0 };
        if (d->last_sync_ctr && cudaMemcpy(c, d->last_sync_ctr + 3, 8, cudaMemcpyDeviceToHost) != cudaSuccess) {
                return -2;
        }
        st->scans = d->last_sync_scans, st->rounds = (int) c[0], st->subsequences = (long) c[1];
        return 0;
}

UGB_API int ugb200_jpeg_decoder_expect(ugb200_jpeg_decoder *d, int width, int height)
{
        if (!d || width < 0 || height < 0) {
                return -1;
        }
        d->expect_w = width, d->expect_h = height;
        return 0;
}

UGB_API int ugb200_jpeg_decoder_set_upsampling(ugb200_jpeg_decoder *d, int mode)
{
        if (!d || (mode != UGB200_JPEG_UPSAMPLE_REPLICATE && mode != UGB200_JPEG_UPSAMPLE_FANCY)) {
                return -1;
        }
        d->upsampling = mode;
        return 0;
}

/// ugb200_jpeg_decode, ugb200_jpeg_decode_cs and ugb200_jpeg_decode_to: color_space is one of NATIVE, Y601, Y601FULL, Y709, AUTO; out_cs (the space of
/// UYVY, I420 and VUYA output) one of NATIVE, Y601, Y601FULL, Y709; gray_ok: one-component streams are decoded (ugb200_jpeg_decode_to), else -4 as ever
static int decode(ugb200_jpeg_decoder *d, const uint8_t *stream, size_t len, void *dst, int dst_is_device, long dst_pitch, int out_codec, int rshift, int gshift,
                  int bshift, int color_space, int out_cs, bool gray_ok = false)
{
        const long dst_pitch_arg = dst_pitch;
        if (!d || !stream || !dst || len > 0xFFFFFFF0u) {
                return -1;
        }
        if (out_codec != UGB_UYVY && out_codec != UGB_RGB && out_codec != UGB_RGBA && out_codec != UGB_VUYA && out_codec != UGB_I420) {
                return -4;
        }
        static const int timing = getenv("UGB200_JPEG_TIMING") ? atoi(getenv("UGB200_JPEG_TIMING")) : 0;  // 1: stage times of the host side on stderr; 2: + device stages
        const auto t_start = std::chrono::steady_clock::now();
        auto lap = [&](const char *what) {
                if (timing) {
                        if (what[0] == '+') {  // device stages: wait for the stream, so that the lap is the stage's own time (serialises the pipeline)
                                if (timing < 2) {
                                        return;
                                }
                                cudaStreamSynchronize(d->stream);
                        }
                        fprintf(stderr, "[jpeg decode] %-14s %8.3f ms\n", what, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_start).count());
                }
        };
        if (d->expect_w > 0) {  // the SOF dimensions are untrusted input and decide how much is written to dst: check them before anything else
                parsed head;
                const int hrc = parse_stream(stream, len, head, nullptr, false);
                if (hrc != 0) {
                        return hrc;
                }
                if (head.g.w != d->expect_w || head.g.h != d->expect_h) {
                        return -3;
                }
        }
        ugb200_jpeg_decoder::host_slot &H = d->hs[d->frame_no++ & 1];
        if (H.pending) {
                cudaEventSynchronize(H.uploaded);  // the uploads of the frame before last left this slot long ago
                cudaEventSynchronize(H.stream_up);
                H.pending = false;
        }
        lap("slot free");
        parsed P;
        P.seg_begin.swap(d->seg_begin), P.seg_end.swap(d->seg_end);  // last frame's capacity
        P.seg_begin.clear(), P.seg_end.clear();
        memset(H.tables, 0, sizeof(dec_tables));
        memcpy(H.tables->zz, kZigzag, 64);
        if (len > H.stream_cap) {  // pinned pages on the GPU's NUMA node (cuda_wrapper_malloc_host_near falls back to cudaMallocHost)
                if (H.stream) {
                        cuda_wrapper_free_host(H.stream);
                }
                H.stream = nullptr, H.stream_cap = 0;
                int device = 0;
                cudaGetDevice(&device);
                const size_t want = len + len / 4 + 4096;
                if (cuda_wrapper_malloc_host_near((void **) &H.stream, want, device) != 0) {
                        return -2;
                }
                H.stream_cap = want;
        }
        // Streams with ONE scan holding all components (UltraGrid's UYVY streams, interleaved RGB): the host reads the headers in front of the SOS and
        // copies the stream to pinned memory; the restart markers are found on the device (jpeg_marker_*_kernel).  Everything else - several scans,
        // whose later SOS headers lie behind entropy-coded data - takes the host scan below.
        size_t scan_data = 0;
        bool device_scan = false, multi = false;
        int rc = 0;
        const bool host_only = d->host_once;
        d->host_once = false;
        if (d->scan_mode != 1 && !host_only && len <= (1u << 30) && (d->scan_mode == 2 || len >= (1u << 20))) {
                rc = parse_stream(stream, len, P, H.tables, false, nullptr, &scan_data);
                device_scan = rc == 0 && P.g.nscans == 1 && P.g.s[0].ns == P.g.ncomp && scan_data > 0;
                if (rc == 0 && !device_scan && P.g.nscans == 1 && P.g.s[0].ns == 1 && P.g.s[0].comp[0] == 0 && P.g.ncomp == 3 && scan_data > 0 && P.have_q[P.g.c[1].tq] &&
                    P.have_q[P.g.c[2].tq]) {
                        // one scan per component, in component order, is what the first SOS promises (GPUJPEG's RGB streams): scans 2 and 3 are laid out as the
                        // host parser would lay them out, their table selectors come from the device, and the device checks the promise
                        dec_geom &g = P.g;
                        for (int id = 0; id < 4; ++id) {  // the kernel reads table id k of scans 2 and 3 from slot k: the first scan took slots by id
                                table_slot(P.hd, H.tables, id);
                        }
                        for (int j = 1; j < 3; ++j) {
                                dec_scan &S = g.s[j];
                                const dec_comp &c = g.c[j];
                                S.ns = 1, S.comp[0] = j, S.td[0] = 0, S.ta[0] = 2;  // table slots: the kernel takes the selectors from the device
                                S.mcux = ((g.w * c.h + g.hmax - 1) / g.hmax + 7) / 8;
                                S.nmcu = S.mcux * (((g.h * c.v + g.vmax - 1) / g.vmax + 7) / 8);
                                S.seg0 = g.s[j - 1].seg0 + g.s[j - 1].nseg;
                                S.nseg = g.ri ? (S.nmcu + g.ri - 1) / g.ri : 1;
                        }
                        g.nscans = 3;
                        device_scan = multi = true;
                }
                if (!device_scan) {  // start over on the host path (tables and geometry are rebuilt there)
                        P.g = dec_geom{}, P.adobe = -1, P.have_sof = false;
                        memset(P.have_q, 0, sizeof P.have_q);
                        P.hd = huff_defs{};
                        memset(H.tables, 0, sizeof(dec_tables));
                        memcpy(H.tables->zz, kZigzag, 64);
                }
        }
        std::vector<uint64_t> &markers = d->markers;
        if (device_scan) {
                const int nt = len > (4u << 20) ? kMaxScanThreads : len > (1u << 20) ? 4 : 1;
                if (nt == 1) {
                        stage_copy(H.stream, stream, len);
                } else {
                        const size_t chunk = (len / nt + 63) & ~(size_t) 63;
                        auto piece = [&](int i) {
                                const size_t lo = std::min(len, chunk * i), hi = i == nt - 1 ? len : std::min(len, chunk * (i + 1));
                                stage_copy(H.stream + lo, stream + lo, hi - lo);
                        };
                        d->pool.parallel(nt - 1, [&](int w) { piece(w + 1); }, [&] { piece(0); });
                }
                lap("stage");
        } else {
                // one pass over the caller's (pageable) buffer: copy it to the pinned staging buffer and collect the marker candidates, split over a
                // few threads when the stream is large (an 8K frame is 5-50 MB)
                markers.clear();
                collect_markers(stream, len, &d->pool, H.stream, markers, d->scan_part);
                lap("scan+stage");
                rc = parse_stream(stream, len, P, H.tables, true, &markers);
        }
        struct give_back {  // the segment vectors return to the decoder on every path out of this function
                parsed &p;
                ugb200_jpeg_decoder *dec;
                ~give_back() { p.seg_begin.swap(dec->seg_begin), p.seg_end.swap(dec->seg_end); }
        } give_back_guard{ P, d };
        if (rc != 0) {
                return rc;
        }
        lap("parse");
        P.g.ntables = multi ? 4 : 0;  // multi: scans 2 and 3 take their selectors from the device, any of slots 0..3 (zeroed when undefined)
        for (int k = 0; k < kTables; ++k) {
                P.g.ntables = P.hd.taken[k] ? k + 1 : P.g.ntables;
        }
        const dec_geom &g = P.g;
        if (g.ncomp == 1 && !gray_ok) {
                return -4;
        }
        const size_t nseg = multi ? (size_t) (g.s[2].seg0 + g.s[2].nseg) : device_scan ? (size_t) g.s[0].nseg : P.seg_begin.size();
        d->last_nseg = nseg;
        const long plane_bytes = (long) g.nblocks * 64;
        // Four components (R G B A): packed to RGBA when RGBA is asked for - with other shifts than (0, 8, 16) the packed frame then goes through the
        // RGBA -> RGBA line converter, as vc_copylineRGBA re-shifts it (alpha becomes 0xFF) - and to RGB (the first three planes) for any other
        // output, which then takes the routes of an RGB stream
        const int stream_codec = native_codec(P);
        const bool alpha = stream_codec == UGB_RGBA;
        const bool reshift = alpha && out_codec == UGB_RGBA && !(rshift == 0 && gshift == 8 && bshift == 16);
        const int native = alpha && out_codec != UGB_RGBA ? UGB_RGB : stream_codec;
        const long npitch = native == UGB_UYVY ? (long) ((g.w + 1) / 2) * 4 : native == UGB_RGB ? (long) g.w * 3 : (long) g.w * 4;
        const long opitch = out_codec == UGB_UYVY ? (long) ((g.w + 1) / 2) * 4 : out_codec == UGB_RGB ? (long) g.w * 3 : (long) g.w * 4;
        // RGB and RGBA output of a YCbCr stream in a colour space (ugb200_jpeg_decode_cs); AUTO takes the stream's, and one that declares RGB is not transformed
        const int cs = color_space == UGB200_JPEG_CS_AUTO ? declared_color_space(P) : color_space;
        if (cs < 0) {
                return cs;
        }
        const int conv_cs = (native == UGB_UYVY || native == UGB_VUYA) && (out_codec == UGB_RGB || out_codec == UGB_RGBA) && cs != UGB200_JPEG_CS_RGB ? cs
                                                                                                                                               : UGB200_JPEG_CS_NATIVE;
        // UYVY, I420 and VUYA output in a colour space (ugb200_jpeg_decode_to): a YCbCr stream's samples go through the matrix between the two spaces
        // before they are packed.  RGB and four-component streams reach YCbCr through UltraGrid's BT.709 line converters only.
        const bool ycc_out = out_codec == UGB_UYVY || out_codec == UGB_I420 || out_codec == UGB_VUYA;
        const bool ycc_stream = (native == UGB_UYVY || native == UGB_VUYA) && cs != UGB200_JPEG_CS_RGB;
        if (ycc_out && !ycc_stream && (out_cs == UGB200_JPEG_CS_Y601 || out_cs == UGB200_JPEG_CS_Y601FULL)) {
                return -4;
        }
        const bool matrix = ycc_out && ycc_stream && cs != UGB200_JPEG_CS_NATIVE && out_cs != UGB200_JPEG_CS_NATIVE && cs != out_cs;
        const ycc_matrix ym = matrix ? ycc_matrix_between(cs, out_cs) : ycc_matrix{};
        if (dst_pitch == 0) {
                dst_pitch = opitch;
        }
        if (!dgrow(H.d_stream, H.d_stream_cap, len + 16) || !dgrow(d->planes, d->planes_cap, (size_t) plane_bytes) || !dgrow(d->coef, d->coef_cap, (size_t) g.nblocks * 64) ||
            !dgrow(d->d_seg, d->seg_cap, 2 * nseg) || !dgrow(d->native, d->native_cap, (size_t) npitch * g.h + 64) || !hgrow(H.seg, H.seg_cap, 2 * nseg)) {
                return -2;
        }
        cudaStream_t s = d->stream;
        const uint32_t *dev_scans = nullptr;
        // the upload goes over the copy stream: it may start as soon as the kernels of the frame before last have read this slot's device copy, i.e. it
        // runs under the kernels of the previous frame; this frame's kernels wait for it
        uint8_t *const d_stream = H.d_stream;
        if (H.consumed_pending) {
                cudaStreamWaitEvent(d->copy, H.consumed, 0);
        }
        cudaMemcpyAsync(d_stream, H.stream, len, cudaMemcpyHostToDevice, d->copy);
        cudaEventRecord(H.stream_up, d->copy);
        cudaStreamWaitEvent(s, H.stream_up, 0);
        lap("+stream on the device");
        if (device_scan) {
                const unsigned pieces = (unsigned) ((len + kMarkThreads * 16 - 1) / (kMarkThreads * 16));
                if (!dgrow(d->d_marks, d->marks_cap, len / 2 + 2) || !dgrow(d->d_mark_cnt, d->mark_cnt_cap, (size_t) pieces + kMetaWords)) {
                        return -2;
                }
                uint32_t *meta = d->d_mark_cnt + pieces;
                dev_scans = multi ? meta : nullptr;
                jpeg_marker_count_kernel<<<pieces, kMarkThreads, 0, s>>>(d_stream, len, scan_data, d->d_mark_cnt);
                jpeg_marker_scan_kernel<<<1, 1024, 0, s>>>(d->d_mark_cnt, (int) pieces, meta);
                jpeg_marker_write_kernel<<<pieces, kMarkThreads, 0, s>>>(d_stream, len, scan_data, d->d_mark_cnt, d->d_marks, meta);
                if (multi) {
                        jpeg_marker_bounds_kernel<<<1, 32, 0, s>>>(d_stream, (uint32_t) len, d->d_marks, meta, (uint32_t) scan_data, g.nscans,
                                                                   (uint32_t) P.comp_id[0] | (uint32_t) P.comp_id[1] << 8 | (uint32_t) P.comp_id[2] << 16);
                        jpeg_marker_segments_multi_kernel<<<(unsigned) ((nseg + 255) / 256), 256, 0, s>>>(d->d_marks, meta, g.nscans, g.s[1].seg0, g.s[2].seg0, (int) nseg, d->d_seg,
                                                                                                           d->d_seg + nseg);
                        // The verdict must be known before the Huffman kernel is queued (an irregular stream is decoded by the host parser's rules instead).
                        // The wait covers the upload and four small kernels of THIS frame - and whatever the stream still holds of the frame before, which
                        // the device works on anyway; the host side of the next frame still overlaps this frame's Huffman and IDCT kernels.
                        if (cudaMemcpyAsync(d->h_flag, meta + kMetaError, 4, cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) {
                                return -2;
                        }
                        lap("verdict");
                        if (*d->h_flag != 0) {
                                d->host_once = true;
                                return decode(d, stream, len, dst, dst_is_device, dst_pitch_arg, out_codec, rshift, gshift, bshift, color_space, out_cs, gray_ok);
                        }
                } else {
                        jpeg_marker_segments_kernel<<<(unsigned) ((nseg + 255) / 256), 256, 0, s>>>(d->d_marks, meta, (uint32_t) scan_data, (uint32_t) len, (int) nseg, d->d_seg,
                                                                                                     d->d_seg + nseg);
                }
        } else {
                memcpy(H.seg, P.seg_begin.data(), nseg * 4), memcpy(H.seg + nseg, P.seg_end.data(), nseg * 4);
                cudaMemcpyAsync(d->d_seg, H.seg, 2 * nseg * 4, cudaMemcpyHostToDevice, s);
        }
        cudaMemcpyAsync(d->d_tables, H.tables, sizeof(dec_tables), cudaMemcpyHostToDevice, s);
        cudaEventRecord(H.uploaded, s);
        H.pending = true;
        lap("uploads queued");
        lap("+segments on the device");
        // Does every block of the coefficient array belong to exactly one scan's MCU grid?  (Interleaved scans cover the padded planes by construction; a
        // one-component scan covers ceil(w_c / 8) x ceil(h_c / 8) blocks, which is the whole plane only without MCU padding; a component no scan names - a
        // truncated multi-scan stream - is covered by nobody.)  Then the Huffman kernel writes whole blocks and the array is not cleared.
        bool full = true;
        {
                int seen[4] = { 0, 0, 0, 0 };
                for (int j = 0; j < g.nscans; ++j) {
                        const dec_scan &S = g.s[j];
                        for (int k = 0; k < S.ns; ++k) {
                                ++seen[S.comp[k]];
                        }
                        if (S.ns == 1) {
                                const dec_comp &c = g.c[S.comp[0]];
                                full = full && S.mcux == c.bw && S.nmcu == c.bw * c.bh;
                        }
                }
                for (int i = 0; i < g.ncomp; ++i) {
                        full = full && seen[i] == 1;
                }
        }
        const unsigned hgrid = (unsigned) ((nseg + kHuffThreads - 1) / kHuffThreads);
        const size_t hsmem = kTablesSmem + (size_t) kHuffThreads * 128;
        // Huffman route: restart segments of few MCUs keep one thread each; longer ones (every scan without DRI) are decoded by the self-synchronising
        // route, whose parallelism does not depend on the stream's restart interval.  The segment length in MCUs is the same for every scan of a stream.
        const bool sync = d->sync_mode == 2 || (d->sync_mode == 0 && (g.ri == 0 || g.ri >= kSyncMinMcus));
        d->last_sync_ctr = nullptr, d->last_sync_scans = 0;
        if (sync) {
                const int sub = d->sync_bytes;
                const size_t cap = len / (size_t) sub + nseg + 1;  // a segment of n bytes has at most n / sub + 1 subsequences
                if (d->sync_grid == 0) {
                        int dev = 0, sms = 0, per_sm = 0;
                        cudaGetDevice(&dev);
                        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
                        cudaFuncSetAttribute(jpeg_sync_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) kTablesSmem);
                        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, jpeg_sync_kernel, kSyncThreads, kTablesSmem);
                        d->sync_grid = sms * std::max(1, per_sm);
                }
                const int grid = (int) std::min((size_t) d->sync_grid, (cap + kSyncThreads - 1) / kSyncThreads);
                const size_t words = (nseg + 1) + 4 * cap + 2 * kSyncVals * cap + cap + (size_t) kSyncVals * grid + 8;
                if (cap > 0xFFFFFFF0u || !dgrow(d->d_sync, d->sync_cap, words)) {
                        return -2;
                }
                sync_bufs B;
                uint32_t *w = d->d_sync;
                B.sub_first = w, w += nseg + 1;
                B.entry = (sync_point *) w, w += 2 * cap;
                B.exitp = (sync_point *) w, w += 2 * cap;
                B.res = w, w += kSyncVals * cap;
                B.scan = w, w += kSyncVals * cap;
                B.dirty = w, w += cap;
                B.cta = w, w += (size_t) kSyncVals * grid;
                B.ctr = w;
                cudaMemsetAsync(B.ctr, 0, 8 * 4, s);
                jpeg_sync_table_kernel<<<1, 1024, 0, s>>>(d->d_seg, d->d_seg + nseg, (int) nseg, sub, B.sub_first);
                const uint8_t *a_stream = d_stream;
                const uint32_t *a_begin = d->d_seg, *a_end = d->d_seg + nseg;
                int a_nseg = (int) nseg;
                const dec_tables *a_tables = d->d_tables;
                dec_geom a_g = g;
                uint32_t a_cap = (uint32_t) cap;
                void *args[] = { &a_stream, &a_begin, &a_end, &a_nseg, (void *) &sub, &a_tables, &a_g, &dev_scans, &B, &a_cap };
                if (cudaLaunchCooperativeKernel((const void *) jpeg_sync_kernel, grid, kSyncThreads, args, kTablesSmem, s) != cudaSuccess) {
                        return -2;
                }
                lap("+sync rounds + scan");
                const unsigned wgrid = (unsigned) ((cap + kHuffThreads - 1) / kHuffThreads);
                if (full) {
                        jpeg_sync_write_kernel<true><<<wgrid, kHuffThreads, hsmem, s>>>(d_stream, d->d_seg, d->d_seg + nseg, (int) nseg, sub, d->d_tables, g, d->coef,
                                                                                       dev_scans, B, (uint32_t) cap);
                } else {
                        cudaMemsetAsync(d->coef, 0, (size_t) g.nblocks * 128, s);
                        jpeg_sync_write_kernel<false><<<wgrid, kHuffThreads, hsmem, s>>>(d_stream, d->d_seg, d->d_seg + nseg, (int) nseg, sub, d->d_tables, g, d->coef,
                                                                                        dev_scans, B, (uint32_t) cap);
                }
                lap("+sync write");
                d->last_sync_ctr = B.ctr, d->last_sync_scans = g.nscans;
        } else if (full) {
                jpeg_decode_huffman_kernel<true><<<hgrid, kHuffThreads, hsmem, s>>>(d_stream, d->d_seg, d->d_seg + nseg, d->d_tables, g, d->coef, dev_scans);
        } else {
                cudaMemsetAsync(d->coef, 0, (size_t) g.nblocks * 128, s);
                lap("+coefficients cleared");
                jpeg_decode_huffman_kernel<false><<<hgrid, kHuffThreads, hsmem, s>>>(d_stream, d->d_seg, d->d_seg + nseg, d->d_tables, g, d->coef, dev_scans);
        }
        cudaEventRecord(H.consumed, s);  // nothing behind this kernel reads the stream
        H.consumed_pending = true;
        const bool direct = native == out_codec && dst_is_device && !reshift;
        uint8_t *nat = direct ? (uint8_t *) dst : d->native;
        // the caller's RGB / RGBA in a colour space, or any output of the fused kernel: into dst when it is on the device, else into staging and across
        const bool fused = native == UGB_UYVY, to_out = conv_cs != UGB200_JPEG_CS_NATIVE || (fused && (out_codec == UGB_RGB || out_codec == UGB_RGBA));
        if (to_out && !dst_is_device && !dgrow(d->staging, d->staging_cap, (size_t) opitch * g.h + 64)) {
                return -2;
        }
        uint8_t *const conv = dst_is_device ? (uint8_t *) dst : d->staging;
        const long cpitch = dst_is_device ? dst_pitch : opitch;
        const conv_params cp = { rshift, gshift, bshift, 0 };
        // I420 of a 4:2:2, 4:2:0 or grayscale stream: the fused kernel writes the three tight planes (GPUJPEG_420_U8_P0P1P2, gpujpeg.c:113-116) itself
        const bool planar = fused && out_codec == UGB_I420;
        const size_t i420_bytes = (size_t) g.w * g.h + 2 * (size_t) ((g.w + 1) / 2) * ((g.h + 1) / 2);
        if (planar && !dst_is_device && !dgrow(d->staging, d->staging_cap, i420_bytes + 64)) {
                return -2;
        }
        if (fused) {  // 4:2:2 and 4:2:0: IDCT, chroma replication and packing (or conversion) in one kernel, no component planes
                const bool uyvy_out = !to_out;
                uint8_t *o = planar ? (dst_is_device ? (uint8_t *) dst : d->staging) : uyvy_out ? nat : conv;
                const long op = planar ? g.w : uyvy_out ? (direct ? dst_pitch : npitch) : cpitch;
                const bool gray = g.ncomp == 1;
                const dim3 grid((unsigned) (((gray ? (g.c[0].bw + 1) / 2 : g.c[1].bw) + 31) / 32), (unsigned) (gray ? g.c[0].bh : g.c[1].bh));
                const bool vec = !(15 & (size_t) o) && !(op & 15);
                const int kind = planar ? 8 : uyvy_out ? 0 : out_codec == UGB_RGB ? (conv_cs == UGB200_JPEG_CS_NATIVE ? UGB200_JPEG_CS_Y709 : conv_cs) : 4 + conv_cs;
                // interpolated chroma (ugb200_jpeg_decoder_set_upsampling): RGB / RGBA of a 4:2:2 or 4:2:0 stream in a colour space only
                const bool fancy = d->upsampling == UGB200_JPEG_UPSAMPLE_FANCY && !gray && conv_cs != UGB200_JPEG_CS_NATIVE;
                auto launch = [&](auto v, auto gr) {
                        constexpr int V = decltype(v)::value;
                        constexpr bool G = decltype(gr)::value;
                        constexpr int NT = 32 * (G ? 2 : 2 * V + 2);
                        auto run = [&](auto e, auto m) {
                                jpeg_idct_packed_kernel<V, typename decltype(e)::type, decltype(m)::value, G><<<grid, NT, 0, s>>>(d->coef, d->d_tables, g, o, op, vec, cp, ym);
                        };
                        const std::false_type plain;
                        if constexpr (!G) {
                                if (fancy) {
                                        switch (kind) {
                                        case UGB200_JPEG_CS_Y709: run(type_tag<epi_fancy<ycbcr_709, false>>(), plain); break;
                                        case UGB200_JPEG_CS_Y601: run(type_tag<epi_fancy<ycbcr_601, false>>(), plain); break;
                                        case UGB200_JPEG_CS_Y601FULL: run(type_tag<epi_fancy<ycbcr_601_full, false>>(), plain); break;
                                        case 4 + UGB200_JPEG_CS_Y709: run(type_tag<epi_fancy<ycbcr_709, true>>(), plain); break;
                                        case 4 + UGB200_JPEG_CS_Y601: run(type_tag<epi_fancy<ycbcr_601, true>>(), plain); break;
                                        default: run(type_tag<epi_fancy<ycbcr_601_full, true>>(), plain); break;
                                        }
                                        return;
                                }
                        }
                        switch (kind) {
                        case 0: matrix ? run(type_tag<epi_uyvy>(), std::true_type()) : run(type_tag<epi_uyvy>(), plain); break;
                        case UGB200_JPEG_CS_Y709: run(type_tag<epi_rgb>(), plain); break;
                        case UGB200_JPEG_CS_Y601: run(type_tag<epi_cs_rgb<ycbcr_601>>(), plain); break;
                        case UGB200_JPEG_CS_Y601FULL: run(type_tag<epi_cs_rgb<ycbcr_601_full>>(), plain); break;
                        case 4 + UGB200_JPEG_CS_NATIVE: run(type_tag<epi_rgba>(), plain); break;
                        case 4 + UGB200_JPEG_CS_Y709: run(type_tag<epi_cs_rgba<ycbcr_709>>(), plain); break;
                        case 4 + UGB200_JPEG_CS_Y601: run(type_tag<epi_cs_rgba<ycbcr_601>>(), plain); break;
                        case 8: matrix ? run(type_tag<epi_i420>(), std::true_type()) : run(type_tag<epi_i420>(), plain); break;
                        default: run(type_tag<epi_cs_rgba<ycbcr_601_full>>(), plain); break;
                        }
                };
                if (gray) {
                        launch(std::integral_constant<int, 1>(), std::true_type());
                } else if (g.c[0].v == 2) {
                        launch(std::integral_constant<int, 2>(), std::false_type());
                } else {
                        launch(std::integral_constant<int, 1>(), std::false_type());
                }
        } else {
                jpeg_idct_kernel<<<(g.nblocks + 127) / 128, 128, 0, s>>>(d->coef, d->d_tables, g, d->planes);
                if (matrix) {
                        jpeg_planes_ycc_kernel<<<(unsigned) (((long) g.c[0].bw * g.c[0].bh * 16 + 255) / 256), 256, 0, s>>>(d->planes, g, ym);
                }
                if (to_out) {  // 4:4:4 YCbCr in a colour space: per pixel over the planes
                        const dim3 grid((unsigned) ((g.w + 255) / 256), (unsigned) g.h);
                        const bool rgba = out_codec == UGB_RGBA;
                        if (conv_cs == UGB200_JPEG_CS_Y709) {
                                rgba ? jpeg_planes_cs_kernel<ycbcr_709, true><<<grid, 256, 0, s>>>(d->planes, g, conv, cpitch, cp)
                                     : jpeg_planes_cs_kernel<ycbcr_709, false><<<grid, 256, 0, s>>>(d->planes, g, conv, cpitch, cp);
                        } else if (conv_cs == UGB200_JPEG_CS_Y601) {
                                rgba ? jpeg_planes_cs_kernel<ycbcr_601, true><<<grid, 256, 0, s>>>(d->planes, g, conv, cpitch, cp)
                                     : jpeg_planes_cs_kernel<ycbcr_601, false><<<grid, 256, 0, s>>>(d->planes, g, conv, cpitch, cp);
                        } else {
                                rgba ? jpeg_planes_cs_kernel<ycbcr_601_full, true><<<grid, 256, 0, s>>>(d->planes, g, conv, cpitch, cp)
                                     : jpeg_planes_cs_kernel<ycbcr_601_full, false><<<grid, 256, 0, s>>>(d->planes, g, conv, cpitch, cp);
                        }
                }
        }
        if (cudaGetLastError() != cudaSuccess) {
                return -2;
        }
        lap("kernels queued");
        lap("+huffman + idct");
        if (planar) {
                if (dst_is_device) {
                        return 0;
                }
                return cudaMemcpyAsync(dst, d->staging, i420_bytes, cudaMemcpyDeviceToHost, s) == cudaSuccess && cudaStreamSynchronize(s) == cudaSuccess ? 0 : -2;
        }
        if (to_out) {
                if (dst_is_device) {
                        return 0;
                }
                return cudaMemcpy2DAsync(dst, dst_pitch, conv, cpitch, opitch, g.h, cudaMemcpyDeviceToHost, s) == cudaSuccess && cudaStreamSynchronize(s) == cudaSuccess ? 0 : -2;
        }
        if (!fused) {  // component planes -> the stream's native packed format
                struct ugb200_from_planar_data fp;
                memset(&fp, 0, sizeof fp);
                fp.width = g.w, fp.height = g.h, fp.out_data = nat, fp.out_pitch = (unsigned) (direct ? dst_pitch : npitch);
                for (int i = 0; i < 3; ++i) {
                        fp.in_data[i] = d->planes + g.c[i].plane_off, fp.in_linesize[i] = (unsigned) (g.c[i].bw * 8);
                }
                fp.in_depth = 8;
                if (alpha) {  // planes in G, B, R, A order (from_planar.c:335-366); all four have the same line size
                        for (int i = 0; i < 4; ++i) {
                                const dec_comp &c = g.c[i == 3 ? 3 : (i + 1) % 3];
                                fp.in_data[i] = d->planes + c.plane_off, fp.in_linesize[i] = (unsigned) (c.bw * 8);
                        }
                }
                if (alpha) {
                        rc = native == UGB_RGBA ? ugb200_gbrap_to_rgba(&fp, s) : ugb200_gbrap_to_rgb(&fp, s);
                } else if (native == UGB_RGB) {
                        rc = ugb200_rgbpXX_to_rgb(&fp, s);
                } else {
                        rc = ugb200_yuv444p_to_vuya(&fp, s);
                }
                if (rc != 0) {
                        return rc;
                }
        }
        if (direct) {
                return 0;
        }
        if (out_codec == UGB_I420) {  // GPUJPEG_420_U8_P0P1P2 (gpujpeg.c:113-116): Y, then Cb, then Cr plane, tightly packed
                const size_t cw = (size_t) (g.w + 1) / 2, chh = (size_t) (g.h + 1) / 2, total = (size_t) g.w * g.h + 2 * cw * chh;
                uint8_t *uy = nat;
                long uy_pitch = npitch;
                if (native != UGB_UYVY) {
                        if (!ugb200_pixfmt_supported(native, UGB_UYVY) || !dgrow(d->staging, d->staging_cap, (size_t) ((g.w + 1) / 2) * 4 * g.h + total + 64)) {
                                return -4;
                        }
                        uy = d->staging, uy_pitch = (long) ((g.w + 1) / 2) * 4;
                        rc = ugb200_pixfmt_convert(native, UGB_UYVY, uy, uy_pitch, nat, npitch, (int) uy_pitch, g.h, (long) npitch * g.h, 0, 8, 16, s);
                        if (rc != 0) {
                                return rc;
                        }
                } else if (!dgrow(d->staging, d->staging_cap, total + 64)) {
                        return -2;
                }
                uint8_t *planes_out = dst_is_device ? (uint8_t *) dst : d->staging + (native != UGB_UYVY ? (size_t) uy_pitch * g.h : 0);
                struct ugb200_to_planar_data tp;
                memset(&tp, 0, sizeof tp);
                tp.width = g.w, tp.height = g.h, tp.in_data = uy;
                tp.out_data[0] = planes_out, tp.out_data[1] = planes_out + (size_t) g.w * g.h, tp.out_data[2] = tp.out_data[1] + cw * chh;
                tp.out_linesize[0] = (unsigned) g.w, tp.out_linesize[1] = tp.out_linesize[2] = (unsigned) cw;
                if (uy_pitch != (long) ((g.w + 1) / 2) * 4) {
                        return -4;
                }
                rc = ugb200_uyvy_to_i420(&tp, s);
                if (rc != 0 || dst_is_device) {
                        return rc;
                }
                return cudaMemcpyAsync(dst, planes_out, total, cudaMemcpyDeviceToHost, s) == cudaSuccess && cudaStreamSynchronize(s) == cudaSuccess ? 0 : -2;
        }
        // native -> requested codec (UltraGrid's own line converters), then to the caller
        uint8_t *result = nat;
        long rpitch = npitch;
        if (native != out_codec || reshift) {
                if (!ugb200_pixfmt_supported(native, out_codec)) {
                        return -4;
                }
                uint8_t *conv;
                if (dst_is_device) {
                        conv = (uint8_t *) dst, rpitch = dst_pitch;
                } else {
                        if (!dgrow(d->staging, d->staging_cap, (size_t) opitch * g.h + 64)) {
                                return -2;
                        }
                        conv = d->staging, rpitch = opitch;
                }
                const int len_out = out_codec == UGB_UYVY ? ((g.w + 1) / 2) * 4 : out_codec == UGB_RGB ? g.w * 3 : g.w * 4;
                rc = ugb200_pixfmt_convert(native, out_codec, conv, rpitch, nat, npitch, len_out, g.h, (long) npitch * g.h, rshift, gshift, bshift, s);
                if (rc != 0) {
                        return rc;
                }
                result = conv;
                if (dst_is_device) {
                        return 0;
                }
        }
        if (dst_is_device) {
                return cudaMemcpy2DAsync(dst, dst_pitch, result, rpitch, opitch, g.h, cudaMemcpyDeviceToDevice, s) == cudaSuccess ? 0 : -2;
        }
        if (cudaMemcpy2DAsync(dst, dst_pitch, result, rpitch, opitch, g.h, cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) {
                return -2;
        }
        return 0;
}

UGB_API int ugb200_jpeg_decode(ugb200_jpeg_decoder *d, const uint8_t *stream, size_t len, void *dst, int dst_is_device, long dst_pitch, int out_codec,
                               int rshift, int gshift, int bshift)
{
        return decode(d, stream, len, dst, dst_is_device, dst_pitch, out_codec, rshift, gshift, bshift, UGB200_JPEG_CS_NATIVE, UGB200_JPEG_CS_NATIVE);
}

UGB_API int ugb200_jpeg_decode_cs(ugb200_jpeg_decoder *d, const uint8_t *stream, size_t len, void *dst, int dst_is_device, long dst_pitch, int out_codec,
                                  int rshift, int gshift, int bshift, int color_space)
{
        if (color_space != UGB200_JPEG_CS_NATIVE && color_space != UGB200_JPEG_CS_Y601 && color_space != UGB200_JPEG_CS_Y601FULL &&
            color_space != UGB200_JPEG_CS_Y709 && color_space != UGB200_JPEG_CS_AUTO) {
                return -1;
        }
        return decode(d, stream, len, dst, dst_is_device, dst_pitch, out_codec, rshift, gshift, bshift, color_space, UGB200_JPEG_CS_NATIVE);
}

UGB_API int ugb200_jpeg_decode_to(ugb200_jpeg_decoder *d, const uint8_t *stream, size_t len, void *dst, int dst_is_device, long dst_pitch, int out_codec,
                                  int rshift, int gshift, int bshift, int stream_cs, int out_cs)
{
        if (stream_cs != UGB200_JPEG_CS_NATIVE && stream_cs != UGB200_JPEG_CS_Y601 && stream_cs != UGB200_JPEG_CS_Y601FULL && stream_cs != UGB200_JPEG_CS_Y709 &&
            stream_cs != UGB200_JPEG_CS_AUTO) {
                return -1;
        }
        if (out_cs != UGB200_JPEG_CS_NATIVE && out_cs != UGB200_JPEG_CS_Y601 && out_cs != UGB200_JPEG_CS_Y601FULL && out_cs != UGB200_JPEG_CS_Y709) {
                return -1;
        }
        return decode(d, stream, len, dst, dst_is_device, dst_pitch, out_codec, rshift, gshift, bshift, stream_cs, out_cs, true);
}

}  // extern "C"
