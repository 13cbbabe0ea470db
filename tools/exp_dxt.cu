// Experiment harness (not product code): where the time of the fused UYVY -> DXT1 encode goes, and the launch shapes / loop structures it
// was chosen from.  Every variant is timed with CUDA events on four rotating 8K frames (265 MB, more than L2) and compared byte for byte
// with the output of the shipped entry point.
//   shipped             ugb200_uyvy_to_dxt1_async as the library launches it (dxt_uyvy_kernel<1,2,false>: skew_t64_m12)
//   oneshot_bB_tT_mM    one thread = B blocks, T-thread CTAs, __launch_bounds__(T, M), one CTA per T B-block strip of a block row
//   compute_only_*      the one-shot kernel with its input words made from the thread index and a runtime seed (no loads)
//   memory_only_*       the one-shot loads and store with trivial work in between
//   skew_tT_mM          one-shot, the two blocks of a thread one phase apart (dxt1_encode_uyvy_pair_skewed)
//   persist_*           persistent grid (SMs x resident CTAs), static round-robin of 64-block items per warp; pf1 = next item loaded into
//                       registers before the current one is encoded, pf0 = no look-ahead, l2 = next item prefetched into L2 only
// Build: nvcc -O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a --expt-relaxed-constexpr -o tools/exp_dxt tools/exp_dxt.cu
// Run:   tools/exp_dxt [rounds, default 60]
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../ultragrid_b200/csrc/dxt_kernels.cu"

namespace ugb {

enum { ENCODE = 0, COMPUTE_ONLY = 1, MEMORY_ONLY = 2, SKEWED = 3 };

template <int BPT>
__device__ __forceinline__ void load_words(const uint8_t *p, long step, uint32_t (&w)[4][2 * BPT])
{
#pragma unroll
        for (int y = 0; y < 4; ++y, p += step) {
                if (BPT == 1) {
                        const uint2 v = ld_stream_v2(p);
                        w[y][0] = v.x, w[y][1] = v.y;
                } else {
#pragma unroll
                        for (int q = 0; q < BPT / 2; ++q) {
                                const uint4 v = ld_stream_v4(p + 16 * q);
                                w[y][4 * q] = v.x, w[y][4 * q + 1] = v.y, w[y][4 * q + 2] = v.z, w[y][4 * q + 3] = v.w;
                        }
                }
        }
}

template <int BPT, int MODE>
__device__ __forceinline__ void encode_store(const uint32_t (&w)[4][2 * BPT], uint2 *o, bool store = true)
{
        uint2 res[BPT];
        if (MODE == MEMORY_ONLY) {
#pragma unroll
                for (int k = 0; k < BPT; ++k) {
                        res[k] = make_uint2(w[0][2 * k] ^ w[1][2 * k] ^ w[2][2 * k] ^ w[3][2 * k], w[0][2 * k + 1] ^ w[1][2 * k + 1] ^ w[2][2 * k + 1] ^ w[3][2 * k + 1]);
                }
        } else if (MODE == SKEWED) {
                static_assert(MODE != SKEWED || BPT == 2, "the skewed encode takes two blocks");
                const uint4 v[4] = { make_uint4(w[0][0], w[0][1], w[0][2], w[0][3]), make_uint4(w[1][0], w[1][1], w[1][2], w[1][3]),
                                     make_uint4(w[2][0], w[2][1], w[2][2], w[2][3]), make_uint4(w[3][0], w[3][1], w[3][2], w[3][3]) };
                const uint4 r = dxt1_encode_uyvy_pair_skewed(v);
                res[0] = make_uint2(r.x, r.y), res[BPT - 1] = make_uint2(r.z, r.w);
        } else {
#pragma unroll
                for (int k = 0; k < BPT; ++k) {
                        const uint32_t wk[4][2] = { { w[0][2 * k], w[0][2 * k + 1] }, { w[1][2 * k], w[1][2 * k + 1] },
                                                    { w[2][2 * k], w[2][2 * k + 1] }, { w[3][2 * k], w[3][2 * k + 1] } };
                        res[k] = dxt1_encode_uyvy_packed(wk);
                }
        }
        if (!store) {
                return;
        }
        if (BPT == 1) {
                *o = res[0];
        } else {
#pragma unroll
                for (int k = 0; k < BPT; k += 2) {
                        *(uint4 *) (o + k) = make_uint4(res[k].x, res[k].y, res[k + 1].x, res[k + 1].y);
                }
        }
}

/// one-shot grid, as shipped: x over groups of BPT blocks of a block row, y = block row
template <int BPT, int TPB, int MINB, int MODE>
__global__ void __launch_bounds__(TPB, MINB) exp_oneshot_kernel(const uint8_t *__restrict__ src, uint2 *__restrict__ out, int wb, int h, long pitch, uint32_t seed)
{
        const int gx = blockIdx.x * blockDim.x + threadIdx.x;
        const int by = blockIdx.y;
        if (gx >= wb / BPT) {
                return;
        }
        uint32_t w[4][2 * BPT];
        if (MODE == COMPUTE_ONLY) {  // words the compiler cannot know: a hash of the position and a runtime seed
                const uint32_t base = ((uint32_t) by * 0x9E3779B1u + (uint32_t) gx) * 0x85EBCA6Bu ^ seed;
#pragma unroll
                for (int y = 0; y < 4; ++y) {
#pragma unroll
                        for (int k = 0; k < 2 * BPT; ++k) {
                                w[y][k] = base * (2u * (8 * y + k) + 1u) + seed;
                        }
                }
        } else {
                load_words<BPT>(src + (long) (by * 4) * pitch + (long) gx * (8 * BPT), pitch, w);
        }
        encode_store<BPT, MODE>(w, out + ((long) by * wb + (long) gx * BPT));
}

/// persistent grid, two blocks per thread: warp g of W takes the items (32 pairs of one block row) g, g + W, ...; the look-ahead (PF) and the
/// encode (MODE) are knobs
template <int TPB, int MINB, int MODE, int PF>
__global__ void __launch_bounds__(TPB, MINB) exp_persist_kernel(const uint8_t *__restrict__ src, uint2 *__restrict__ out, int wb, int h, long pitch, uint32_t)
{
        const int pairs = wb / 2, segs = (pairs + 31) / 32, hb = h / 4;
        const int lane = threadIdx.x & 31;
        const int warp = blockIdx.x * (TPB / 32) + (threadIdx.x >> 5), nwarps = gridDim.x * (TPB / 32);
        const int dby = nwarps / segs, dseg = nwarps - dby * segs;
        int by = warp / segs, seg = warp - by * segs;
        auto addr = [&](int row, int item) { return src + (long) (4 * row) * pitch + (long) min(item * 32 + lane, pairs - 1) * 16; };
        uint32_t nxt[4][4];
        if (PF == 1 && by < hb) {
                load_words<2>(addr(by, seg), pitch, nxt);
        }
        while (by < hb) {
                uint32_t w[4][4];
                if (PF == 1) {
#pragma unroll
                        for (int y = 0; y < 4; ++y) {
#pragma unroll
                                for (int k = 0; k < 4; ++k) {
                                        w[y][k] = nxt[y][k];
                                }
                        }
                } else {
                        load_words<2>(addr(by, seg), pitch, w);
                }
                const int gx = seg * 32 + lane, cur = by;
                seg += dseg, by += dby;
                if (seg >= segs) {
                        seg -= segs, ++by;
                }
                if (by < hb) {
                        if (PF == 1) {
                                load_words<2>(addr(by, seg), pitch, nxt);
                        } else if (PF == 2) {
                                const uint8_t *p = addr(by, seg);
#pragma unroll
                                for (int y = 0; y < 4; ++y, p += pitch) {
                                        asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
                                }
                        }
                }
                encode_store<2, MODE>(w, out + ((long) cur * wb + 2 * gx), gx < pairs);
        }
}

__global__ void fill_kernel(uint32_t *p, long nwords, uint32_t seed, int w_words, int h)
{
        for (long i = (long) blockIdx.x * blockDim.x + threadIdx.x; i < nwords; i += (long) gridDim.x * blockDim.x) {
                uint32_t x = (uint32_t) i * 2654435761u ^ seed;
                x ^= x << 13, x ^= x >> 17, x ^= x << 5;
                x *= 0x9E3779B1u;
                x ^= x >> 15;
                const int row = (int) (i / w_words);
                if (seed == 1u) {  // frame 0 also carries flat and smooth regions (flat-block path, near-flat blocks)
                        if (row < h / 16) {
                                x = 0x80808080u;
                        } else if (row < h / 8) {
                                const uint32_t v = (uint32_t) ((i % w_words) * 255 / w_words);
                                x = 0x80008000u | v << 8 | ((v + (row & 1)) & 0xff) << 24;
                        } else if (row < h / 4) {
                                x = (x & 0x03030303u) + 0x40804080u;  // low-amplitude noise
                        }
                }
                p[i] = x;
        }
}

}  // namespace ugb

typedef void (*kern_t)(const uint8_t *, uint2 *, int, int, long, uint32_t);
struct variant {
        std::string name;
        int bpt, tpb;
        bool persistent;  // grid = SMs x resident CTAs
        int mode;
        kern_t kern;      // nullptr: the shipped entry point
        std::vector<float> us;
};

#define O(B, T, M) { "oneshot_b" #B "_t" #T "_m" #M, B, T, false, ugb::ENCODE, ugb::exp_oneshot_kernel<B, T, M, ugb::ENCODE>, {} }
#define C(B, T, M) { "compute_only_b" #B "_t" #T "_m" #M, B, T, false, ugb::COMPUTE_ONLY, ugb::exp_oneshot_kernel<B, T, M, ugb::COMPUTE_ONLY>, {} }
#define MO(B, T, M) { "memory_only_b" #B "_t" #T "_m" #M, B, T, false, ugb::MEMORY_ONLY, ugb::exp_oneshot_kernel<B, T, M, ugb::MEMORY_ONLY>, {} }
#define K(T, M) { "skew_t" #T "_m" #M, 2, T, false, ugb::SKEWED, ugb::exp_oneshot_kernel<2, T, M, ugb::SKEWED>, {} }
#define P(T, M, PF) { "persist_t" #T "_m" #M "_pf" #PF, 2, T, true, ugb::ENCODE, ugb::exp_persist_kernel<T, M, ugb::ENCODE, PF>, {} }
#define PK(T, M) { "persist_skew_t" #T "_m" #M "_pf1", 2, T, true, ugb::SKEWED, ugb::exp_persist_kernel<T, M, ugb::SKEWED, 1>, {} }
#define PM(T, M) { "persist_memory_only_t" #T "_m" #M, 2, T, true, ugb::MEMORY_ONLY, ugb::exp_persist_kernel<T, M, ugb::MEMORY_ONLY, 1>, {} }

int main(int argc, char **argv)
{
        const int W = 7680, H = 4320, rounds = argc > 1 ? atoi(argv[1]) : 60;
        const long frame = (long) W * H * 2;
        std::vector<variant> vs = {
                { "shipped", 2, 0, false, ugb::ENCODE, nullptr, {} },
                C(2, 64, 12), MO(2, 64, 12), PM(128, 4),
                O(2, 64, 12), O(2, 64, 10), O(2, 128, 5), O(2, 128, 4), O(1, 64, 12), O(4, 64, 8),
                K(64, 12), K(64, 10), K(128, 5), K(128, 4),
                P(128, 4, 1), P(256, 2, 1), P(128, 5, 2), PK(128, 4),
        };
        int dev = 0, sms = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaDeviceProp prop;
        cudaGetDeviceProperties(&prop, dev);
        printf("device %s, %d SMs\n", prop.name, sms);

        uint8_t *src[4];
        uint2 *out, *ref;
        for (int i = 0; i < 4; ++i) {
                cudaMalloc(&src[i], frame + 256);
                ugb::fill_kernel<<<sms * 8, 256>>>((uint32_t *) src[i], frame / 4, (uint32_t) (i + 1), W * 2 / 4, H);
        }
        const size_t out_bytes = (size_t) W * H / 2;
        cudaMalloc(&out, out_bytes);
        cudaMalloc(&ref, out_bytes);
        std::vector<uint8_t> h_ref(out_bytes), h_out(out_bytes);
        ugb200_uyvy_to_dxt1_async(src[0], ref, W, H, 0, nullptr);
        if (cudaDeviceSynchronize() != cudaSuccess) {
                printf("setup failed: %s\n", cudaGetErrorString(cudaGetLastError()));
                return 1;
        }
        cudaMemcpy(h_ref.data(), ref, out_bytes, cudaMemcpyDeviceToHost);
        auto launch = [&](const variant &v, dim3 grid, int i) {
                if (!v.kern) {
                        ugb200_uyvy_to_dxt1_async(src[i & 3], out, W, H, 0, nullptr);
                } else {
                        v.kern<<<grid, v.tpb>>>(src[i & 3], out, W / 4, H, (long) W * 2, 0x9E3779B9u * (i + 1));
                }
        };
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0), cudaEventCreate(&e1);
        const int wb = W / 4, hb = H / 4;
        std::vector<dim3> grids;
        for (variant &v : vs) {  // attributes, grid, bit-exactness, warm-up
                int occ = 0, regs = 0;
                size_t spill = 0;
                if (v.kern) {
                        cudaFuncAttributes fa;
                        cudaFuncGetAttributes(&fa, (const void *) v.kern);
                        regs = fa.numRegs, spill = fa.localSizeBytes;
                        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (const void *) v.kern, v.tpb, 0);
                }
                grids.push_back(v.persistent ? dim3(sms * occ) : dim3((wb / v.bpt + v.tpb - 1) / std::max(v.tpb, 1), hb));
                cudaMemset(out, 0xEE, out_bytes);
                launch(v, grids.back(), 0);
                cudaMemcpy(h_out.data(), out, out_bytes, cudaMemcpyDeviceToHost);
                const char *check = v.mode == ugb::ENCODE || v.mode == ugb::SKEWED ? (memcmp(h_out.data(), h_ref.data(), out_bytes) ? "MISMATCH" : "bit-exact") : "-";
                const cudaError_t err = cudaGetLastError();
                printf("%-30s regs %3d spill %3zu B  CTAs/SM %2d  warps/SM %2d  %s %s\n", v.name.c_str(), regs, spill, occ, occ * v.tpb / 32, check,
                       err == cudaSuccess ? "" : cudaGetErrorString(err));
        }
        // The card is power-capped, so its SM clock wanders by tens of percent over seconds.  Variants are therefore timed in short windows
        // (`iters` launches, a few ms), one window per variant per round with the starting variant rotated, over many rounds: every variant
        // sees the same spread of clocks, and the median over rounds compares them.
        const int nv = (int) vs.size(), iters = 40;
        for (int round = 0; round < rounds; ++round) {
                for (int k = 0; k < nv; ++k) {
                        const int i = (k + round) % nv;
                        launch(vs[i], grids[i], round);
                        cudaEventRecord(e0);
                        for (int it = 0; it < iters; ++it) {
                                launch(vs[i], grids[i], it);
                        }
                        cudaEventRecord(e1);
                        cudaEventSynchronize(e1);
                        float ms;
                        cudaEventElapsedTime(&ms, e0, e1);
                        vs[i].us.push_back(ms / iters * 1e3f);
                }
        }
        if (cudaGetLastError() != cudaSuccess) {
                printf("timing failed\n");
                return 1;
        }
        printf("\nus per 8K frame over %d rounds of %d-launch windows: median [quartiles]  (median / median of shipped)\n", rounds, iters);
        float ship = 0;
        for (variant &v : vs) {
                std::sort(v.us.begin(), v.us.end());
                const size_t n = v.us.size();
                if (!v.kern) {
                        ship = v.us[n / 2];
                }
                printf("%-30s %7.2f  [%7.2f %7.2f]  %.3f\n", v.name.c_str(), v.us[n / 2], v.us[n / 4], v.us[3 * n / 4], v.us[n / 2] / ship);
        }
        return 0;
}
