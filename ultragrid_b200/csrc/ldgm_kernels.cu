/* LDGM forward error correction (include/ugb200_ldgm.h): the parity encode and the peeling decode of the reference's LDGM coder
 * (ldgm/src/ldgm-session.cpp, ldgm-session-cpu.cpp), byte-exact, sm_90a.
 *
 * Encode, one kernel: a CTA owns a few words (C) of every packet and a block of rows.  Its threads split the rows into chunks; each
 * thread XORs its rows' data packets and keeps a running XOR inside its chunk (written to the parity packets), the chunk totals are
 * scanned in shared memory, the block's total is published for the blocks below it, and each thread XORs the carry (chunks above in the
 * block, blocks above in the matrix) into its rows.  The staircase is that two-level prefix XOR: no second pass, nothing on the host.
 *
 * Decode, two kernels, no host round trip: ldgm_schedule_kernel (one CTA) replays the reference's sequential peeling on the graph alone,
 * with a count of unknown neighbours per check kept up to date as packets are recovered, so a warp finds the next check with exactly one
 * unknown neighbour by ballot.  Each recovery gets a level one above the highest level it reads (received packets are level 0); the
 * recoveries are bucketed by level.  ldgm_apply_kernel (cooperative grid) then does the XORs of one level at a time with a grid-wide
 * barrier between levels.  A packet is recovered once, by the first check that would recover it in the reference's order, and only
 * read at higher levels, so no two threads write the same bytes and nothing depends on scheduling. */
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <new>
#include <utility>
#include <vector>

#include "../../include/ugb200_ldgm.h"

namespace cg = cooperative_groups;

namespace {

constexpr int kMaxKM = 8191;          // k and m: MAX_K of src/rtp/ldgm.cpp; m is bounded the same way
constexpr int kMaxW = 128;            // MAX_W of ldgm-session.cpp
constexpr int kMaxPacket = 65535;     // LDGM_session::packet_size is an unsigned short
constexpr int kMaxHdr = 256;
constexpr int kEncThreads = 512;
constexpr int kApplyThreads = 256;
constexpr int kSchedThreads = 1024;
constexpr size_t kSchedStageMax = 200 * 1024;  // of the 227 KB of shared memory a CTA may have

template <typename U> __device__ __forceinline__ U xor_w(U a, U b) { return a ^ b; }
template <> __device__ __forceinline__ uint4 xor_w(uint4 a, uint4 b) { return make_uint4(a.x ^ b.x, a.y ^ b.y, a.z ^ b.z, a.w ^ b.w); }
template <typename U> __device__ __forceinline__ U zero_w() { return U(0); }
template <> __device__ __forceinline__ uint4 zero_w() { return make_uint4(0, 0, 0, 0); }

/// cross-CTA state of one encode launch: CTAs take tickets in launch order; ticket t is row block t / col_tiles of column tile
/// t % col_tiles, so every CTA a row block waits for took an earlier ticket and is already running
struct ldgm_enc_grid {
        unsigned long long *ticket;  // never reset: this launch's tickets start at `base`
        int *flag;                   // [row_blocks * col_tiles] = epoch once the block's XOR total is in agg
        void *agg;                   // [row_blocks][nw] words
        unsigned long long base;
        int epoch, col_tiles, row_blocks, rows_per_block;
};

/// parity of C words of every packet for one block of rows: the rows split into kEncThreads / C chunks, a running XOR per chunk, the
/// chunk totals scanned in shared memory, the totals of the row blocks above taken from global memory, the carry XORed into the rows.
/// `nw` words per packet of sizeof(U) bytes.
template <typename U, int C>
__global__ void __launch_bounds__(kEncThreads) ldgm_encode_kernel(const U *__restrict__ data, U *__restrict__ parity, const int *__restrict__ pcm,
                                                               int k, int m, int w_f, int nw, ldgm_enc_grid g)
{
        constexpr int R = kEncThreads / C;
        __shared__ U carry[R][C];
        __shared__ int ticket;
        if (threadIdx.x == 0) {
                ticket = (int) (atomicAdd(g.ticket, 1ull) - g.base);
        }
        __syncthreads();
        const int rb = ticket / g.col_tiles, ct = ticket % g.col_tiles;
        const int c = threadIdx.x % C, r = threadIdx.x / C;
        const int col = ct * C + c;
        const int b0 = rb * g.rows_per_block, b1 = min(b0 + g.rows_per_block, m);
        const int rows = (b1 - b0 + R - 1) / R;
        const int j0 = min(b0 + r * rows, b1), j1 = min(j0 + rows, b1);
        U acc = zero_w<U>();
        if (col < nw) {
                for (int j = j0; j < j1; ++j) {
                        const int *row = pcm + (size_t) j * w_f;
                        for (int e = 0; e < w_f; ++e) {
                                const int idx = __ldg(row + e);
                                if (idx > -1 && idx < k) {
                                        acc = xor_w(acc, __ldg(data + (size_t) idx * nw + col));
                                }
                        }
                        parity[(size_t) j * nw + col] = acc;
                }
        }
        carry[r][c] = acc;
        __syncthreads();
        U *agg = (U *) g.agg;
        if (r == 0) {  // exclusive scan of the chunk totals of column c; the block's total goes to the row blocks below
                U run = zero_w<U>();
                for (int i = 0; i < R; ++i) {
                        const U t = carry[i][c];
                        carry[i][c] = run;
                        run = xor_w(run, t);
                }
                if (rb + 1 < g.row_blocks && col < nw) {
                        agg[(size_t) rb * nw + col] = run;
                }
                __threadfence();
        }
        __syncthreads();
        if (threadIdx.x == 0 && rb + 1 < g.row_blocks) {
                atomicExch(&g.flag[rb * g.col_tiles + ct], g.epoch);
        }
        if (r == 0 && rb > 0) {  // the XOR of every row above this block
                U pre = zero_w<U>();
                for (int p = 0; p < rb; ++p) {
                        const volatile int *f = g.flag + p * g.col_tiles + ct;
                        while (*f != g.epoch) {
                                __nanosleep(64);
                        }
                        __threadfence();
                        if (col < nw) {
                                pre = xor_w(pre, __ldcg(agg + (size_t) p * nw + col));
                        }
                }
                for (int i = 0; i < R; ++i) {
                        carry[i][c] = xor_w(carry[i][c], pre);
                }
        }
        __syncthreads();
        const U in = carry[r][c];
        if (col < nw && (rb > 0 || r > 0)) {
                for (int j = j0; j < j1; ++j) {
                        U *p = parity + (size_t) j * nw + col;
                        *p = xor_w(*p, in);
                }
        }
}

/// int32 overall size, the video header, zeros from the end of the frame to the end of the k data packets (the frame itself is copied
/// by cudaMemcpyAsync)
struct ldgm_hdr_args {
        int overall;
        int hdr_size;
        unsigned char hdr[kMaxHdr];
};
__global__ void ldgm_layout_kernel(unsigned char *out, ldgm_hdr_args a, int pad_begin, int pad_end)
{
        for (int i = threadIdx.x; blockIdx.x == 0 && i < 4 + a.hdr_size; i += blockDim.x) {
                out[i] = i < 4 ? (unsigned char) ((unsigned) a.overall >> (8 * i)) : a.hdr[i - 4];
        }
        for (int i = pad_begin + blockIdx.x * blockDim.x + threadIdx.x; i < pad_end; i += gridDim.x * blockDim.x) {
                out[i] = 0;
        }
}

/// device state of one decode: the schedule kernel writes it, the apply kernel reads it
struct ldgm_sched {
        int *fire_con;      // [k + m] recoveries bucketed by level: check index, or -1 = zero the packet
        int *fire_node;     // [k + m] the packet written
        int *level_start;   // [k + m + 2] bucket b is fire_*[level_start[b] .. level_start[b + 1])
        int *raw_con;       // [k + m] recoveries in the reference's order, before bucketing
        int *raw_node;
        int *meta;          // [0] number of levels, [1] data packets left unknown
};

/// the reference's peeling (decode_frame + iterate) on the graph alone.  `done` comes in as the received packets; dynamic shared memory:
/// done[k+m] u8, zeroed[k+m] u8, level[k+m] u16, cnt[m] int, hist[k+m+2] int.
__global__ void __launch_bounds__(kSchedThreads) ldgm_schedule_kernel(const int *pcm, const int *col_ptr,
                                                                     const int *col_idx, const unsigned char *__restrict__ done_in,
                                                                     int k, int m, int w_f, int staged, ldgm_sched s)
{
        extern __shared__ __align__(16) unsigned char smem[];
        const int n = k + m;
        int *cnt = (int *) smem;
        int *hist = cnt + m;
        unsigned short *level = (unsigned short *) (hist + n + 2);
        unsigned char *done = (unsigned char *) (level + n);
        unsigned char *zeroed = done + n;
        __shared__ int undone_data, nfire, nlevels;
        if (staged) {  // the sweeps chase pcm -> col_ptr -> col_idx: keep the chain in shared memory when it fits
                int *sp = (int *) (((uintptr_t) (zeroed + n) + 15) & ~(uintptr_t) 15);
                const int nnz = col_ptr[n];
                for (int i = threadIdx.x; i < m * w_f; i += blockDim.x) {
                        sp[i] = pcm[i];
                }
                for (int i = threadIdx.x; i <= n; i += blockDim.x) {
                        sp[m * w_f + i] = col_ptr[i];
                }
                for (int i = threadIdx.x; i < nnz; i += blockDim.x) {
                        sp[m * w_f + n + 1 + i] = col_idx[i];
                }
                pcm = sp, col_ptr = sp + m * w_f, col_idx = sp + m * w_f + n + 1;
        }

        if (threadIdx.x == 0) {
                undone_data = 0, nfire = 0, nlevels = 0;
        }
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
                done[i] = done_in[i];
                zeroed[i] = 0;
                level[i] = 0;
        }
        for (int i = threadIdx.x; i < n + 2; i += blockDim.x) {
                hist[i] = 0;
        }
        __syncthreads();
        int local = 0;
        for (int i = threadIdx.x; i < k; i += blockDim.x) {
                local += !done[i];
        }
        for (int j = threadIdx.x; j < m; j += blockDim.x) {  // unknown neighbours of check j, repeated entries counted as often as they occur
                int u = 0;
                for (int e = 0; e < w_f; ++e) {
                        const int idx = pcm[(size_t) j * w_f + e];
                        u += idx > -1 && !done[idx];
                }
                cnt[j] = u;
        }
        atomicAdd(&undone_data, local);
        __syncthreads();

        if (threadIdx.x < 32) {  // one warp replays the sweeps in the reference's order
                const int lane = threadIdx.x;
                int left = undone_data, fired = 0;
                for (int sweep = 0; sweep < 4 && left > 0; ++sweep) {
                        int j = 0;
                        while (j < m) {
                                const unsigned b = __ballot_sync(~0u, j + lane < m && cnt[j + lane] == 1);
                                if (!b) {
                                        j += 32;
                                        continue;
                                }
                                const int f = j + __ffs(b) - 1;
                                const int *row = pcm + (size_t) f * w_f;
                                int ent[kMaxW / 32];  // this lane's entries of the row, read once
                                int r = -1, others = 0, lvl = 0;
#pragma unroll
                                for (int q = 0; q < kMaxW / 32; ++q) {  // the single unknown neighbour
                                        const int e = lane + 32 * q;
                                        ent[q] = e < w_f ? row[e] : -1;
                                        if (ent[q] > -1 && !done[ent[q]]) {
                                                r = ent[q];
                                        }
                                }
                                r = __reduce_max_sync(~0u, r);
                                if (r < 0) {  // cannot happen while cnt is consistent; never index done[-1]
                                        j = f + 1;
                                        continue;
                                }
#pragma unroll
                                for (int q = 0; q < kMaxW / 32; ++q) {
                                        if (ent[q] > -1 && ent[q] != r) {
                                                ++others;
                                                lvl = max(lvl, (int) level[ent[q]]);
                                        }
                                }
                                others = (int) __reduce_add_sync(~0u, (unsigned) others);
                                lvl = __reduce_max_sync(~0u, lvl);
                                if (others > 0) {  // iterate(): the packet is rebuilt from the check's other neighbours and is then known
                                        __syncwarp();
                                        if (lane == 0) {
                                                done[r] = 1;
                                                level[r] = (unsigned short) (lvl + 1);
                                                s.raw_con[fired] = f;
                                                s.raw_node[fired] = r;
                                        }
                                        for (int e = col_ptr[r] + lane; e < col_ptr[r + 1]; e += 32) {
                                                atomicSub(&cnt[col_idx[e]], 1);
                                        }
                                        ++fired;
                                        left -= r < k;
                                } else if (lane == 0) {  // a check with no other neighbour zeroes the packet and leaves it unknown
                                        zeroed[r] = 1;
                                }
                                __syncwarp();
                                j = f + 1;
                        }
                }
                if (lane == 0) {
                        nfire = fired;
                        undone_data = left;
                }
        }
        __syncthreads();

        // buckets: level L >= 1 holds the recoveries of level L; bucket 1 also zeroes the packets that end unknown and were zeroed
        // (lost data packets, and packets a check zeroed), which nothing reads
        for (int i = threadIdx.x; i < nfire; i += blockDim.x) {
                const int L = level[s.raw_node[i]];
                atomicAdd(&hist[L], 1);
                atomicMax(&nlevels, L);
        }
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
                if (!done[i] && (i < k || zeroed[i])) {
                        atomicAdd(&hist[1], 1);
                        atomicMax(&nlevels, 1);
                }
        }
        __syncthreads();
        if (threadIdx.x == 0) {  // levels are few in practice (a chain of staircase recoveries at worst)
                int run = 0;
                for (int L = 0; L <= nlevels + 1; ++L) {
                        const int h = hist[L];
                        hist[L] = run;
                        s.level_start[L] = run;
                        run += h;
                }
                s.meta[0] = nlevels;
                s.meta[1] = undone_data;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < nfire; i += blockDim.x) {
                const int node = s.raw_node[i];
                const int at = atomicAdd(&hist[level[node]], 1);
                s.fire_con[at] = s.raw_con[i];
                s.fire_node[at] = node;
        }
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
                if (!done[i] && (i < k || zeroed[i])) {
                        const int at = atomicAdd(&hist[1], 1);
                        s.fire_con[at] = -1;
                        s.fire_node[at] = i;
                }
        }
}

/// the XORs of the schedule, one level at a time: packet r = XOR of its check's other neighbours (each entry as often as it occurs)
template <typename U>
__global__ void __launch_bounds__(kApplyThreads) ldgm_apply_kernel(U *buf, const int *__restrict__ pcm, int w_f, int nw, ldgm_sched s)
{
        cg::grid_group grid = cg::this_grid();
        const int nlevels = s.meta[0];
        const long stride = (long) gridDim.x * blockDim.x;
        for (int L = 1; L <= nlevels; ++L) {
                const int b0 = s.level_start[L], b1 = s.level_start[L + 1];
                const long items = (long) (b1 - b0) * nw;
                for (long t = (long) blockIdx.x * blockDim.x + threadIdx.x; t < items; t += stride) {
                        const int f = b0 + (int) (t / nw), w = (int) (t % nw);
                        const int con = s.fire_con[f], r = s.fire_node[f];
                        U acc = zero_w<U>();
                        if (con >= 0) {
                                const int *row = pcm + (size_t) con * w_f;
                                for (int e = 0; e < w_f; ++e) {
                                        const int idx = __ldg(row + e);
                                        if (idx > -1 && idx != r) {
                                                acc = xor_w(acc, buf[(size_t) idx * nw + w]);
                                        }
                                }
                        }
                        buf[(size_t) r * nw + w] = acc;
                }
                if (L < nlevels) {
                        grid.sync();
                }
        }
}

}  // namespace

struct ugb200_ldgm {
        cudaStream_t stream = nullptr;
        int k = 0, m = 0, w_f = 0;
        int *d_pcm = nullptr, *d_col_ptr = nullptr, *d_col_idx = nullptr;
        unsigned char *d_buf = nullptr;  // packets staged for the host calls
        size_t buf_cap = 0;
        unsigned char *d_done = nullptr, *h_done = nullptr;
        ldgm_sched sched{};
        int *h_meta = nullptr;
        int apply_grid[4] = {0, 0, 0, 0};  // co-resident CTAs of each ldgm_apply_kernel instantiation
        size_t sched_smem = 0;
        int smem_optin = 0;                 // the largest dynamic shared memory the schedule kernel can have on this device
        bool sched_staged = false;          // the matrix and its column lists fit in the schedule kernel's shared memory
        int sms = 0;
        unsigned long long *d_ticket = nullptr, tickets = 0;
        int *d_flag = nullptr, flag_cap = 0, epoch = 0;
        void *d_agg = nullptr;
        size_t agg_cap = 0;
};

namespace {

void free_matrix(ugb200_ldgm *s)
{
        cudaFree(s->d_pcm), cudaFree(s->d_col_ptr), cudaFree(s->d_col_idx), cudaFree(s->d_done);
        cudaFree(s->sched.fire_con), cudaFree(s->sched.fire_node), cudaFree(s->sched.level_start), cudaFree(s->sched.raw_con);
        cudaFree(s->sched.raw_node), cudaFree(s->sched.meta);
        cudaFreeHost(s->h_done), cudaFreeHost(s->h_meta);
        s->d_pcm = s->d_col_ptr = s->d_col_idx = nullptr;
        s->d_done = s->h_done = nullptr;
        s->h_meta = nullptr;
        s->sched = ldgm_sched{};
        s->k = s->m = s->w_f = 0;
}

int ensure_buf(ugb200_ldgm *s, size_t bytes)
{
        if (bytes <= s->buf_cap) {
                return 0;
        }
        cudaStreamSynchronize(s->stream);
        cudaFree(s->d_buf);
        s->d_buf = nullptr;
        s->buf_cap = 0;
        if (cudaMalloc(&s->d_buf, bytes) != cudaSuccess) {
                return -2;
        }
        s->buf_cap = bytes;
        return 0;
}

/// word width: the widest of 16/8/4/1 bytes dividing both the packet size and the buffer's address
int word_bytes(int ps, uintptr_t addr)
{
        for (int b : {16, 8, 4}) {
                if (ps % b == 0 && addr % b == 0) {
                        return b;
                }
        }
        return 1;
}

template <typename U>
int launch_encode_t(ugb200_ldgm *s, const void *data, void *parity, int ps)
{
        constexpr int C = 32 / sizeof(U) > 0 ? 32 / sizeof(U) : 1;  // a 32-byte sector of each row per warp step
        constexpr int R = kEncThreads / C;
        const int nw = ps / (int) sizeof(U);
        const int col_tiles = (nw + C - 1) / C;
        if (!s->sms) {
                int dev = 0;
                cudaGetDevice(&dev);
                cudaDeviceGetAttribute(&s->sms, cudaDevAttrMultiProcessorCount, dev);
        }
        // rows split over CTAs until the grid covers the GPU twice, each CTA keeping at least one row per chunk
        int row_blocks = std::max(1, std::min((2 * s->sms + col_tiles - 1) / col_tiles, (s->m + R - 1) / R));
        const int rows_per_block = (s->m + row_blocks - 1) / row_blocks;
        row_blocks = (s->m + rows_per_block - 1) / rows_per_block;
        const int grid = row_blocks * col_tiles;
        const size_t agg_bytes = (size_t) row_blocks * ps;
        if (!s->d_ticket && (cudaMalloc(&s->d_ticket, sizeof(unsigned long long)) != cudaSuccess ||
                             cudaMemsetAsync(s->d_ticket, 0, sizeof(unsigned long long), s->stream) != cudaSuccess)) {
                return -2;
        }
        if (grid > s->flag_cap || agg_bytes > s->agg_cap) {
                cudaStreamSynchronize(s->stream);
                cudaFree(s->d_flag), cudaFree(s->d_agg);
                s->d_flag = nullptr, s->d_agg = nullptr, s->flag_cap = 0, s->agg_cap = 0;
                const int fc = std::max(grid, 1024);
                const size_t ac = std::max(agg_bytes, (size_t) 1 << 16);
                if (cudaMalloc(&s->d_flag, sizeof(int) * fc) != cudaSuccess || cudaMalloc(&s->d_agg, ac) != cudaSuccess ||
                    cudaMemsetAsync(s->d_flag, 0, sizeof(int) * fc, s->stream) != cudaSuccess) {
                        return -2;
                }
                s->flag_cap = fc, s->agg_cap = ac;
        }
        ldgm_enc_grid g{s->d_ticket, s->d_flag, s->d_agg, s->tickets, ++s->epoch, col_tiles, row_blocks, rows_per_block};
        ldgm_encode_kernel<U, C><<<grid, kEncThreads, 0, s->stream>>>((const U *) data, (U *) parity, s->d_pcm, s->k, s->m, s->w_f, nw, g);
        if (cudaGetLastError() != cudaSuccess) {
                return -2;
        }
        s->tickets += grid;  // only a launched grid draws tickets: a failed launch leaves base and counter in step
        return 0;
}

int launch_encode(ugb200_ldgm *s, const void *data, void *parity, int ps)
{
        switch (word_bytes(ps, (uintptr_t) data | (uintptr_t) parity)) {
        case 16: return launch_encode_t<uint4>(s, data, parity, ps);
        case 8: return launch_encode_t<unsigned long long>(s, data, parity, ps);
        case 4: return launch_encode_t<uint32_t>(s, data, parity, ps);
        default: return -1;  // ps is a multiple of 4 and the buffers are at least 4-byte aligned (checked by the callers)
        }
}

long layout(const ugb200_ldgm *s, long payload, int *ps_out)
{
        const long align = (long) s->k * 4;
        const long data = (payload + 4 + align - 1) / align * align;
        const long ps = data / s->k;
        if (ps > kMaxPacket) {
                return -1;
        }
        *ps_out = (int) ps;
        return data + (long) s->m * ps;
}

template <typename U>
int launch_apply_t(ugb200_ldgm *s, int slot, int ps)
{
        if (!s->apply_grid[slot]) {
                int dev = 0, sms = 0, per_sm = 0;
                cudaGetDevice(&dev);
                cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
                cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ldgm_apply_kernel<U>, kApplyThreads, 0);
                s->apply_grid[slot] = sms * std::max(1, per_sm);
        }
        U *buf = (U *) s->d_buf;
        int nw = ps / (int) sizeof(U);
        void *args[] = {&buf, &s->d_pcm, &s->w_f, &nw, &s->sched};
        return cudaLaunchCooperativeKernel((const void *) ldgm_apply_kernel<U>, s->apply_grid[slot], kApplyThreads, args, 0, s->stream) ==
                       cudaSuccess ? 0 : -2;
}

/// which packets decode_frame counts as received: (offset, length) merged where one ends exactly where the next begins, then a packet
/// is received when the last merged range starting at or before it reaches its end
void received_packets(const int *ranges, int n_ranges, int p, int nodes, unsigned char *done)
{
        std::vector<std::pair<int, int>> v;
        v.reserve(n_ranges);
        for (int i = 0; i < n_ranges; ++i) {
                v.emplace_back(ranges[2 * i], ranges[2 * i + 1]);
        }
        std::stable_sort(v.begin(), v.end(), [](const auto &a, const auto &b) { return a.first < b.first; });
        std::vector<std::pair<int, int>> map;  // std::map<int, int> semantics: a repeated offset keeps its last length
        for (const auto &e : v) {
                if (!map.empty() && map.back().first == e.first) {
                        map.back().second = e.second;
                } else {
                        map.push_back(e);
                }
        }
        std::vector<std::pair<long, long>> merged;
        for (size_t i = 0; i < map.size();) {
                const long start = map[i].first;
                long length = map[i].second;
                while (++i < map.size() && start + length == map[i].first) {
                        length += map[i].second;
                }
                merged.emplace_back(start, length);
        }
        size_t at = 0;
        for (int i = 0; i < nodes; ++i) {
                const long off = (long) i * p;
                while (at < merged.size() && merged[at].first <= off) {
                        ++at;
                }
                done[i] = at > 0 && merged[at - 1].first + merged[at - 1].second >= off + p;
        }
}

}  // namespace

extern "C" {

ugb200_ldgm *ugb200_ldgm_create(cuda_wrapper_stream_t stream)
{
        ugb200_ldgm *s = new (std::nothrow) ugb200_ldgm;
        if (s) {
                s->stream = (cudaStream_t) stream;
        }
        return s;
}

void ugb200_ldgm_destroy(ugb200_ldgm *s)
{
        if (!s) {
                return;
        }
        cudaStreamSynchronize(s->stream);
        free_matrix(s);
        cudaFree(s->d_buf), cudaFree(s->d_ticket), cudaFree(s->d_flag), cudaFree(s->d_agg);
        delete s;
}

int ugb200_ldgm_set_matrix(ugb200_ldgm *s, const int *pcm, int k, int m, int w_f)
{
        if (!s || !pcm || k < 1 || k > kMaxKM || m < 1 || m > kMaxKM || w_f < 2 || w_f > kMaxW) {
                return -1;
        }
        const int n = k + m;
        std::vector<int> col_ptr(n + 1, 0), col_idx;
        for (long i = 0; i < (long) m * w_f; ++i) {
                if (pcm[i] < -1 || pcm[i] >= n) {
                        return -1;
                }
                col_ptr[pcm[i] + 1] += pcm[i] > -1;
        }
        for (int i = 0; i < n; ++i) {
                col_ptr[i + 1] += col_ptr[i];
        }
        col_idx.resize(std::max(1, col_ptr[n]));
        std::vector<int> fill(col_ptr.begin(), col_ptr.end() - 1);
        for (int j = 0; j < m; ++j) {
                for (int e = 0; e < w_f; ++e) {
                        const int idx = pcm[(size_t) j * w_f + e];
                        if (idx > -1) {
                                col_idx[fill[idx]++] = j;
                        }
                }
        }
        cudaStreamSynchronize(s->stream);
        free_matrix(s);
        bool ok = cudaMalloc(&s->d_pcm, sizeof(int) * m * w_f) == cudaSuccess &&
                  cudaMalloc(&s->d_col_ptr, sizeof(int) * (n + 1)) == cudaSuccess &&
                  cudaMalloc(&s->d_col_idx, sizeof(int) * col_idx.size()) == cudaSuccess && cudaMalloc(&s->d_done, n) == cudaSuccess &&
                  cudaMalloc(&s->sched.fire_con, sizeof(int) * n) == cudaSuccess && cudaMalloc(&s->sched.fire_node, sizeof(int) * n) == cudaSuccess &&
                  cudaMalloc(&s->sched.level_start, sizeof(int) * (n + 2)) == cudaSuccess &&
                  cudaMalloc(&s->sched.raw_con, sizeof(int) * n) == cudaSuccess && cudaMalloc(&s->sched.raw_node, sizeof(int) * n) == cudaSuccess &&
                  cudaMalloc(&s->sched.meta, sizeof(int) * 2) == cudaSuccess && cudaMallocHost(&s->h_done, n) == cudaSuccess &&
                  cudaMallocHost(&s->h_meta, sizeof(int) * 2) == cudaSuccess;
        ok = ok && cudaMemcpy(s->d_pcm, pcm, sizeof(int) * m * w_f, cudaMemcpyHostToDevice) == cudaSuccess &&
             cudaMemcpy(s->d_col_ptr, col_ptr.data(), sizeof(int) * (n + 1), cudaMemcpyHostToDevice) == cudaSuccess &&
             cudaMemcpy(s->d_col_idx, col_idx.data(), sizeof(int) * col_idx.size(), cudaMemcpyHostToDevice) == cudaSuccess;
        s->sched_smem = (size_t) m * 4 + (size_t) (n + 2) * 4 + (size_t) n * 2 + (size_t) n * 2;
        const size_t staged = (s->sched_smem + 15) / 16 * 16 + sizeof(int) * ((size_t) m * w_f + n + 1 + col_ptr[n]);
        s->sched_staged = staged <= kSchedStageMax;
        if (s->sched_staged) {
                s->sched_smem = staged;
        }
        int dev = 0, optin = 0;
        cudaFuncAttributes fa{};
        ok = ok && cudaGetDevice(&dev) == cudaSuccess &&
             cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) == cudaSuccess &&
             cudaFuncGetAttributes(&fa, ldgm_schedule_kernel) == cudaSuccess;
        s->smem_optin = optin - (int) fa.sharedSizeBytes;  // the kernel's static shared memory counts against the same opt-in limit
        ok = ok && s->sched_smem <= (size_t) s->smem_optin;
        if (!ok) {
                free_matrix(s);
                return -2;
        }
        s->k = k, s->m = m, s->w_f = w_f;
        return 0;
}

long ugb200_ldgm_buffer_size(const ugb200_ldgm *s, int payload_size, int *packet_size)
{
        int ps = 0;
        if (!s || payload_size < 0) {
                return -1;
        }
        if (!s->k) {
                return -3;
        }
        const long total = layout(s, payload_size, &ps);
        if (total >= 0 && packet_size) {
                *packet_size = ps;
        }
        return total;
}

int ugb200_ldgm_encode(ugb200_ldgm *s, const void *data, void *parity, int packet_size)
{
        if (!s || !data || !parity || packet_size <= 0 || packet_size % 4 || packet_size > kMaxPacket) {
                return -1;
        }
        if (!s->k) {
                return -3;
        }
        const size_t dbytes = (size_t) s->k * packet_size, pbytes = (size_t) s->m * packet_size;
        if (ensure_buf(s, dbytes + pbytes)) {
                return -2;
        }
        if (cudaMemcpyAsync(s->d_buf, data, dbytes, cudaMemcpyHostToDevice, s->stream) != cudaSuccess ||
            launch_encode(s, s->d_buf, s->d_buf + dbytes, packet_size) ||
            cudaMemcpyAsync(parity, s->d_buf + dbytes, pbytes, cudaMemcpyDeviceToHost, s->stream) != cudaSuccess ||
            cudaStreamSynchronize(s->stream) != cudaSuccess) {
                return -2;
        }
        return 0;
}

int ugb200_ldgm_encode_frame(ugb200_ldgm *s, const void *hdr, int hdr_size, const void *frame, int frame_size, void *out,
                             size_t out_capacity, int *out_size)
{
        int ps = 0;
        if (!s || (hdr_size && !hdr) || hdr_size < 0 || (frame_size && !frame) || frame_size < 0 || !out || !out_size ||
            (long) hdr_size + frame_size > INT32_MAX - 4) {
                return -1;
        }
        if (!s->k) {
                return -3;
        }
        const int overall = hdr_size + frame_size;
        const long total = layout(s, overall, &ps);
        if (total < 0) {
                return -1;
        }
        if ((size_t) total > out_capacity) {
                return -5;
        }
        unsigned char *o = (unsigned char *) out;
        memcpy(o, &overall, 4);
        if (hdr_size) {
                memcpy(o + 4, hdr, hdr_size);
        }
        if (frame_size) {
                memcpy(o + 4 + hdr_size, frame, frame_size);
        }
        memset(o + 4 + overall, 0, (size_t) s->k * ps - 4 - overall);
        *out_size = (int) total;
        return ugb200_ldgm_encode(s, o, o + (size_t) s->k * ps, ps);
}

int ugb200_ldgm_encode_device(ugb200_ldgm *s, const void *hdr, int hdr_size, const void *frame, int frame_size, void *out,
                              size_t out_capacity, int *out_size)
{
        int ps = 0;
        if (!s || (hdr_size && !hdr) || hdr_size < 0 || hdr_size > kMaxHdr || (frame_size && !frame) || frame_size < 0 || !out ||
            !out_size || (uintptr_t) out % 4 || (long) hdr_size + frame_size > INT32_MAX - 4) {
                return -1;
        }
        if (!s->k) {
                return -3;
        }
        const int overall = hdr_size + frame_size;
        const long total = layout(s, overall, &ps);
        if (total < 0) {
                return -1;
        }
        if ((size_t) total > out_capacity) {
                return -5;
        }
        unsigned char *o = (unsigned char *) out;
        const long dbytes = (long) s->k * ps;
        ldgm_hdr_args a;
        a.overall = overall;
        a.hdr_size = hdr_size;
        if (hdr_size) {
                memcpy(a.hdr, hdr, hdr_size);
        }
        if (frame_size && cudaMemcpyAsync(o + 4 + hdr_size, frame, frame_size, cudaMemcpyDeviceToDevice, s->stream) != cudaSuccess) {
                return -2;
        }
        const int pad = (int) (dbytes - 4 - overall);
        ldgm_layout_kernel<<<std::max(1, std::min(64, (pad + 255) / 256)), 256, 0, s->stream>>>(o, a, 4 + overall, (int) dbytes);
        if (cudaGetLastError() != cudaSuccess) {
                return -2;
        }
        *out_size = (int) total;
        return launch_encode(s, o, o + dbytes, ps);
}

int ugb200_ldgm_decode(ugb200_ldgm *s, void *buf, int buf_size, const int *ranges, int n_ranges, int *frame_size)
{
        if (!s || !buf || buf_size < 0 || n_ranges < 0 || (n_ranges && !ranges) || !frame_size) {
                return -1;
        }
        if (!s->k) {
                return -3;
        }
        const int k = s->k, m = s->m, n = k + m;
        const int p = buf_size / n;
        if (p <= 0 || p > kMaxPacket) {
                return -1;
        }
        unsigned char *b = (unsigned char *) buf;
        cudaStreamSynchronize(s->stream);  // h_done is reused
        received_packets(ranges, n_ranges, p, n, s->h_done);
        bool all = true;
        for (int i = 0; i < k && all; ++i) {
                all = s->h_done[i];
        }
        if (all) {  // nothing to peel: decode_frame runs no sweep and leaves the buffer as it is
                memcpy(frame_size, b, 4);
                return 0;
        }
        const size_t bytes = (size_t) n * p;
        if (ensure_buf(s, bytes)) {
                return -2;
        }
        if (cudaMemcpyAsync(s->d_buf, b, bytes, cudaMemcpyHostToDevice, s->stream) != cudaSuccess ||
            cudaMemcpyAsync(s->d_done, s->h_done, n, cudaMemcpyHostToDevice, s->stream) != cudaSuccess) {
                return -2;
        }
        // the limit belongs to the kernel, not to the session: raised to the device's opt-in maximum before every launch, it can never have
        // been lowered below this session's need by another session's matrix
        if (cudaFuncSetAttribute(ldgm_schedule_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, s->smem_optin) != cudaSuccess) {
                return -2;
        }
        ldgm_schedule_kernel<<<1, kSchedThreads, s->sched_smem, s->stream>>>(s->d_pcm, s->d_col_ptr, s->d_col_idx, s->d_done, k, m, s->w_f,
                                                                             s->sched_staged, s->sched);
        if (cudaGetLastError() != cudaSuccess) {
                return -2;
        }
        int rc;
        switch (word_bytes(p, 0)) {
        case 16: rc = launch_apply_t<uint4>(s, 0, p); break;
        case 8: rc = launch_apply_t<unsigned long long>(s, 1, p); break;
        case 4: rc = launch_apply_t<uint32_t>(s, 2, p); break;
        default: rc = launch_apply_t<unsigned char>(s, 3, p); break;
        }
        if (rc || cudaMemcpyAsync(b, s->d_buf, bytes, cudaMemcpyDeviceToHost, s->stream) != cudaSuccess ||
            cudaMemcpyAsync(s->h_meta, s->sched.meta, sizeof(int) * 2, cudaMemcpyDeviceToHost, s->stream) != cudaSuccess ||
            cudaStreamSynchronize(s->stream) != cudaSuccess) {
                return -2;
        }
        if (s->h_meta[1] == 0) {
                memcpy(frame_size, b, 4);
        } else {
                *frame_size = 0;
        }
        return 0;
}

}  // extern "C"
