// The Huffman state machine of the JPEG decoder, shared by both decode routes and by a CPU test:
//   - jpeg_decode_huffman_kernel (one thread per restart segment) decodes whole blocks with decode_block;
//   - the self-synchronising route (jpeg_sync_*_kernel, for segments of many MCUs) cuts a segment's bytes into subsequences and steps through them
//     symbol by symbol with walk_count / decode_block, reading through pos_reader, whose position is an address in the stuffed stream;
//   - tests/test_jpeg_decode_sync.py compiles this header for the host and runs both routes sequentially.
// What the decoder does with ANY bytes between a segment's begin and end is defined here: 0xFF 0x00 inside the segment reads as 0xFF, a lone 0xFF as
// itself, zero bits are fed past the end; a code that is not in the table skips 16 bits and yields symbol 0 (no DC difference / EOB); a run or ZRL past
// position 63 still consumes its value bits and stores nothing.
#pragma once
#include <stdint.h>
#include <string.h>

#ifndef __CUDACC__
#define UGB_HD
#else
#define UGB_HD __host__ __device__
#endif

namespace ugb {

constexpr int kLook = 9;
/// Huffman table slots.  A DHT definition is built into a slot when a scan first uses it: table id k (DC Th 0, 1 = 0, 1; AC Th 0, 1 = 2, 3)
/// goes to slot k when that slot is free, otherwise to the lowest free one.  A table redefined between scans (T.81 B.2.4.2) thus gets a slot
/// of its own, and every scan keeps the tables it was coded with.  In a valid stream each component appears in one scan and uses one DC and
/// one AC table, and only definitions that a scan uses take a slot: four components never need more than eight.
constexpr int kTables = 8;

struct dec_tables {
        uint16_t lut[kTables][1 << kLook];  // (length << 8) | symbol for codes of up to kLook bits, 0 = longer code
        int maxcode[kTables][18];           // T.81 F.2.2.3, -1 = no code of that length
        int valoff[kTables][17];            // valptr - mincode
        uint8_t vals[kTables][256];
        uint8_t zz[64];
        float m[4][64];               // dequantisation x AAN scale, natural order
};

struct dec_comp {
        int h, v, tq;
        int bw, bh;     // blocks per row / rows of the padded plane
        int blk_off;    // first block of the component in the coefficient buffer
        long plane_off; // first byte of the plane in the plane buffer
};
struct dec_scan {
        int ns, comp[4], td[4], ta[4];  // td, ta: table slots of dec_tables
        int mcux, nmcu;
        int seg0, nseg;  // segments [seg0, seg0 + nseg)
};
struct dec_geom {
        int w, h, ncomp, hmax, vmax, ri, nscans, nblocks;  // ncomp 3, or 4 (R G B A, all 1x1)
        int ntables;  // Huffman table slots in use: [0, ntables) (the Huffman kernel copies only those to shared memory)
        dec_comp c[4];
        dec_scan s[4];
};

/// the bits / values have passed the Kraft check of the parser
inline void build_table(dec_tables &t, int tab, const uint8_t *bits, const uint8_t *vals, int n)
{
        memset(t.lut[tab], 0, sizeof t.lut[tab]);
        memcpy(t.vals[tab], vals, n);
        int code = 0, k = 0;
        for (int l = 1; l <= 16; ++l) {
                t.valoff[tab][l] = k - code;
                for (int i = 0; i < bits[l - 1]; ++i, ++k, ++code) {
                        if (l <= kLook) {
                                for (int fill = 0; fill < (1 << (kLook - l)); ++fill) {
                                        t.lut[tab][(code << (kLook - l)) | fill] = (uint16_t) (l << 8 | vals[k]);
                                }
                        }
                }
                t.maxcode[tab][l] = bits[l - 1] ? code - 1 : -1;
                code <<= 1;
        }
        t.maxcode[tab][17] = 0x7fffffff;
}

// ---- per symbol: any reader with peek(n) (the next n bits, 1 <= n <= 32) and skip(n), holding at least 33 bits after refill() -----------------

/// T.81 F.2.2.3 with a kLook-bit look-up table, then the min/max-code walk from kLook + 1 to 16 bits
template <class R>
UGB_HD inline int decode_symbol(R &r, const dec_tables *t, int tab)
{
        const uint32_t e = t->lut[tab][r.peek(kLook)];
        if (e) {
                r.skip(e >> 8);
                return e & 0xff;
        }
        const uint32_t v16 = r.peek(16);
        for (int l = kLook + 1; l <= 16; ++l) {
                const int code = (int) (v16 >> (16 - l));
                if (code <= t->maxcode[tab][l]) {
                        r.skip(l);
                        return t->vals[tab][t->valoff[tab][l] + code];
                }
        }
        r.skip(16);
        return 0;  // corrupt stream
}
/// F.2.2.1, n in 0..15 (0: a DC symbol of a damaged table whose low nibble is 0 - no value bits, no difference)
template <class R>
UGB_HD inline int receive_extend(R &r, int n)
{
        if (n == 0) {
                return 0;
        }
        const int v = (int) r.peek(n);
        r.skip(n);
        return v < (1 << (n - 1)) ? v - (1 << n) + 1 : v;
}
/// the DC difference behind DC symbol tt
template <class R>
UGB_HD inline uint32_t dc_diff(R &r, int tt)
{
        return tt ? (uint32_t) receive_extend(r, tt & 15) : 0u;
}
/// AC symbol rs at zig-zag position i (F.2.2.2): false = EOB; otherwise i moves past the coefficient and store(i, v) is called for one at i < 64
template <class R, class Store>
UGB_HD inline bool ac_symbol(R &r, int rs, int &i, Store &&store)
{
        const int run = rs >> 4, sz = rs & 15;
        if (sz == 0) {
                if (run != 15) {
                        return false;  // EOB
                }
                i += 16;
                return true;
        }
        i += run;
        const int v = receive_extend(r, sz);  // refill guarantees >= 33 bits: 16 + 15 fit
        if (i < 64) {
                store(i, v);
        }
        ++i;
        return true;
}
/// one whole block: DC difference added to `pred` (kept modulo 2^32, stored as its low 16 bits), sink.dc(pred), then sink(i, v) per coefficient
template <class R, class Sink>
UGB_HD inline void decode_block(R &r, const dec_tables *t, int td, int ta, uint32_t &pred, Sink &&sink)
{
        r.refill();
        const int tt = decode_symbol(r, t, td);
        r.refill();
        pred += dc_diff(r, tt);
        sink.dc(pred);
        for (int i = 1; i < 64;) {
                r.refill();
                const int rs = decode_symbol(r, t, ta);
                if (!ac_symbol(r, rs, i, sink)) {
                        break;
                }
        }
}

/// the blocks of one MCU in coding order (T.81 A.2.3): scan component k, then rows by, then columns bx of its h x v blocks; one block per MCU in
/// a one-component scan
struct mcu_layout {
        int bpm;
        uint8_t k[10], bx[10], by[10];
};
UGB_HD inline mcu_layout layout_of(const dec_geom &g, const dec_scan &S)
{
        mcu_layout L;
        L.bpm = 0;
        for (int k = 0; k < S.ns; ++k) {
                const dec_comp &c = g.c[S.comp[k]];
                const int nh = S.ns == 1 ? 1 : c.h, nv = S.ns == 1 ? 1 : c.v;
                for (int by = 0; by < nv; ++by) {
                        for (int bx = 0; bx < nh; ++bx) {
                                if (L.bpm < 10) {
                                        L.k[L.bpm] = (uint8_t) k, L.bx[L.bpm] = (uint8_t) bx, L.by[L.bpm] = (uint8_t) by;
                                        ++L.bpm;
                                }
                        }
                }
        }
        return L;
}

// ---- the self-synchronising route -------------------------------------------------------------------------------------------------------------

/// Reads the segment [begin, end) of `s` as the one-thread reader does, and knows where it is: (q, b) is the address in the STUFFED stream of the
/// byte holding the next unread bit, and its bit (0 = MSB).  Addresses from `end` on are a virtual zero tail.  The skipped byte of a stuffed pair
/// is never a position, so every symbol boundary has one address, whichever thread decodes it.  `s` must be readable up to end + 12.
struct pos_reader {
        const uint8_t *s;
        uint32_t end;
        uint64_t q;
        int b;
        uint64_t acc;     // bits from (q, b) on, MSB first
        int nbits, used;  // valid bits in acc, bits consumed since acc was loaded
        bool plain;       // no stuffed byte among the bytes of acc: the position is (q, b) + used

        UGB_HD uint64_t next(uint64_t a) const { return a + 1 < end && s[a] == 0xFF && s[a + 1] == 0 ? a + 2 : a + 1; }
        UGB_HD static bool has_ff(uint64_t w)  // some byte of w is 0xFF
        {
                const uint64_t v = ~w;
                return ((v - 0x0101010101010101ull) & ~v & 0x8080808080808080ull) != 0;
        }
        UGB_HD uint64_t load8(uint64_t a) const  // bytes a .. a + 7, big-endian
        {
#ifdef __CUDA_ARCH__
                const uint32_t *wa = (const uint32_t *) ((size_t) (s + a) & ~(size_t) 3);
                const uint32_t w0 = __ldg(wa), w1 = __ldg(wa + 1), w2 = __ldg(wa + 2), sh = 8 * (uint32_t) ((size_t) (s + a) & 3);
                const uint32_t lo = __funnelshift_r(w0, w1, sh), hi = __funnelshift_r(w1, w2, sh);
                return (uint64_t) __byte_perm(lo, 0, 0x0123) << 32 | __byte_perm(hi, 0, 0x0123);
#else
                uint64_t w;
                memcpy(&w, s + a, 8);
                return __builtin_bswap64(w);
#endif
        }
        UGB_HD void load()
        {
                uint64_t w;
                plain = true;
                if (q + 8 <= end && !has_ff(w = load8(q))) {
                } else {
                        w = 0;
                        uint64_t a = q;
                        for (int k = 0; k < 8; ++k) {
                                w = w << 8 | (a < end ? s[a] : 0u);
                                const uint64_t n = next(a);
                                plain = plain && n == a + 1;
                                a = n;
                        }
                }
                acc = w << b, nbits = 64 - b, used = 0;
        }
        UGB_HD void start(uint64_t q0, int b0)
        {
                q = q0, b = b0;
                load();
        }
        /// moves (q, b) to the next unread bit
        UGB_HD void settle()
        {
                int bits = b + used;
                if (plain) {
                        q += (uint64_t) (bits >> 3);
                } else {
                        for (; bits >= 8; bits -= 8) {
                                q = next(q);
                        }
                }
                b = bits & 7, used = 0;
        }
        UGB_HD uint64_t pos()  // bit address of the next unread bit
        {
                if (!plain && used) {
                        settle();
                        load();
                }
                return q * 8 + (uint64_t) (b + used);
        }
        UGB_HD void refill()
        {
                if (nbits > 32) {
                        return;
                }
                settle();
                load();
        }
        UGB_HD uint32_t peek(int n) const { return (uint32_t) (acc >> (64 - n)); }
        UGB_HD void skip(int n) { acc <<= n, nbits -= n, used += n; }
};

/// decoder state at a symbol boundary: bit address in the stuffed stream, block of the MCU, zig-zag position (0: the DC symbol is next)
struct sync_point {
        uint32_t byte, tag;  // tag = bit << 16 | blk << 8 | zz
};
UGB_HD inline sync_point make_point(uint64_t bitpos, int blk, int zz) { return { (uint32_t) (bitpos >> 3), (uint32_t) ((bitpos & 7) << 16 | blk << 8 | zz) }; }

/// The count pass of a subsequence: from state (blk, zz) at the reader's position, decodes symbol by symbol up to the first symbol boundary at or after
/// bit address `limit`, where it stops.  Counts the blocks whose DC symbol starts before `limit` and adds their DC differences per scan component.
template <class R>
UGB_HD inline void walk_count(R &r, const dec_tables *t, const int *td, const int *ta, const mcu_layout &L, uint64_t limit, int &blk, int &zz,
                              uint32_t &count, uint32_t sum[4])
{
        while (r.pos() < limit) {
                r.refill();
                const int k = L.k[blk];
                if (zz == 0) {
                        ++count;
                        const int tt = decode_symbol(r, t, td[k]);
                        r.refill();
                        sum[k] += dc_diff(r, tt);
                        zz = 1;
                        continue;
                }
                const int rs = decode_symbol(r, t, ta[k]);
                int i = zz;
                if (!ac_symbol(r, rs, i, [](int, int) {}) || i >= 64) {
                        zz = 0, blk = blk + 1 == L.bpm ? 0 : blk + 1;
                } else {
                        zz = i;
                }
        }
}
/// the rest of a block begun before (state zz > 0): decoded, not stored
template <class R>
UGB_HD inline void finish_block(R &r, const dec_tables *t, int ta, int zz)
{
        for (int i = zz; i < 64;) {
                r.refill();
                const int rs = decode_symbol(r, t, ta);
                if (!ac_symbol(r, rs, i, [](int, int) {})) {
                        break;
                }
        }
}

/// bit address where subsequence `local` of a segment starts: every `sub_bytes` bytes from `begin`, one byte on when that byte is the skipped half of a
/// stuffed pair (so that the start is a byte the one-thread reader reads)
UGB_HD inline uint64_t sub_start(const uint8_t *s, uint32_t begin, uint32_t end, int local, int sub_bytes)
{
        uint64_t a = (uint64_t) begin + (uint64_t) local * (uint64_t) sub_bytes;
        if (local > 0 && a < end && s[a - 1] == 0xFF && s[a] == 0) {
                ++a;
        }
        return a * 8;
}
/// subsequences of a segment of `bytes` bytes (an empty segment has one: it decodes zero bits)
UGB_HD inline int sub_count(uint32_t bytes, int sub_bytes) { return bytes == 0 ? 1 : (int) ((bytes + (uint32_t) sub_bytes - 1) / (uint32_t) sub_bytes); }

}  // namespace ugb
