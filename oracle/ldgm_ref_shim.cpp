// extern "C" face of the UNMODIFIED reference LDGM coder (ldgm/src/ldgm-session.cpp, ldgm-session-cpu.cpp, tanner.cpp) and matrix
// generator (ldgm/matrix-gen/matrix-generator.cpp, ldpc-matrix.cpp), built by ldgm.mk into _ref/libldgm_ref.so: the CPU oracle of
// include/ugb200_ldgm.h.  Test infrastructure, not part of the product.
#include <stdlib.h>
#include <string.h>

#include <map>
#include <string>

#include "ldgm-session-cpu.h"
#include "matrix-generator.h"

namespace {
// reaches the protected members the tests compare against (pcm, max_row_weight) and lets encode_naive run without a frame
struct Probe : LDGM_session_cpu {
        const int *matrix() const { return pcm; }
        int columns() const { return max_row_weight + 2; }
        void set_packet_size(int ps) { packet_size = (unsigned short) ps; }
};
}  // namespace

extern "C" {

__attribute__((visibility("default"))) int ref_ldgm_generate(const char *fname, unsigned k, unsigned m, unsigned c, unsigned seed)
{
        return generate_ldgm_matrix((char *) fname, k, m, c, seed, 0);
}

/// LDGM_session_cpu with set_params(k, m, c) and set_pcMatrix(fname); NULL when the file is refused
__attribute__((visibility("default"))) void *ref_ldgm_create(const char *fname, int k, int m, int c)
{
        Probe *p = new Probe;
        p->set_params(k, m, c);
        try {
                p->set_pcMatrix((char *) fname);
        } catch (const std::string &) {
                delete p;
                return nullptr;
        }
        return p;
}

__attribute__((visibility("default"))) void ref_ldgm_destroy(void *s) { delete (Probe *) s; }

/// copies set_pcMatrix's pcm (m rows of w_f ints) to out; returns w_f
__attribute__((visibility("default"))) int ref_ldgm_pcm(void *s, int m, int *out, long cap)
{
        Probe *p = (Probe *) s;
        const long n = (long) m * p->columns();
        if (out && cap >= n) {
                memcpy(out, p->matrix(), n * sizeof(int));
        }
        return p->columns();
}

/// encode_hdr_frame, copied to out (capacity cap); returns the buffer length or -1
__attribute__((visibility("default"))) int ref_ldgm_encode_hdr_frame(void *s, const char *hdr, int hdr_size, const char *frame, int frame_size,
                                                                     char *out, long cap)
{
        Probe *p = (Probe *) s;
        int n = 0;
        char *buf = p->encode_hdr_frame((char *) hdr, hdr_size, (char *) frame, frame_size, &n);
        if (!buf || n > cap) {
                p->free_out_buf(buf);
                return -1;
        }
        memcpy(out, buf, n);
        p->free_out_buf(buf);
        return n;
}

/// encode (running XOR) or encode_naive (explicit staircase) of k data packets of ps bytes into m parity packets
__attribute__((visibility("default"))) void ref_ldgm_encode_raw(void *s, char *data, char *parity, int ps, int naive)
{
        Probe *p = (Probe *) s;
        p->set_packet_size(ps);
        if (naive) {
                p->encode_naive(data, parity);
        } else {
                p->encode(data, parity);
        }
}

/// decode_frame on buf in place; ranges = n (offset, length) pairs inserted into the std::map in order; returns *frame_size
__attribute__((visibility("default"))) int ref_ldgm_decode(void *s, char *buf, int buf_size, const int *ranges, int n)
{
        std::map<int, int> valid;
        for (int i = 0; i < n; ++i) {
                valid[ranges[2 * i]] = ranges[2 * i + 1];
        }
        int frame_size = -1;
        ((Probe *) s)->decode_frame(buf, buf_size, &frame_size, valid);
        return frame_size;
}

}  // extern "C"
