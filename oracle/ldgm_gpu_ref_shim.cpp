// extern "C" face of the UNMODIFIED reference GPU coder LDGM_session_gpu (ldgm/src/gpu.cu, ldgm-session-gpu.cpp), built for sm_90a by
// ldgm.mk into _ref/libldgm_gpu_ref.so: the second encode oracle of include/ugb200_ldgm.h.  Test infrastructure, not part of the product.
#include <string.h>

#include <string>

#include "ldgm-session-gpu.h"

extern "C" {

__attribute__((visibility("default"))) void *refgpu_ldgm_create(const char *fname, int k, int m, int c)
{
        auto *p = new LDGM_session_gpu;
        p->set_params(k, m, c);
        try {
                p->set_pcMatrix((char *) fname);
        } catch (const std::string &) {
                delete p;
                return nullptr;
        }
        return p;
}

__attribute__((visibility("default"))) void refgpu_ldgm_destroy(void *s) { delete (LDGM_session_gpu *) s; }

/// encode_hdr_frame, copied to out (capacity cap); the buffer length or -1
__attribute__((visibility("default"))) int refgpu_ldgm_encode_hdr_frame(void *s, const char *hdr, int hdr_size, const char *frame,
                                                                        int frame_size, char *out, long cap)
{
        auto *p = (LDGM_session_gpu *) s;
        int n = 0;
        char *buf = p->encode_hdr_frame((char *) hdr, hdr_size, (char *) frame, frame_size, &n);
        if (!buf || n > cap) {
                return -1;
        }
        memcpy(out, buf, n);
        p->free_out_buf(buf);
        return n;
}
}
