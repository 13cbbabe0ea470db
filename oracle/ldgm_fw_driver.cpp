// TEST INFRASTRUCTURE - the host side of UltraGrid's LDGM path for tests/test_ldgm.py: the UNMODIFIED module loader (lib_common.cpp in
// _ref/libugframework.so) and the UNMODIFIED LDGM_session base class and CPU coder (ldgm/src/*.cpp), linked by ldgm.mk into
// _ref/libldgm_fw.so.  A module is dlopen()ed as open_all() does (lib_common.cpp:197), the factory is looked up exactly as
// src/rtp/ldgm.cpp:224-231 does, and both sessions are driven only through LDGM_session *.  Never part of the product.
#include <dlfcn.h>
#include <stdio.h>
#include <string.h>

#include <map>
#include <string>

#include "ldgm-session-cpu.h"
#include "lib_common.h"
#include "rtp/ldgm.hpp"

extern "C" {
#define API __attribute__((visibility("default")))

API int ldf_load_module(const char *path)
{
        if (!dlopen(path, RTLD_NOW | RTLD_GLOBAL)) {
                fprintf(stderr, "ldf_load_module: %s\n", dlerror());
                return -1;
        }
        return 0;
}

/// gpu: the factory load_library("ldgm_gpu", LIBRARY_CLASS_UNDEFINED, LDGM_GPU_API_VERSION) returns; else LDGM_session_cpu
API void *ldf_create(int gpu)
{
        if (!gpu) {
                return static_cast<LDGM_session *>(new LDGM_session_cpu());
        }
        auto loader = reinterpret_cast<LDGM_session *(*)()>(
                const_cast<void *>(load_library("ldgm_gpu", LIBRARY_CLASS_UNDEFINED, LDGM_GPU_API_VERSION)));
        return loader ? loader() : nullptr;
}

API void ldf_destroy(void *s) { delete static_cast<LDGM_session *>(s); }

/// set_params + set_pcMatrix, as ldgm::set_params does (src/rtp/ldgm.cpp:163-206)
API int ldf_set(void *s, int k, int m, int c, const char *matrix_file)
{
        auto *p = static_cast<LDGM_session *>(s);
        p->set_params(k, m, c);
        try {
                p->set_pcMatrix(const_cast<char *>(matrix_file));
        } catch (const std::string &) {
                return -1;
        }
        return 0;
}

/// encode_hdr_frame, copied to out, then free_out_buf; the buffer length, or -1
API int ldf_encode(void *s, const char *hdr, int hdr_size, const char *frame, int frame_size, char *out, long cap)
{
        auto *p = static_cast<LDGM_session *>(s);
        int n = 0;
        char *buf = p->encode_hdr_frame(const_cast<char *>(hdr), hdr_size, const_cast<char *>(frame), frame_size, &n);
        if (!buf) {
                return -1;
        }
        const int ok = n <= cap;
        if (ok) {
                memcpy(out, buf, n);
        }
        p->free_out_buf(buf);
        return ok ? n : -1;
}

/// decode_frame on buf in place; *frame_size, or -1 when the returned pointer is not buf + 4
API int ldf_decode(void *s, char *buf, int buf_size, const int *ranges, int n)
{
        std::map<int, int> valid;
        for (int i = 0; i < n; ++i) {
                valid[ranges[2 * i]] = ranges[2 * i + 1];
        }
        int frame_size = -1;
        char *payload = static_cast<LDGM_session *>(s)->decode_frame(buf, buf_size, &frame_size, valid);
        return payload == buf + 4 ? frame_size : -1;
}
}
