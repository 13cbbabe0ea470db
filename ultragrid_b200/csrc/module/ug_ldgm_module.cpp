/* The `ldgm_gpu` module in UltraGrid's REAL ABI: what src/rtp/ldgm.cpp:214-238 loads with load_library("ldgm_gpu",
 * LIBRARY_CLASS_UNDEFINED, LDGM_GPU_API_VERSION) when it is given `--param ldgm-device=GPU`, in place of the reference's
 * src/rtp/ldgm_gpu.cpp + ldgm/src/ldgm-session-gpu.cpp.  Compiled against the reference's own ldgm/src/ldgm-session.h, src/rtp/ldgm.hpp and
 * src/lib_common.h; the coding runs in libugb200 (include/ugb200_ldgm.h), byte-exact to LDGM_session_cpu.
 *
 * ldgm.cpp keeps the factory's result as unique_ptr<LDGM_session> and calls the base class's non-virtual set_params / set_pcMatrix /
 * encode_hdr_frame, which come from the host binary; only the virtual methods are implemented here.  encode_hdr_frame memsets and copies
 * into the buffer alloc_buf returns, so that buffer is pinned host memory from a pool, given back by free_out_buf. */
#include <stdio.h>
#include <string.h>

#include <map>
#include <mutex>
#include <vector>

#include "ldgm-session.h"
#include "lib_common.h"
#include "rtp/ldgm.hpp"

#include "../../../include/ugb200_ldgm.h"

namespace {

class LDGM_session_ugb200 : public LDGM_session {
public:
        LDGM_session_ugb200()
        {
                if (cuda_wrapper_stream_create(&stream) != 0) {
                        stream = nullptr;
                }
                coder = ugb200_ldgm_create(stream);
        }

        ~LDGM_session_ugb200() override
        {
                ugb200_ldgm_destroy(coder);
                for (auto &b : pool) {
                        cuda_wrapper_free_host(b.first);
                }
                if (stream) {
                        cuda_wrapper_stream_destroy(stream);
                }
        }

        void encode(char *data, char *parity) override
        {
                if (upload_matrix() != 0 || ugb200_ldgm_encode(coder, data, parity, packet_size) != 0) {
                        fprintf(stderr, "[ldgm_gpu] encode failed\n");
                }
        }

        /// the reference's encode_naive writes the same bytes as encode (an explicit staircase instead of a running XOR)
        void encode_naive(char *data, char *parity) override { encode(data, parity); }

        void *alloc_buf(int size) override
        {
                std::lock_guard<std::mutex> lk(lock);
                for (size_t i = 0; i < pool.size(); ++i) {
                        if (!pool[i].second.in_use && pool[i].second.size >= (size_t) size) {
                                pool[i].second.in_use = true;
                                return pool[i].first;
                        }
                }
                for (size_t i = 0; i < pool.size(); ++i) {  // a free buffer too small for this frame: replace it
                        if (!pool[i].second.in_use) {
                                cuda_wrapper_free_host(pool[i].first);
                                pool.erase(pool.begin() + i);
                                break;
                        }
                }
                void *p = nullptr;
                if (cuda_wrapper_malloc_host(&p, size) != 0) {
                        return nullptr;
                }
                pool.push_back({p, {(size_t) size, true}});
                return p;
        }

        void free_out_buf(char *buf) override
        {
                std::lock_guard<std::mutex> lk(lock);
                for (auto &b : pool) {
                        if (b.first == buf) {
                                b.second.in_use = false;
                        }
                }
        }

        char *decode_frame(char *received, int buf_size, int *frame_size, std::map<int, int> valid_data) override
        {
                std::vector<int> ranges;
                ranges.reserve(2 * valid_data.size());
                for (const auto &r : valid_data) {
                        ranges.push_back(r.first);
                        ranges.push_back(r.second);
                }
                packet_size = (unsigned short) (buf_size / (param_k + param_m));
                if (upload_matrix() != 0 ||
                    ugb200_ldgm_decode(coder, received, buf_size, ranges.data(), (int) valid_data.size(), frame_size) != 0) {
                        fprintf(stderr, "[ldgm_gpu] decode failed\n");
                        *frame_size = 0;
                }
                return received + LDGM_session::HEADER_SIZE;
        }

private:
        struct slot {
                size_t size;
                bool in_use;
        };

        /// set_pcMatrix is not virtual: the matrix goes to the device the first time it is used after a change
        int upload_matrix()
        {
                if (!pcm) {
                        return -3;
                }
                if (pcm == uploaded && param_k == up_k && param_m == up_m) {
                        return 0;
                }
                const int rc = ugb200_ldgm_set_matrix(coder, pcm, param_k, param_m, max_row_weight + 2);
                if (rc == 0) {
                        uploaded = pcm, up_k = param_k, up_m = param_m;
                }
                return rc;
        }

        cuda_wrapper_stream_t stream = nullptr;
        ugb200_ldgm *coder = nullptr;
        const int *uploaded = nullptr;
        int up_k = 0, up_m = 0;
        std::mutex lock;
        std::vector<std::pair<void *, slot>> pool;
};

LDGM_session *new_ldgm_session_ugb200() { return new LDGM_session_ugb200(); }

}  // namespace

REGISTER_MODULE(ldgm_gpu, reinterpret_cast<const void *>(new_ldgm_session_ugb200), LIBRARY_CLASS_UNDEFINED, LDGM_GPU_API_VERSION);
