/* LDGM forward error correction on the GPU — the C ABI behind the `ldgm_gpu` session (ultragrid_b200/modules/ultragrid_ldgm_gpu.so),
 * byte-exact to the reference's CPU coder LDGM_session_cpu (ldgm/src/ldgm-session.cpp, ldgm-session-cpu.cpp).
 *
 * Matrix: `pcm` is the compact parity-check matrix exactly as LDGM_session::set_pcMatrix leaves it: m rows of w_f ints, each entry a
 *   node index (data packets 0..k-1, parity packets k..k+m-1, the staircase included) or -1.  1 <= k, m <= 8191, 2 <= w_f <= 128.
 * Frame layout (LDGM_session::encode_hdr_frame): int32 overall_size = hdr_size + frame_size, the header, the frame, zeros up to a
 *   multiple of k*4 bytes; packet size ps = that length / k (at most 65535, the reference keeps it in an unsigned short); then m parity
 *   packets of ps bytes, parity[j] = parity[j-1] ^ XOR{ data[i] : i in row j, 0 <= i < k }.
 * Decode (LDGM_session_cpu::decode_frame): a packet is received when the last merged (offset, length) range starting at or before it covers
 *   it; lost data packets are zeroed, then at most four Gauss-Seidel peeling sweeps over the m checks in row order, stopping when every
 *   data packet is known.  The device computes the sweep's schedule itself and replays its XORs level by level, so the bytes, including
 *   recovered parity packets, do not depend on thread scheduling.
 * Return codes: 0 ok, -1 bad arguments, -2 CUDA failure, -3 no matrix set, -5 output capacity too small.
 * Calls on one session are ordered on its stream; the host calls return when the results are in host memory. */
#ifndef UGB200_LDGM_H
#define UGB200_LDGM_H

#include <stddef.h>

#include "cuda_wrapper.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ugb200_ldgm ugb200_ldgm;

/* A coding session whose work runs on `stream` of the current device.  NULL on failure. */
UGB_API ugb200_ldgm *ugb200_ldgm_create(cuda_wrapper_stream_t stream);
UGB_API void ugb200_ldgm_destroy(ugb200_ldgm *s);

/* LDGM_session::set_params + set_pcMatrix: copies the matrix (host memory) to the device. */
UGB_API int ugb200_ldgm_set_matrix(ugb200_ldgm *s, const int *pcm, int k, int m, int w_f);

/* Size of the encoded buffer for a payload (header + frame) of `payload_size` bytes; *packet_size gets ps.  Negative on error. */
UGB_API long ugb200_ldgm_buffer_size(const ugb200_ldgm *s, int payload_size, int *packet_size);

/* LDGM_session::encode: `data` holds k packets of `packet_size` bytes, `parity` receives m packets (both host memory; pinned memory
 * avoids a staging copy).  packet_size is a positive multiple of 4, at most 65535. */
UGB_API int ugb200_ldgm_encode(ugb200_ldgm *s, const void *data, void *parity, int packet_size);

/* LDGM_session::encode_hdr_frame from host memory into `out` (host, pinned preferred) of `out_capacity` bytes; *out_size gets its length. */
UGB_API int ugb200_ldgm_encode_frame(ugb200_ldgm *s, const void *hdr, int hdr_size, const void *frame, int frame_size, void *out,
                                     size_t out_capacity, int *out_size);

/* The same layout and parity from a DEVICE frame (any alignment) into a DEVICE buffer, asynchronously on the session's stream; `hdr` is
 * host memory of at most 256 bytes, read before the call returns.  Lets a frame the JPEG encoder left on the device be coded before its
 * single copy to the host. */
UGB_API int ugb200_ldgm_encode_device(ugb200_ldgm *s, const void *hdr, int hdr_size, const void *frame, int frame_size, void *out,
                                      size_t out_capacity, int *out_size);

/* LDGM_session_cpu::decode_frame on `buf` (host, buf_size bytes, updated in place): `ranges` holds n_ranges (offset, length) pairs of
 * received bytes, treated as a std::map<int, int> (a repeated offset keeps its last length).  *frame_size gets the header's
 * overall_size when every data packet is known, else 0; the payload starts at buf + 4. */
UGB_API int ugb200_ldgm_decode(ugb200_ldgm *s, void *buf, int buf_size, const int *ranges, int n_ranges, int *frame_size);

#ifdef __cplusplus
}
#endif

#endif
