// The two compress modules in UltraGrid's REAL ABI.
//
// This file is compiled against the reference's own headers (-I$(REF)/src, `make -C ultragrid_b200/csrc module`; no header is copied):
// struct video_frame (src/types.h:303-343), video_frame_pool (src/utils/video_frame_pool.h), video_compress_info and
// VIDEO_COMPRESS_ABI_VERSION (src/video_compress.h:71,221-236), REGISTER_MODULE (src/lib_common.h:124-160).  The result is
//     ultragrid_b200/modules/ultragrid_vcompress_cuda_dxt.so     replaces the module built from src/video_compress/cuda_dxt.cpp
//     ultragrid_b200/modules/ultragrid_vcompress_gpujpeg.so      replaces the module built from src/video_compress/gpujpeg.cpp
// in the form an unmodified UltraGrid loads from lib/ultragrid/ (lib_common.cpp:186-204: dlopen, the constructor of REGISTER_MODULE calls the
// host's register_library).  Everything CUDA happens behind the C ABI of libugb200.so (include/*.h), as in ../host/video_compress.cpp - that file
// is the same logic against mirror types for use without the reference tree (Python driver, bench); this one is the drop-in.
// tests/test_real_module.py loads both through the reference's own lib_common.cpp + video_compress.cpp (oracle/_ref/libugframework.so).
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <strings.h>
#include <thread>
#include <vector>

#include "host.h"                    // cuda_devices, cuda_devices_count, INIT_NOERR
#include "lib_common.h"              // REGISTER_MODULE, LIBRARY_CLASS_VIDEO_COMPRESS
#include "types.h"                   // video_frame, video_desc, codec_t, mem_location_t
#include "utils/synchronized_queue.h"
#include "utils/video_frame_pool.h"
#include "video_codec.h"             // vc_get_linesize, vc_get_datalen, get_codec_name
#include "video_compress.h"          // video_compress_info, VIDEO_COMPRESS_ABI_VERSION
#include "video_frame.h"             // video_desc_from_frame, video_desc_eq

#include "../host/gpujpeg_opts.h"
#include "../../../include/cuda_dxt.h"
#include "../../../include/ugb200.h"
#include "../../../include/ugb200_jpeg.h"
#include "../../../include/ugb200_vcompress.h"

using std::shared_ptr;

namespace {

/// pinned host memory for the pooled output frames (the role of cuda_buffer_data_allocator, cuda_dxt.cpp:68-83), on the GPU's NUMA node
struct pinned_allocator : public video_frame_pool_allocator {
        int device;
        explicit pinned_allocator(int dev) : device(dev) {}
        void *allocate(size_t size) override
        {
                void *ptr = nullptr;
                return cuda_wrapper_malloc_host_near(&ptr, size, device) == CUDA_WRAPPER_SUCCESS ? ptr : nullptr;
        }
        void deallocate(void *ptr) override { cuda_wrapper_free_host(ptr); }
        video_frame_pool_allocator *clone() const override { return new pinned_allocator(*this); }
};

bool dev_grow(char *&p, size_t &cap, size_t need)
{
        if (need <= cap) {
                return true;
        }
        if (p) {
                cuda_wrapper_free(p);
        }
        p = nullptr, cap = 0;
        if (cuda_wrapper_malloc((void **) &p, need) != CUDA_WRAPPER_SUCCESS) {
                return false;
        }
        cap = need;
        return true;
}

/// the line converter the device will run: best of `candidates` for `in` (ranking of get_best_decoder_from, pixfmt_conv.c:3148-3172)
codec_t pick_input_codec(codec_t in, std::initializer_list<codec_t> candidates)
{
        int cand[8], n = 0;
        for (codec_t c : candidates) {
                cand[n++] = (int) c;
        }
        return (codec_t) ugb200_get_best_decoder_from((int) in, cand, n);
}

// =====================================================================================================================
// cuda_dxt: synchronous tile API like the reference module (cuda_dxt.cpp:186-266)
// =====================================================================================================================
struct state_cuda_dxt {
        struct video_desc saved_desc {};
        codec_t in_codec = VIDEO_CODEC_NONE, out_codec = DXT1;
        cuda_wrapper_stream_t stream = nullptr;
        char *cuda_src = nullptr, *cuda_in = nullptr, *cuda_out = nullptr;
        size_t src_cap = 0, in_cap = 0, out_cap = 0, out_len = 0;
        video_frame_pool pool{ 0, pinned_allocator((int) cuda_devices[0]) };
};

void cuda_dxt_done(void *state)
{
        auto *s = (state_cuda_dxt *) state;
        for (char *p : { s->cuda_src, s->cuda_in, s->cuda_out }) {
                if (p) {
                        cuda_wrapper_free(p);
                }
        }
        if (s->stream) {
                cuda_wrapper_stream_destroy(s->stream);
        }
        delete s;
}

void *cuda_dxt_init(struct module *, const char *fmt)
{
        auto *s = new state_cuda_dxt();
        if (fmt && fmt[0] != '\0') {  // cuda_dxt.cpp:108-119
                if (strcasecmp(fmt, "DXT5") == 0) {
                        s->out_codec = DXT5;
                } else if (strcasecmp(fmt, "DXT1") == 0) {
                        s->out_codec = DXT1;
                } else {
                        printf("usage:\n\t-c cuda_dxt[:DXT1|:DXT5]\n");
                        delete s;
                        return strcasecmp(fmt, "help") == 0 ? INIT_NOERR : nullptr;
                }
        }
        return s;
}

bool cuda_dxt_configure(state_cuda_dxt *s, struct video_desc desc)
{
        if (desc.width % 4 != 0 || desc.height % 4 != 0) {
                fprintf(stderr, "[CUDA DXT] frame size must be divisible by 4\n");
                return false;
        }
        s->in_codec = pick_input_codec(desc.color_spec, { RGB, UYVY });  // cuda_dxt.cpp:153-154
        if (s->in_codec == VIDEO_CODEC_NONE) {
                fprintf(stderr, "[CUDA DXT] Unsupported codec: %s\n", get_codec_name(desc.color_spec));
                return false;
        }
        if (!s->stream && cuda_wrapper_stream_create(&s->stream) != CUDA_WRAPPER_SUCCESS) {
                return false;
        }
        s->out_len = (size_t) desc.width * desc.height / (s->out_codec == DXT1 ? 2 : 1);  // cuda_dxt.cpp:176
        if (!dev_grow(s->cuda_src, s->src_cap, vc_get_datalen(desc.width, desc.height, desc.color_spec) + 64) ||
            !dev_grow(s->cuda_in, s->in_cap, vc_get_datalen(desc.width, desc.height, s->in_codec) + 64) || !dev_grow(s->cuda_out, s->out_cap, s->out_len)) {
                fprintf(stderr, "[CUDA DXT] Could not allocate CUDA buffers: %s\n", cuda_wrapper_last_error_string());
                return false;
        }
        struct video_desc compressed = desc;
        compressed.color_spec = s->out_codec;
        compressed.tile_count = 1;
        s->pool.reconfigure(compressed, s->out_len);
        return true;
}

shared_ptr<video_frame> cuda_dxt_compress_tile(void *state, shared_ptr<video_frame> tx)
{
        auto *s = (state_cuda_dxt *) state;
        if (!tx) {
                return {};
        }
        cuda_wrapper_set_device((int) cuda_devices[0]);  // cuda_dxt.cpp:194
        const struct video_desc desc = video_desc_from_frame(tx.get());
        if (!video_desc_eq(desc, s->saved_desc)) {
                if (!cuda_dxt_configure(s, desc)) {
                        fprintf(stderr, "[CUDA DXT] Reconfiguration failed!\n");
                        s->saved_desc = {};
                        return {};
                }
                s->saved_desc = desc;
        }
        const unsigned w = desc.width, h = desc.height;
        const char *in = tx->tiles[0].data;
        if (tx->mem_location == CPU_MEM) {  // the frame as captured goes up; any conversion runs on the device (the reference converts on the CPU first, :207-220)
                if (cuda_wrapper_memcpy_async(s->cuda_src, in, vc_get_datalen(w, h, desc.color_spec), CUDA_WRAPPER_MEMCPY_HOST_TO_DEVICE, s->stream) !=
                    CUDA_WRAPPER_SUCCESS) {
                        return {};
                }
                in = s->cuda_src;
        }
        if (desc.color_spec != s->in_codec) {
                if (ugb200_pixfmt_convert((int) desc.color_spec, (int) s->in_codec, s->cuda_in, vc_get_linesize(w, s->in_codec), in, vc_get_linesize(w, desc.color_spec),
                                          vc_get_linesize(w, s->in_codec), (int) h, (long) vc_get_datalen(w, h, desc.color_spec), 0, 8, 16, s->stream) != 0) {
                        cuda_wrapper_stream_synchronize(s->stream);
                        return {};
                }
                in = s->cuda_in;
        }
        int rc;
        if (s->in_codec == UYVY) {  // fused: no 4:4:4 intermediate (reference: cuda_yuv422_to_yuv444 + cuda_yuv_to_dxt*, :223-257)
                rc = s->out_codec == DXT1 ? ugb200_uyvy_to_dxt1_async(in, s->cuda_out, (int) w, (int) h, 0, s->stream)
                                          : ugb200_uyvy_to_dxt6_async(in, s->cuda_out, (int) w, (int) h, 0, s->stream);
        } else {
                rc = s->out_codec == DXT1 ? ugb200_rgb_to_dxt1_async(in, s->cuda_out, (int) w, (int) h, s->stream)
                                          : ugb200_rgb_to_dxt6_async(in, s->cuda_out, (int) w, (int) h, s->stream);
        }
        shared_ptr<video_frame> out = rc == 0 ? s->pool.get_frame() : shared_ptr<video_frame>();
        if (!out || cuda_wrapper_memcpy_async(out->tiles[0].data, s->cuda_out, s->out_len, CUDA_WRAPPER_MEMCPY_DEVICE_TO_HOST, s->stream) != CUDA_WRAPPER_SUCCESS ||
            cuda_wrapper_stream_synchronize(s->stream) != CUDA_WRAPPER_SUCCESS) {
                cuda_wrapper_stream_synchronize(s->stream);
                fprintf(stderr, "[CUDA DXT] Encoding failed: %s\n", cuda_wrapper_last_error_string());
                return {};
        }
        out->tiles[0].data_len = (unsigned) s->out_len;
        vf_copy_metadata(out.get(), tx.get());
        return out;
}

const struct video_compress_info cuda_dxt_info = {
        cuda_dxt_init, cuda_dxt_done, nullptr, cuda_dxt_compress_tile, nullptr, nullptr, nullptr, nullptr, nullptr,
};

// =====================================================================================================================
// gpujpeg: asynchronous frame API, one worker (thread + encoder + stream) per entry of cuda_devices[] (gpujpeg.cpp:446-466,643-722)
// =====================================================================================================================
struct state_gpujpeg;

struct jpeg_worker {
        state_gpujpeg *parent;
        int device_id;
        ugb200_jpeg_encoder *encoder = nullptr;
        cuda_wrapper_stream_t stream = nullptr;
        char *cuda_src = nullptr, *cuda_conv = nullptr;
        size_t src_cap = 0, conv_cap = 0;
        codec_t enc_input_codec = VIDEO_CODEC_NONE;
        struct video_desc saved_desc {};
        video_frame_pool pool;
        synchronized_queue<shared_ptr<video_frame>, 1> in_queue;
        std::thread thread;
        bool occupied = false;

        jpeg_worker(state_gpujpeg *p, int dev) : parent(p), device_id(dev), pool(0, pinned_allocator(dev)) {}
        shared_ptr<video_frame> compress_step(shared_ptr<video_frame> tx);
        void compress(shared_ptr<video_frame> frame);
        void run();
        ~jpeg_worker();
};

struct state_gpujpeg {
        gpujpeg_opts opts;
        int lanes = 3;
        std::vector<jpeg_worker *> workers;
        bool threaded = false;
        synchronized_queue<shared_ptr<video_frame>, -1> out_queue;
        std::map<uint32_t, shared_ptr<video_frame>> out_frames;
        std::mutex occupancy_lock;
        std::condition_variable worker_finished;
        uint32_t in_seq = 0, out_seq = 0;
        size_t ended_count = 0;
};

jpeg_worker::~jpeg_worker()
{
        cuda_wrapper_set_device(device_id);
        if (encoder) {
                ugb200_jpeg_encoder_destroy(encoder);
        }
        if (cuda_src) {
                cuda_wrapper_free(cuda_src);
        }
        if (cuda_conv) {
                cuda_wrapper_free(cuda_conv);
        }
        if (stream) {
                cuda_wrapper_stream_destroy(stream);
        }
}

shared_ptr<video_frame> jpeg_worker::compress_step(shared_ptr<video_frame> tx)  // gpujpeg.cpp:557-634
{
        cuda_wrapper_set_device(device_id);
        if (!encoder && (cuda_wrapper_stream_create(&stream) != CUDA_WRAPPER_SUCCESS || !(encoder = ugb200_jpeg_encoder_create(stream)))) {
                fprintf(stderr, "[GPUJPEG] Failed to create encoder on device %d\n", device_id);
                return {};
        }
        const struct video_desc desc = video_desc_from_frame(tx.get());
        const unsigned w = desc.width, h = desc.height;
        if (!video_desc_eq(desc, saved_desc)) {  // configure_with, :256-369
                // I420 as it is (gpujpeg.cpp:262-266); RGBA with `alpha` as it is, four components (:227-236)
                enc_input_codec = desc.color_spec == I420                          ? I420
                                  : desc.color_spec == RGBA && parent->opts.alpha ? RGBA
                                                                                  : pick_input_codec(desc.color_spec, { UYVY, RGB });
                if (enc_input_codec == VIDEO_CODEC_NONE) {
                        fprintf(stderr, "[GPUJPEG] Unsupported codec: %s\n", get_codec_name(desc.color_spec));
                        return {};
                }
                if (!parent->opts.check_against_input(enc_input_codec == RGB    ? jpeg_input::RGB
                                                      : enc_input_codec == I420 ? jpeg_input::I420
                                                      : enc_input_codec == RGBA ? jpeg_input::RGBA
                                                                                : jpeg_input::UYVY)) {
                        return {};
                }
                struct video_desc compressed = desc;
                compressed.color_spec = JPEG;
                compressed.tile_count = 1;
                pool.reconfigure(compressed, (size_t) w * h * 3 + 4096);  // :355
                saved_desc = desc;
        }
        const char *in = tx->tiles[0].data;
        if (tx->mem_location == CPU_MEM) {
                const size_t n = vc_get_datalen(w, h, desc.color_spec);
                if (!dev_grow(cuda_src, src_cap, n + 64) || cuda_wrapper_memcpy_async(cuda_src, in, n, CUDA_WRAPPER_MEMCPY_HOST_TO_DEVICE, stream) != CUDA_WRAPPER_SUCCESS) {
                        return {};
                }
                in = cuda_src;
        }
        if (desc.color_spec != enc_input_codec) {  // on the device instead of the CPU decoder of :592-605
                if (!dev_grow(cuda_conv, conv_cap, vc_get_datalen(w, h, enc_input_codec) + 64) ||
                    ugb200_pixfmt_convert((int) desc.color_spec, (int) enc_input_codec, cuda_conv, vc_get_linesize(w, enc_input_codec), in, vc_get_linesize(w, desc.color_spec),
                                          vc_get_linesize(w, enc_input_codec), (int) h, (long) vc_get_datalen(w, h, desc.color_spec), 0, 8, 16, stream) != 0) {
                        return {};
                }
                in = cuda_conv;
        }
        struct ugb200_jpeg_params_ex p;
        ugb200_jpeg_default_params_ex(&p);
        if (parent->opts.quality != -1) {
                p.base.quality = parent->opts.quality;
        }
        p.base.restart_interval = parent->opts.restart_interval;
        p.base.interleaved = parent->opts.interleaved ? 1 : 0;
        p.subsampling = parent->opts.subsampling;  // as checked against the input: the input's own layout
        p.color_space = parent->opts.internal_cs;
        if (enc_input_codec == RGBA) {
                p.subsampling = 4444;  // GPUJPEG_SUBSAMPLING_4444, gpujpeg.cpp:316-328
        }
        shared_ptr<video_frame> out = pool.get_frame();
        size_t size = 0;
        if (!out || ugb200_jpeg_encode_into_ex(encoder, in, 1, 0, (int) w, (int) h, (int) enc_input_codec, &p, (uint8_t *) out->tiles[0].data, (size_t) w * h * 3 + 4096, &size) != 0) {
                return {};
        }
        out->tiles[0].data_len = (unsigned) size;
        vf_copy_metadata(out.get(), tx.get());
        return out;
}

void jpeg_worker::compress(shared_ptr<video_frame> frame)  // gpujpeg.cpp:185-203
{
        if (!frame) {
                parent->out_queue.push({});
                return;
        }
        const uint32_t seq = frame->seq;
        shared_ptr<video_frame> keep = frame;
        shared_ptr<video_frame> out = compress_step(std::move(frame));
        if (!out) {
                if (stream) {
                        cuda_wrapper_stream_synchronize(stream);  // an H2D from the input frame may still be queued
                }
                struct video_desc d {};
                d.tile_count = 1;
                out = shared_ptr<video_frame>(vf_alloc_desc(d), vf_free);  // an empty frame marks the error, pop() skips it (:194-198)
                out->tiles[0].data_len = 0;
        }
        out->seq = seq;
        parent->out_queue.push(out);
}

void jpeg_worker::run()  // gpujpeg.cpp:209-225
{
        cuda_wrapper_bind_thread_to_device(device_id);
        while (true) {
                shared_ptr<video_frame> frame = in_queue.pop();
                if (!frame) {
                        compress({});
                        break;
                }
                compress(std::move(frame));
                {
                        std::lock_guard<std::mutex> lk(parent->occupancy_lock);
                        occupied = false;
                }
                parent->worker_finished.notify_one();
        }
}

void gpujpeg_done(void *state)
{
        auto *s = (state_gpujpeg *) state;
        for (jpeg_worker *w : s->workers) {
                if (w->thread.joinable()) {
                        w->in_queue.push({});
                        w->thread.join();
                }
                delete w;
        }
        delete s;
}

void *gpujpeg_init(struct module *, const char *opts)
{
        auto *s = new state_gpujpeg();
        if (!s->opts.parse(opts)) {  // gpujpeg.cpp:371-424
                delete s;
                return nullptr;
        }
        if (s->opts.help) {
                gpujpeg_opts::usage();
                delete s;
                return INIT_NOERR;
        }
        s->lanes = s->opts.lanes;
        for (int l = 0; l < s->lanes; ++l) {
                for (unsigned i = 0; i < cuda_devices_count; ++i) {
                        s->workers.push_back(new jpeg_worker(s, (int) cuda_devices[i]));
                }
        }
        s->threaded = s->workers.size() > 1;
        if (s->threaded) {
                for (jpeg_worker *w : s->workers) {
                        w->thread = std::thread(&jpeg_worker::run, w);
                }
        }
        return s;
}

void gpujpeg_push(void *state, shared_ptr<video_frame> in_frame)  // gpujpeg.cpp:643-676
{
        auto *s = (state_gpujpeg *) state;
        if (in_frame) {
                in_frame->seq = s->in_seq++;
        }
        if (!s->threaded) {
                s->workers[0]->compress(std::move(in_frame));
                return;
        }
        if (!in_frame) {
                for (jpeg_worker *w : s->workers) {
                        w->in_queue.push({});
                }
                return;
        }
        size_t index = 0;
        std::unique_lock<std::mutex> lk(s->occupancy_lock);
        s->worker_finished.wait(lk, [s, &index] {
                for (index = 0; index < s->workers.size(); ++index) {
                        if (!s->workers[index]->occupied) {
                                return true;
                        }
                }
                return false;
        });
        s->workers[index]->occupied = true;
        lk.unlock();
        s->workers[index]->in_queue.push(std::move(in_frame));
}

shared_ptr<video_frame> gpujpeg_pop(void *state)  // gpujpeg.cpp:688-722
{
        auto *s = (state_gpujpeg *) state;
        while (true) {
                auto it = s->out_frames.find(s->out_seq);
                if (it != s->out_frames.end()) {
                        shared_ptr<video_frame> frame = it->second;
                        s->out_frames.erase(it);
                        s->out_seq += 1;
                        if (frame->tiles[0].data_len == 0) {
                                continue;
                        }
                        return frame;
                }
                shared_ptr<video_frame> frame = s->out_queue.pop();
                if (!frame) {
                        if (++s->ended_count == s->workers.size()) {
                                return {};
                        }
                        continue;
                }
                if (frame->seq == s->out_seq) {
                        s->out_seq += 1;
                        if (frame->tiles[0].data_len == 0) {
                                continue;
                        }
                        return frame;
                }
                s->out_frames[frame->seq] = frame;
        }
}

const struct video_compress_info gpujpeg_info = {
        gpujpeg_init, gpujpeg_done, nullptr, nullptr, gpujpeg_push, gpujpeg_pop, nullptr, nullptr, nullptr,
};

}  // namespace

#if defined UGB_MODULE_CUDA_DXT
REGISTER_MODULE(cuda_dxt, &cuda_dxt_info, LIBRARY_CLASS_VIDEO_COMPRESS, VIDEO_COMPRESS_ABI_VERSION);
#elif defined UGB_MODULE_GPUJPEG
REGISTER_MODULE(gpujpeg, &gpujpeg_info, LIBRARY_CLASS_VIDEO_COMPRESS, VIDEO_COMPRESS_ABI_VERSION);
#else
#error "define UGB_MODULE_CUDA_DXT or UGB_MODULE_GPUJPEG"
#endif
