// video_compress framework + the two compress modules of this library, host side (g++ only, no CUDA headers: everything goes
// through the cuda_wrapper / cuda_dxt / ugb200 C ABI exactly as UltraGrid modules do).
//
//   framework   src/video_compress.cpp:285-420,583-601   proxy state, API-shape dispatch, result queue
//   cuda_dxt    src/video_compress/cuda_dxt.cpp          tile API, synchronous; here: pinned pool, one stream,
//                                                        on-device input conversion, fused UYVY->DXT kernel
//   GPUJPEG     src/video_compress/gpujpeg.cpp           async frame API, one worker thread + encoder per entry of
//                                                        cuda_devices[], sequence-number reordering on pop (:643-722)
#include "video_compress.h"

#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <deque>
#include <map>
#include <mutex>
#include <string>
#include <strings.h>
#include <thread>
#include <vector>

#include "../../../include/cuda_dxt.h"
#include "../../../include/ugb200_jpeg.h"
#include "../../../include/ugb200_vcompress.h"
#include "gpujpeg_opts.h"
#include "video_codec.h"

unsigned int cuda_devices[MAX_CUDA_DEVICES] = { 0 };
unsigned int cuda_devices_count = 1;

// ---- registry (src/lib_common.cpp:73-85,186-204) -------------------------------------------------------------------
namespace {
struct lib_entry {
        std::string name;
        const void *info;
        enum library_class cls;
        int abi;
};
std::vector<lib_entry> &libraries()
{
        static std::vector<lib_entry> v;
        return v;
}
}  // namespace

void register_library(const char *name, const void *info, enum library_class cls, int abi_version)
{
        libraries().push_back(lib_entry{ name, info, cls, abi_version });
}
const void *load_library(const char *name, enum library_class cls, int abi_version)
{
        for (const lib_entry &e : libraries()) {
                if (strcasecmp(e.name.c_str(), name) == 0 && e.cls == cls && e.abi == abi_version) {
                        return e.info;
                }
        }
        return nullptr;
}

int get_libraries_for_class(enum library_class cls, int abi_version, const char **names, const void **infos, int max)
{
        int n = 0;
        for (const lib_entry &e : libraries()) {
                if (e.cls == cls && e.abi == abi_version && n < max) {
                        names[n] = e.name.c_str(), infos[n] = e.info;
                        ++n;
                }
        }
        return n;
}

// ---- pinned frame pool ------------------------------------------------------------------------------------------
// One free list per CUDA device: a frame that is pinned next to GPU k (cuda_wrapper_malloc_host_near) is only handed out for GPU k
// again, so that no D2H crosses the socket interconnect on a two-socket box.
namespace {
struct pinned_pool {
        std::mutex m;
        std::multimap<size_t, void *> free_bufs[MAX_CUDA_DEVICES + 1];
        ~pinned_pool()
        {
                for (auto &fb : free_bufs) {
                        for (auto &kv : fb) {
                                cuda_wrapper_free_host(kv.second);
                        }
                }
        }
};
pinned_pool &pool()
{
        static pinned_pool p;
        return p;
}
uint64_t now_ns()
{
        return (uint64_t) std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
}  // namespace

std::shared_ptr<video_frame> pinned_pool_get(size_t bytes, int device)
{
        const int list = device >= 0 && device < MAX_CUDA_DEVICES ? device : MAX_CUDA_DEVICES;
        void *buf = nullptr;
        {
                std::lock_guard<std::mutex> lk(pool().m);
                auto &fb = pool().free_bufs[list];
                auto it = fb.lower_bound(bytes);
                if (it != fb.end() && it->first <= bytes * 2) {
                        buf = it->second;
                        bytes = it->first;
                        fb.erase(it);
                }
        }
        if (!buf && cuda_wrapper_malloc_host_near(&buf, bytes, device) != CUDA_WRAPPER_SUCCESS) {
                return {};
        }
        video_frame *f = new video_frame();
        f->tile_count = 1;
        f->tiles[0].data = (char *) buf;
        const size_t cap = bytes;
        return std::shared_ptr<video_frame>(f, [cap, list](video_frame *fr) {  // back to the pool when the last reference drops
                {
                        std::lock_guard<std::mutex> lk(pool().m);
                        pool().free_bufs[list].emplace(cap, fr->tiles[0].data);
                }
                delete fr;
        });
}

// =====================================================================================================================
// module: cuda_dxt
// =====================================================================================================================
namespace {

#define CHECK_CUDA(cmd, msg, action)                                                                                                       \
        do {                                                                                                                               \
                if ((cmd) != CUDA_WRAPPER_SUCCESS) {                                                                                       \
                        fprintf(stderr, "[CUDA DXT] %s: %s\n", msg, cuda_wrapper_last_error_string());                                     \
                        action;                                                                                                            \
                }                                                                                                                          \
        } while (0)

/// one in-flight frame: own stream and buffers, so that the H2D of frame n+1 overlaps the kernel + D2H of frame n
struct dxt_slot {
        cuda_wrapper_stream_t stream = nullptr;
        char *cuda_src_buffer = nullptr;  ///< frame as captured, device memory
        char *cuda_in_buffer = nullptr;   ///< frame converted to in_codec (only when a conversion is needed)
        char *cuda_out_buffer = nullptr;
        std::shared_ptr<video_frame> in, out;
        bool busy = false;
};

struct state_video_compress_cuda_dxt {
        enum { DEPTH = 3 };
        struct video_desc saved_desc {};
        dxt_slot slots[DEPTH];
        codec_t in_codec = VIDEO_CODEC_NONE, out_codec = DXT1;
        decoder_t decoder{ VIDEO_CODEC_NONE, VIDEO_CODEC_NONE };
        size_t out_len = 0;
        unsigned head = 0, tail = 0;  ///< next slot to fill / oldest slot in flight
        std::deque<std::shared_ptr<video_frame>> ready;
        bool ended = false;
        std::mutex m;
        std::condition_variable cv;
};

void *cuda_dxt_compress_init(struct module *, const char *fmt)
{
        auto *s = new state_video_compress_cuda_dxt();
        if (fmt && fmt[0] != '\0') {  // cuda_dxt.cpp:108-119
                if (strcasecmp(fmt, "DXT5") == 0) {
                        s->out_codec = DXT5;
                } else if (strcasecmp(fmt, "DXT1") == 0) {
                        s->out_codec = DXT1;
                } else {
                        printf("usage:\n\t-c cuda_dxt[:DXT1|:DXT5]\n");
                        delete s;
                        return nullptr;
                }
        }
        return s;
}

void cleanup(state_video_compress_cuda_dxt *s)
{
        for (dxt_slot &sl : s->slots) {
                for (char **p : { &sl.cuda_src_buffer, &sl.cuda_in_buffer, &sl.cuda_out_buffer }) {
                        if (*p) {
                                cuda_wrapper_free(*p);
                                *p = nullptr;
                        }
                }
        }
}

bool configure_with(state_video_compress_cuda_dxt *s, struct video_desc desc)
{
        cleanup(s);
        if (desc.width % 4 || desc.height % 4) {
                fprintf(stderr, "[CUDA DXT] frame size must be divisible by 4\n");
                return false;
        }
        const codec_t supported_codecs[] = { RGB, UYVY, VIDEO_CODEC_NONE };  // cuda_dxt.cpp:153-154
        s->decoder = get_best_decoder_from(desc.color_spec, supported_codecs, &s->in_codec);
        if (!s->decoder) {
                fprintf(stderr, "[CUDA DXT] Unsupported codec: %s\n", get_codec_name(desc.color_spec));
                return false;
        }
        s->out_len = (size_t) desc.width * desc.height / (s->out_codec == DXT1 ? 2 : 1);  // cuda_dxt.cpp:176
        for (dxt_slot &sl : s->slots) {
                if (!sl.stream) {
                        CHECK_CUDA(cuda_wrapper_stream_create(&sl.stream), "Could not create stream", return false);
                }
                CHECK_CUDA(cuda_wrapper_malloc((void **) &sl.cuda_src_buffer, vc_get_datalen(desc.width, desc.height, desc.color_spec) + 64),
                           "Could not allocate CUDA input buffer", return false);
                if (desc.color_spec != s->in_codec) {
                        CHECK_CUDA(cuda_wrapper_malloc((void **) &sl.cuda_in_buffer, vc_get_datalen(desc.width, desc.height, s->in_codec)),
                                   "Could not allocate CUDA conversion buffer", return false);
                }
                CHECK_CUDA(cuda_wrapper_malloc((void **) &sl.cuda_out_buffer, s->out_len), "Could not allocate CUDA output buffer", return false);
        }
        return true;
}

/// enqueue H2D -> (convert) -> encode -> D2H for one frame on the slot's stream; nothing here waits for the GPU
bool enqueue(state_video_compress_cuda_dxt *s, dxt_slot &sl, const std::shared_ptr<video_frame> &tx)
{
        const struct video_desc desc = video_desc_from_frame(tx.get());
        const unsigned w = desc.width, h = desc.height;
        const char *in = tx->tiles[0].data;
        if (tx->mem_location == CPU_MEM) {  // H2D of the frame as captured; conversion (if any) happens on the device
                CHECK_CUDA(cuda_wrapper_memcpy_async(sl.cuda_src_buffer, in, vc_get_datalen(w, h, tx->color_spec),
                                                     CUDA_WRAPPER_MEMCPY_HOST_TO_DEVICE, sl.stream),
                           "Memcpy failed", return false);
                in = sl.cuda_src_buffer;
        }
        if (tx->color_spec != s->in_codec) {  // replaces the per-row CPU decoder loop of cuda_dxt.cpp:207-220
                const int rc = ugb200_pixfmt_convert(tx->color_spec, s->in_codec, sl.cuda_in_buffer, vc_get_linesize(w, s->in_codec), in,
                                                     vc_get_linesize(w, tx->color_spec), vc_get_linesize(w, s->in_codec), (int) h,
                                                     (long) vc_get_datalen(w, h, tx->color_spec), 0, 8, 16, sl.stream);
                if (rc != 0) {
                        fprintf(stderr, "[CUDA DXT] conversion kernel failed (%d)\n", rc);
                        return false;
                }
                in = sl.cuda_in_buffer;
        }
        int rc;
        if (s->in_codec == UYVY) {  // fused: no 4:4:4 intermediate (reference: cuda_yuv422_to_yuv444 + cuda_yuv_to_dxt*)
                rc = s->out_codec == DXT1 ? ugb200_uyvy_to_dxt1_async(in, sl.cuda_out_buffer, (int) w, (int) h, 0, sl.stream)
                                          : ugb200_uyvy_to_dxt6_async(in, sl.cuda_out_buffer, (int) w, (int) h, 0, sl.stream);
        } else {
                rc = s->out_codec == DXT1 ? ugb200_rgb_to_dxt1_async(in, sl.cuda_out_buffer, (int) w, (int) h, sl.stream)
                                          : ugb200_rgb_to_dxt6_async(in, sl.cuda_out_buffer, (int) w, (int) h, sl.stream);
        }
        if (rc != 0) {
                fprintf(stderr, "[CUDA DXT] Encoding failed (%d)\n", rc);
                return false;
        }
        sl.out = pinned_pool_get(s->out_len, (int) cuda_devices[0]);
        if (!sl.out) {
                return false;
        }
        sl.out->color_spec = s->out_codec, sl.out->fps = tx->fps, sl.out->interlacing = tx->interlacing, sl.out->seq = tx->seq;
        sl.out->tiles[0].width = w, sl.out->tiles[0].height = h, sl.out->tiles[0].data_len = (unsigned) s->out_len;
        CHECK_CUDA(cuda_wrapper_memcpy_async(sl.out->tiles[0].data, sl.cuda_out_buffer, s->out_len, CUDA_WRAPPER_MEMCPY_DEVICE_TO_HOST,
                                             sl.stream),
                   "Memcpy failed", return false);
        return true;
}

/// wait for the oldest frame in flight and move it to the ready queue (lock held)
void retire_oldest(state_video_compress_cuda_dxt *s)
{
        dxt_slot &sl = s->slots[s->tail % state_video_compress_cuda_dxt::DEPTH];
        if (cuda_wrapper_stream_synchronize(sl.stream) != CUDA_WRAPPER_SUCCESS) {
                fprintf(stderr, "[CUDA DXT] Synchronize failed: %s\n", cuda_wrapper_last_error_string());
                sl.out->tiles[0].data_len = 0;  // error marker: skipped by the consumer
        }
        sl.out->compress_end = now_ns();
        s->ready.push_back(std::move(sl.out));
        sl.in.reset();
        sl.busy = false;
        s->tail++;
}

/// async API, push side.  Up to DEPTH frames are in flight; the input frame is held until its result has been produced.
void cuda_dxt_compress_push(void *state, std::shared_ptr<video_frame> tx)
{
        auto *s = (state_video_compress_cuda_dxt *) state;
        std::unique_lock<std::mutex> lk(s->m);
        if (!tx) {  // poison pill
                s->ended = true;
                lk.unlock();
                s->cv.notify_all();
                return;
        }
        cuda_wrapper_set_device((int) cuda_devices[0]);  // cuda_dxt.cpp:194
        const struct video_desc desc = video_desc_from_frame(tx.get());
        if (!video_desc_eq(desc, s->saved_desc)) {
                while (s->tail != s->head) {
                        retire_oldest(s);
                }
                if (configure_with(s, desc)) {
                        s->saved_desc = desc;
                } else {
                        // the reference returns NULL here (cuda_dxt.cpp:198-204).  In the push/pop shape that is an EMPTY frame with this frame's seq:
                        // pop() stays in step with push() (cuda_dxt_compress_tile = push + pop must not block), and since cleanup() has already freed
                        // the device buffers the saved description is forgotten, so that the next good frame configures again
                        fprintf(stderr, "[CUDA DXT] Reconfiguration failed!\n");
                        s->saved_desc = {};
                        std::shared_ptr<video_frame> bad(new video_frame());
                        bad->seq = tx->seq;
                        s->ready.push_back(bad);
                        lk.unlock();
                        s->cv.notify_all();
                        return;
                }
        }
        dxt_slot &sl = s->slots[s->head % state_video_compress_cuda_dxt::DEPTH];
        if (sl.busy) {
                retire_oldest(s);
        }
        if (!enqueue(s, sl, tx)) {  // failed frame: empty marker keeps the sequence complete (video_compress.cpp:396-398)
                std::shared_ptr<video_frame> bad(new video_frame());
                bad->seq = tx->seq;
                cuda_wrapper_stream_synchronize(sl.stream);  // an H2D from tx may already be queued on the slot's stream
                sl.out.reset();
                while (s->tail != s->head) {
                        retire_oldest(s);
                }
                s->ready.push_back(bad);
        } else {
                sl.in = std::move(tx);
                sl.busy = true;
                s->head++;
        }
        lk.unlock();
        s->cv.notify_all();
}

std::shared_ptr<video_frame> cuda_dxt_compress_pop(void *state)
{
        auto *s = (state_video_compress_cuda_dxt *) state;
        std::unique_lock<std::mutex> lk(s->m);
        s->cv.wait(lk, [s] { return !s->ready.empty() || s->tail != s->head || s->ended; });
        if (s->ready.empty() && s->tail != s->head) {
                cuda_wrapper_set_device((int) cuda_devices[0]);
                retire_oldest(s);
        }
        if (s->ready.empty()) {
                return {};  // ended
        }
        std::shared_ptr<video_frame> f = std::move(s->ready.front());
        s->ready.pop_front();
        return f;
}

/// synchronous tile API of the reference module (cuda_dxt.cpp:186-266) = push + pop
std::shared_ptr<video_frame> cuda_dxt_compress_tile(void *state, std::shared_ptr<video_frame> tx)
{
        if (!tx) {
                return {};
        }
        cuda_dxt_compress_push(state, std::move(tx));
        std::shared_ptr<video_frame> out = cuda_dxt_compress_pop(state);
        return out && out->tiles[0].data_len ? out : std::shared_ptr<video_frame>();
}

void cuda_dxt_compress_done(void *state)
{
        auto *s = (state_video_compress_cuda_dxt *) state;
        {
                std::lock_guard<std::mutex> lk(s->m);
                while (s->tail != s->head) {
                        retire_oldest(s);
                }
        }
        cleanup(s);
        for (dxt_slot &sl : s->slots) {
                if (sl.stream) {
                        cuda_wrapper_stream_destroy(sl.stream);
                }
        }
        delete s;
}

// this build: asynchronous shape (frames of a stream overlap on the PCIe link); "cuda_dxt_sync" keeps the reference's tile API
const struct video_compress_info cuda_dxt_info = { cuda_dxt_compress_init, cuda_dxt_compress_done, nullptr, nullptr,
                                                   cuda_dxt_compress_push, cuda_dxt_compress_pop,  nullptr, nullptr,
                                                   nullptr };
REGISTER_MODULE(cuda_dxt, &cuda_dxt_info, LIBRARY_CLASS_VIDEO_COMPRESS, VIDEO_COMPRESS_ABI_VERSION);
const struct video_compress_info cuda_dxt_sync_info = { cuda_dxt_compress_init, cuda_dxt_compress_done, nullptr, cuda_dxt_compress_tile,
                                                        nullptr,                nullptr,                nullptr, nullptr,
                                                        nullptr };
REGISTER_MODULE(cuda_dxt_sync, &cuda_dxt_sync_info, LIBRARY_CLASS_VIDEO_COMPRESS, VIDEO_COMPRESS_ABI_VERSION);

// =====================================================================================================================
// module: GPUJPEG
// =====================================================================================================================
template <class T>
struct synchronized_queue {  // src/utils/synchronized_queue.h
        std::mutex m;
        std::condition_variable cv;
        std::deque<T> q;
        void push(T v)
        {
                {
                        std::lock_guard<std::mutex> lk(m);
                        q.push_back(std::move(v));
                }
                cv.notify_one();
        }
        T pop()
        {
                std::unique_lock<std::mutex> lk(m);
                cv.wait(lk, [this] { return !q.empty(); });
                T v = std::move(q.front());
                q.pop_front();
                return v;
        }
};

struct state_video_compress_gpujpeg;

struct encoder_state {  // one per CUDA device, gpujpeg.cpp:103-252
        state_video_compress_gpujpeg *parent;
        int device_id;
        ugb200_jpeg_encoder *encoder = nullptr;
        cuda_wrapper_stream_t stream = nullptr;
        char *cuda_src = nullptr, *cuda_conv = nullptr;
        size_t src_cap = 0, conv_cap = 0;
        codec_t enc_input_codec = VIDEO_CODEC_NONE;
        struct video_desc saved_desc {};
        synchronized_queue<std::shared_ptr<video_frame>> in_queue;
        std::thread thread;
        bool occupied = false;

        encoder_state(state_video_compress_gpujpeg *p, int dev) : parent(p), device_id(dev) {}
        std::shared_ptr<video_frame> compress_step(std::shared_ptr<video_frame> tx);
        void compress(std::shared_ptr<video_frame> frame);
        void worker();
        ~encoder_state();
};

struct state_video_compress_gpujpeg {
        gpujpeg_opts opts;  // quality, restart interval, interleaved, ... (gpujpeg.cpp:371-424)
        int lanes = 3;  // workers (encoder + stream + thread) per CUDA device: the H2D of one frame overlaps kernel + D2H of the previous ones
        std::vector<encoder_state *> workers;
        bool uses_worker_threads = false;
        synchronized_queue<std::shared_ptr<video_frame>> out_queue;
        std::map<uint32_t, std::shared_ptr<video_frame>> out_frames;
        std::mutex occupancy_lock;
        std::condition_variable worker_finished;
        uint32_t in_seq = 0, out_seq = 0;
        size_t ended_count = 0;
};

encoder_state::~encoder_state()
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

/// gpujpeg.cpp:557-634
std::shared_ptr<video_frame> encoder_state::compress_step(std::shared_ptr<video_frame> tx)
{
        cuda_wrapper_set_device(device_id);  // gpujpeg_set_device, :559
        if (!encoder) {
                if (cuda_wrapper_stream_create(&stream) != CUDA_WRAPPER_SUCCESS || !(encoder = ugb200_jpeg_encoder_create(stream))) {
                        fprintf(stderr, "[GPUJPEG] Failed to create encoder on device %d\n", device_id);
                        return {};
                }
        }
        const struct video_desc desc = video_desc_from_frame(tx.get());
        if (!video_desc_eq(desc, saved_desc)) {  // configure_with, :256-369
                const codec_t supported[] = { UYVY, RGB, VIDEO_CODEC_NONE };
                if (desc.color_spec == I420) {  // planar I420 goes into the encoder as it is (gpujpeg.cpp:262-266)
                        enc_input_codec = I420;
                } else if (!get_best_decoder_from(desc.color_spec, supported, &enc_input_codec)) {
                        fprintf(stderr, "[GPUJPEG] Unsupported codec: %s\n", get_codec_name(desc.color_spec));
                        return {};
                }
                if (!parent->opts.check_against_input(enc_input_codec == RGB ? jpeg_input::RGB : enc_input_codec == I420 ? jpeg_input::I420 : jpeg_input::UYVY)) {
                        return {};
                }
                saved_desc = desc;
        }
        const unsigned w = desc.width, h = desc.height;
        const char *in = tx->tiles[0].data;
        if (tx->mem_location == CPU_MEM) {
                const size_t n = vc_get_datalen(w, h, tx->color_spec);
                if (n + 64 > src_cap) {
                        if (cuda_src) {
                                cuda_wrapper_free(cuda_src);
                        }
                        src_cap = 0;
                        if (cuda_wrapper_malloc((void **) &cuda_src, n + 64) != CUDA_WRAPPER_SUCCESS) {
                                return {};
                        }
                        src_cap = n + 64;
                }
                if (cuda_wrapper_memcpy_async(cuda_src, in, n, CUDA_WRAPPER_MEMCPY_HOST_TO_DEVICE, stream) != CUDA_WRAPPER_SUCCESS) {
                        return {};
                }
                in = cuda_src;
        }
        if (tx->color_spec != enc_input_codec) {  // on-device line conversion instead of the CPU decoder of :592-605
                const size_t n = vc_get_datalen(w, h, enc_input_codec);
                if (n > conv_cap) {
                        if (cuda_conv) {
                                cuda_wrapper_free(cuda_conv);
                        }
                        conv_cap = 0;
                        if (cuda_wrapper_malloc((void **) &cuda_conv, n) != CUDA_WRAPPER_SUCCESS) {
                                return {};
                        }
                        conv_cap = n;
                }
                if (ugb200_pixfmt_convert(tx->color_spec, enc_input_codec, cuda_conv, vc_get_linesize(w, enc_input_codec), in,
                                          vc_get_linesize(w, tx->color_spec), vc_get_linesize(w, enc_input_codec), (int) h,
                                          (long) vc_get_datalen(w, h, tx->color_spec), 0, 8, 16, stream) != 0) {
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
        // the stream goes straight into the pooled (pinned) output frame: no encoder-owned buffer + memcpy as at :629-630
        const size_t out_cap = (size_t) w * h * 3 + 4096;  // :355 plus the header allowance of the encoder's own buffer (ugb200_jpeg.h): tiny or
                                                           // noisy frames at high quality exceed the raw size by their ~600-byte header
        std::shared_ptr<video_frame> out = pinned_pool_get(out_cap, device_id);
        if (!out) {
                return {};
        }
        size_t size = 0;
        if (ugb200_jpeg_encode_into_ex(encoder, in, 1, 0, (int) w, (int) h, enc_input_codec, &p, (uint8_t *) out->tiles[0].data, out_cap, &size) != 0) {  // :624
                return {};
        }
        out->color_spec = JPEG, out->fps = tx->fps, out->interlacing = tx->interlacing;
        out->tiles[0].width = w, out->tiles[0].height = h, out->tiles[0].data_len = (unsigned) size;
        return out;
}

/// gpujpeg.cpp:185-203
void encoder_state::compress(std::shared_ptr<video_frame> frame)
{
        if (frame) {
                const uint32_t seq = frame->seq;
                std::shared_ptr<video_frame> keep = frame;  // a failed step may have queued an asynchronous H2D from this frame: it must
                std::shared_ptr<video_frame> out = compress_step(std::move(frame));  // not be released before the stream is idle
                if (!out && stream) {
                        cuda_wrapper_stream_synchronize(stream);
                }
                keep.reset();
                if (!out) {  // an empty frame marks the error; pop() skips it (:194-198)
                        out = std::shared_ptr<video_frame>(new video_frame());
                        out->tiles[0].data_len = 0;
                }
                out->seq = seq;
                out->compress_end = now_ns();
                parent->out_queue.push(out);
        } else {
                parent->out_queue.push({});
        }
}

/// gpujpeg.cpp:209-225
void encoder_state::worker()
{
        cuda_wrapper_bind_thread_to_device(device_id);  // this thread feeds one GPU: run (and allocate) on that GPU's socket
        while (true) {
                std::shared_ptr<video_frame> frame = in_queue.pop();
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

void *gpujpeg_compress_init(struct module *, const char *opts)
{
        auto *s = new state_video_compress_gpujpeg();
        if (!s->opts.parse(opts) || s->opts.help) {  // gpujpeg.cpp:371-424
                if (s->opts.help) {
                        gpujpeg_opts::usage();
                }
                delete s;
                return nullptr;
        }
        s->lanes = s->opts.lanes;
        for (int l = 0; l < s->lanes; ++l) {  // one encoder per device (:446-466), times `lanes`; lane-major so that the first idle
                for (unsigned i = 0; i < cuda_devices_count; ++i) {  // workers found by push() spread over the devices first
                        s->workers.push_back(new encoder_state(s, (int) cuda_devices[i]));
                }
        }
        s->uses_worker_threads = s->workers.size() > 1;
        if (s->uses_worker_threads) {
                for (encoder_state *w : s->workers) {
                        w->thread = std::thread(&encoder_state::worker, w);
                }
        }
        return s;
}

/// state_video_compress_gpujpeg::push, gpujpeg.cpp:643-676
void gpujpeg_push(void *state, std::shared_ptr<video_frame> in_frame)
{
        auto *s = (state_video_compress_gpujpeg *) state;
        if (in_frame) {
                in_frame->seq = s->in_seq++;
        }
        if (!s->uses_worker_threads) {
                s->workers[0]->compress(std::move(in_frame));
                return;
        }
        if (!in_frame) {  // poison pill to all workers
                for (encoder_state *w : s->workers) {
                        w->in_queue.push({});
                }
                return;
        }
        size_t index = 0;
        std::unique_lock<std::mutex> lk(s->occupancy_lock);
        s->worker_finished.wait(lk, [s, &index] {  // first idle worker
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

/// state_video_compress_gpujpeg::pop, gpujpeg.cpp:688-722: results leave in submission order; failed frames are skipped
std::shared_ptr<video_frame> gpujpeg_pop(void *state)
{
        auto *s = (state_video_compress_gpujpeg *) state;
        while (true) {
                auto it = s->out_frames.find(s->out_seq);
                if (it != s->out_frames.end()) {
                        std::shared_ptr<video_frame> frame = it->second;
                        s->out_frames.erase(it);
                        s->out_seq += 1;
                        if (frame->tiles[0].data_len == 0) {
                                continue;
                        }
                        return frame;
                }
                std::shared_ptr<video_frame> frame = s->out_queue.pop();
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

void gpujpeg_compress_done(void *state)
{
        auto *s = (state_video_compress_gpujpeg *) state;
        if (s->uses_worker_threads) {
                for (encoder_state *w : s->workers) {
                        if (w->thread.joinable()) {
                                w->in_queue.push({});
                                w->thread.join();
                        }
                }
        }
        for (encoder_state *w : s->workers) {
                delete w;
        }
        delete s;
}

const struct video_compress_info gpujpeg_info = { gpujpeg_compress_init, gpujpeg_compress_done, nullptr, nullptr, gpujpeg_push, gpujpeg_pop,
                                                  nullptr,               nullptr,               nullptr };
REGISTER_MODULE(GPUJPEG, &gpujpeg_info, LIBRARY_CLASS_VIDEO_COMPRESS, VIDEO_COMPRESS_ABI_VERSION);

}  // namespace

// =====================================================================================================================
// framework (src/video_compress.cpp)
// =====================================================================================================================
struct compress_state {
        const video_compress_info *funcs = nullptr;
        void *state = nullptr;
        synchronized_queue<std::shared_ptr<video_frame>> queue;  // results of the synchronous API shapes
        bool poisoned = false;
};

int compress_init(struct module *parent, const char *config_string, struct compress_state **state)
{
        std::string cfg = config_string ? config_string : "";
        std::string name = cfg, opts;
        const size_t colon = cfg.find(':');
        if (colon != std::string::npos) {
                name = cfg.substr(0, colon);
                opts = cfg.substr(colon + 1);
        }
        const auto *info = (const video_compress_info *) load_library(name.c_str(), LIBRARY_CLASS_VIDEO_COMPRESS, VIDEO_COMPRESS_ABI_VERSION);
        if (!info) {
                fprintf(stderr, "Unknown or unavailable compression: %s\n", name.c_str());
                return -1;
        }
        void *st = info->init_func(parent, opts.c_str());
        if (!st) {
                return -1;
        }
        *state = new compress_state();
        (*state)->funcs = info;
        (*state)->state = st;
        return 0;
}

/// compress_frame, src/video_compress.cpp:333-402
void compress_frame(struct compress_state *s, std::shared_ptr<video_frame> frame)
{
        if (frame) {
                frame->compress_start = now_ns();
        }
        if (s->funcs->compress_frame_async_push_func) {
                s->funcs->compress_frame_async_push_func(s->state, std::move(frame));
                return;
        }
        if (!frame) {  // poison pill for the synchronous shapes
                s->queue.push({});
                return;
        }
        std::shared_ptr<video_frame> out = s->funcs->compress_tile_func ? s->funcs->compress_tile_func(s->state, frame)
                                                                        : s->funcs->compress_frame_func(s->state, frame);
        if (!out) {  // dropped frame (:396-398): hand an empty marker so that callers can count it
                out = std::shared_ptr<video_frame>(new video_frame());
                out->tiles[0].data_len = 0;
        }
        out->seq = frame->seq;
        out->compress_start = frame->compress_start;
        out->compress_end = now_ns();
        s->queue.push(out);
}

std::shared_ptr<video_frame> compress_pop(struct compress_state *s)
{
        if (s->funcs->compress_frame_async_pop_func) {
                return s->funcs->compress_frame_async_pop_func(s->state);
        }
        return s->queue.pop();
}

void compress_done(struct compress_state *s)
{
        if (!s) {
                return;
        }
        s->funcs->done(s->state);
        delete s;
}

// =====================================================================================================================
// plain-C driver (include/ugb200_vcompress.h)
// =====================================================================================================================
struct ugb200_compress {
        compress_state *cs = nullptr;
        uint32_t seq = 0;
        std::shared_ptr<video_frame> last;  // keeps the frame handed out by ugb200_compress_pop_ref alive
};

extern "C" {

int ugb200_set_cuda_devices(const int *devices, int count)
{
        if (count < 1 || count > MAX_CUDA_DEVICES || !devices) {
                return -1;
        }
        for (int i = 0; i < count; ++i) {
                cuda_devices[i] = (unsigned) devices[i];
        }
        cuda_devices_count = (unsigned) count;
        return 0;
}

ugb200_compress *ugb200_compress_init(const char *config)
{
        compress_state *cs = nullptr;
        if (compress_init(nullptr, config, &cs) != 0) {
                return nullptr;
        }
        auto *s = new ugb200_compress();
        s->cs = cs;
        return s;
}

int ugb200_compress_push(ugb200_compress *s, const void *data, int mem_location, int width, int height, int codec, double fps)
{
        if (!s) {
                return -1;
        }
        if (!data) {
                compress_frame(s->cs, {});
                return 0;
        }
        std::shared_ptr<video_frame> f(new video_frame());
        f->color_spec = (codec_t) codec, f->fps = fps, f->mem_location = mem_location ? CUDA_MEM : CPU_MEM, f->tile_count = 1;
        f->seq = s->seq++;
        f->tiles[0].width = (unsigned) width, f->tiles[0].height = (unsigned) height;
        f->tiles[0].data = (char *) data;
        f->tiles[0].data_len = (unsigned) vc_get_datalen(width, height, (codec_t) codec);
        compress_frame(s->cs, std::move(f));
        return 0;
}

int ugb200_compress_pop(ugb200_compress *s, void *out, size_t cap, size_t *out_len, int *out_codec, unsigned *seq)
{
        if (!s) {
                return -1;
        }
        std::shared_ptr<video_frame> f = compress_pop(s->cs);
        if (!f) {
                return 1;
        }
        if (out_len) {
                *out_len = f->tiles[0].data_len;
        }
        if (out_codec) {
                *out_codec = f->color_spec;
        }
        if (seq) {
                *seq = f->seq;
        }
        if (f->tiles[0].data_len == 0 || f->tiles[0].data_len > cap) {
                return -1;
        }
        memcpy(out, f->tiles[0].data, f->tiles[0].data_len);
        return 0;
}

int ugb200_get_best_decoder_from(int in_codec, const int *candidates, int count)
{
        codec_t cand[UGB_VIDEO_CODEC_COUNT + 1];
        int n = 0;
        for (; n < count && n < UGB_VIDEO_CODEC_COUNT; ++n) {
                cand[n] = (codec_t) candidates[n];
        }
        cand[n] = VIDEO_CODEC_NONE;
        codec_t out = VIDEO_CODEC_NONE;
        return get_best_decoder_from((codec_t) in_codec, cand, &out) ? (int) out : 0;
}

int ugb200_compress_pop_ref(ugb200_compress *s, const void **data, size_t *len, int *out_codec, unsigned *seq)
{
        if (!s || !data || !len) {
                return -1;
        }
        s->last = compress_pop(s->cs);
        if (!s->last) {
                return 1;
        }
        *data = s->last->tiles[0].data;
        *len = s->last->tiles[0].data_len;
        if (out_codec) {
                *out_codec = s->last->color_spec;
        }
        if (seq) {
                *seq = s->last->seq;
        }
        return s->last->tiles[0].data_len ? 0 : -1;
}

void ugb200_compress_done(ugb200_compress *s)
{
        if (s) {
                compress_done(s->cs);
                delete s;
        }
}

}  // extern "C"
