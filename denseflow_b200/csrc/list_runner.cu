// list_runner.cu — video-list dispatch over several GPUs (SURVEY §8 e; BASELINE.json configs[4]).
//
// The reference turns a list.txt into a vector of videos (/root/reference/tools/denseflow.cpp:54-81) and one DenseFlow
// object walks it on GPU 0 (src/denseflow_gpu.cpp:482-489), handing FlowBuffers (item_data, base_start, last_buffer;
// include/dense_flow.h:10-18) to the writer thread, which marks a video done only after its LAST buffer has been
// written (src/denseflow_gpu.cpp:456-470).  Here the same list is drained by W workers — one host thread per entry of
// `devices`, each with its own engine handle, streams and pinned staging — from ONE work queue: an in-process atomic
// counter, or a counter in POSIX shared memory when the workers are separate processes (one process per GPU).  There is
// no data-path collective.  Every entry point runs one scheduler, run_windows, over windows of a video's frames: a worker
// reads a window, computes it and delivers it once every earlier window of the video has been delivered, and the video's
// last window carries the reference's `last_buffer` meaning.  A worker runs the video it took to its end, then takes the
// next one.
//
// The entry points differ in where a window's frames come from and what its outputs are.  dfb_list_run reads gray clips
// in host memory and hands out flows or quantised planes.  dfb_list_run_videos reads the videos as the reference takes
// them (colour frames or `-if` JPEG files) and hands out the files the reference writes: flow JPEGs, PNGs or h5 planes, or
// with step 0 the extracted frames.  dfb_list_run_stream pulls the frames from the caller one window at a time, so a list
// of long videos runs in bounded memory.  dfb_list_run_windows does the same and also shares a video's windows once the
// queue is empty: idle workers join the unfinished videos, so one video runs on every worker and one worker reads a
// window while another computes the last.
//
// This file is a client of the C ABI (dfb_create / dfb_calc_batch_host[_u8] / dfb_process_* / dfb_extract_frames_* /
// dfb_destroy): it adds no arithmetic.
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <climits>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <list>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/denseflow_b200.h"
#include "common.cuh"

struct dfb_queue {
    std::atomic<long> *counter = nullptr;  // lives in the shared mapping
    std::string name;
    int fd = -1;
};

namespace {
using clk = std::chrono::steady_clock;
double seconds_since(clk::time_point t0) { return std::chrono::duration<double>(clk::now() - t0).count(); }

void set_error(char *err, size_t err_len, const std::string &m) {
    if (err && err_len) std::snprintf(err, err_len, "%s", m.c_str());
}
}  // namespace

extern "C" {

int dfb_queue_open(const char *name, int create, dfb_queue **out) {
    if (!name || !out || name[0] != '/') return DFB_ERR_INVALID_ARG;
    *out = nullptr;
    const int fd = shm_open(name, create ? (O_CREAT | O_RDWR) : O_RDWR, 0600);
    if (fd < 0) return DFB_ERR_INVALID_ARG;
    if (create && ftruncate(fd, 64) != 0) {
        close(fd);
        return DFB_ERR_INVALID_ARG;
    }
    void *p = mmap(nullptr, 64, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    if (p == MAP_FAILED) {
        close(fd);
        return DFB_ERR_INVALID_ARG;
    }
    static_assert(sizeof(std::atomic<long>) == sizeof(long) && std::atomic<long>::is_always_lock_free, "plain word in shared memory");
    dfb_queue *q = new dfb_queue();
    q->counter = reinterpret_cast<std::atomic<long> *>(p);
    q->name = name;
    q->fd = fd;
    if (create) q->counter->store(0);
    *out = q;
    return DFB_OK;
}

long dfb_queue_next(dfb_queue *q) { return q ? q->counter->fetch_add(1) : -1; }

void dfb_queue_reset(dfb_queue *q) {
    if (q) q->counter->store(0);
}

void dfb_queue_close(dfb_queue *q, int unlink_name) {
    if (!q) return;
    munmap(q->counter, 64);
    close(q->fd);
    if (unlink_name) shm_unlink(q->name.c_str());
    delete q;
}

struct dfb_list_runner {
    std::string algorithm;
    int max_w = 0, max_h = 0;
    struct Worker {
        int device = 0;
        dfb_handle *h = nullptr;
        int max_w = 0, max_h = 0;           // the frame size h was created for (dfb_list_run_stream grows it)
        dfb_counters retired{};             // counters of the handles this worker replaced during the current run
        dfb::PinnedBuffer<uint8_t> pinned;  // outputs of the one window the worker holds: the copy engines write them straight in
    };
    std::vector<Worker> workers;
};

int dfb_list_open(const char *algorithm, const int *devices, int n_workers, int max_width, int max_height, dfb_list_runner **out, char *err,
                  size_t err_len) {
    if (!out) return DFB_ERR_INVALID_ARG;
    *out = nullptr;
    if (!algorithm || !devices || n_workers < 1 || n_workers > DFB_LIST_MAX_WORKERS || max_width <= 0 || max_height <= 0) {
        set_error(err, err_len, "dfb_list_open: bad arguments");
        return DFB_ERR_INVALID_ARG;
    }
    dfb_list_runner *r = new dfb_list_runner();
    r->algorithm = algorithm;
    r->max_w = max_width;
    r->max_h = max_height;
    r->workers = std::vector<dfb_list_runner::Worker>(n_workers);
    for (int wi = 0; wi < n_workers; ++wi) {
        dfb_list_runner::Worker &w = r->workers[wi];
        w.device = devices[wi];
        w.max_w = max_width;
        w.max_h = max_height;
        if (int rc = dfb_create(algorithm, w.device, max_width, max_height, &w.h)) {
            set_error(err, err_len, "worker " + std::to_string(wi) + ": " + dfb_last_error(nullptr));
            dfb_list_close(r);
            return rc;
        }
    }
    *out = r;
    return DFB_OK;
}

void dfb_list_close(dfb_list_runner *r) {
    if (!r) return;
    for (auto &w : r->workers) dfb_destroy(w.h);
    delete r;  // and with it the workers' pinned rings
}

}  // extern "C"

namespace {

// What reading or computing one window gives: DFB_OK, or the error that ends the run.
struct ItemResult {
    int rc = DFB_OK;
    std::string error;
};

// A chain that saw the frames of video k from f0 on names frame i as "frame i: ..."; the list names it in the video.
std::string video_error(long k, int f0, const char *msg) {
    const std::string m = msg ? msg : "";
    int i = 0, n = 0;
    if (std::sscanf(m.c_str(), "frame %d: %n", &i, &n) == 1 && n > 0)
        return "video " + std::to_string(k) + ": frame " + std::to_string(f0 + i) + ": " + m.substr(n);
    return "video " + std::to_string(k) + ": " + m;
}

// The arguments of dfb_list_run_videos and dfb_list_run_stream that every video of the call shares.
struct VideoArgs {
    int step = 1, astep = 1, bound = 0, save_type = DFB_SAVE_JPG, quality = 95, new_width = 0, new_height = 0, new_short = 0;
    int chunk_flows = 64;
    dfb_files_done_fn done = nullptr;
    void *user = nullptr;
};

// The checks both video entry points make first (`name` leads the message of a malformed call), in this order: the call,
// check_param's bound (src/denseflow_gpu.cpp:23-35: the bound matters only to the flow modes), the quality, the -nw/-nh/-ns
// rule.  Fills a, or writes the message and returns the code.
int check_video_args(const char *name, int step, int bound, int save_type, int quality, int jpeg_exact, int new_width, int new_height,
                     int new_short, int chunk_flows, VideoArgs &a, char *err, size_t err_len) {
    if ((save_type != DFB_SAVE_JPG && save_type != DFB_SAVE_PNG && save_type != DFB_SAVE_H5) || (jpeg_exact != 0 && jpeg_exact != 1)) {
        set_error(err, err_len, std::string(name) + ": bad arguments (save_type is DFB_SAVE_JPG or DFB_SAVE_PNG, jpeg_exact 0 or 1)");
        return DFB_ERR_INVALID_ARG;
    }
    if (step != 0 && bound <= 0) {
        set_error(err, err_len, "bound should > 0!");
        return DFB_ERR_INVALID_ARG;
    }
    const bool writes_jpeg = step == 0 || save_type == DFB_SAVE_JPG;
    if (writes_jpeg && (quality < 1 || quality > 100)) {
        set_error(err, err_len, std::string(name) + ": quality must be in 1..100");
        return DFB_ERR_INVALID_ARG;
    }
    int dw = 0, dh = 0;
    if (int rc = dfb_new_size(1, 1, new_width, new_height, new_short, &dw, &dh)) {
        set_error(err, err_len, dfb_last_error(nullptr));
        return rc;
    }
    a.step = step;
    a.astep = std::abs(step);
    a.bound = bound;
    a.save_type = save_type;
    a.quality = quality;
    a.new_width = new_width;
    a.new_height = new_height;
    a.new_short = new_short;
    a.chunk_flows = chunk_flows > 0 ? chunk_flows : 64;
    return DFB_OK;
}

bool malformed(const dfb_video &v) {
    const bool bgr = v.kind == DFB_VIDEO_BGR;
    return (!bgr && v.kind != DFB_VIDEO_JPEG) || v.n_frames < 0 || (v.n_frames > 0 && (bgr ? !v.bgr : (!v.jpeg || !v.jpeg_len))) ||
           (bgr && (v.width <= 0 || v.height <= 0));
}

// A video's source and destination size.
struct Geometry {
    int sw = 0, sh = 0, dw = 0, dh = 0;
    bool resize = false;
};

// get_new_size (src/denseflow_gpu.cpp:44-80) reads frame 0: a BGR video gives its size, a JPEG file the size in its markers.
// v holds at least one frame, frame 0 at index `off`.
int size_video(const dfb_video &v, int off, const VideoArgs &a, Geometry &g) {
    if (v.kind == DFB_VIDEO_BGR) {
        g.sw = v.width;
        g.sh = v.height;
    } else if (int rc = dfb_jpeg_info(v.jpeg[off], v.jpeg_len[off], &g.sw, &g.sh)) {
        return rc;
    }
    dfb_new_size(g.sw, g.sh, a.new_width, a.new_height, a.new_short, &g.dw, &g.dh);
    g.resize = g.dw != g.sw || g.dh != g.sh;
    return DFB_OK;
}

// Frames first .. first + n - 1 of a video: frame first + i is v->bgr[off + i] or v->jpeg[off + i].  `ends`: no frame follows.
struct Window {
    const dfb_video *v = nullptr;
    int off = 0, n = 0;
    bool ends = false;
};

// The outputs of a window: flows [f0, f0 + m) read frames f0 .. f0 + m - 1 + |step|; with step 0 every frame is an output.
int window_outputs(const VideoArgs &a, const Window &win) { return a.step != 0 ? std::max(win.n - a.astep, 0) : win.n; }

// One window of video idx through the chains.  fetch(f0, max_n, win) returns an ItemResult and fills win with frames f0 ..
// f0 + max_n - 1, fewer when the video ends there; g is the video's geometry by the time fetch returns a window with a
// frame.  A window serves up to chunk_flows outputs, so consecutive windows overlap by |step| frames (the overlap the
// reference keeps between its own <= 512-frame batches, src/denseflow_gpu.cpp:182-189,204-205) and indices stay global
// (FlowBuffer::base_start).  Once every file of the window is in the worker's pinned ring, deliver(f0, m, win.ends, files,
// lens) hands them on; a failure returns before it.
template <typename Fetch, typename Deliver>
ItemResult run_window(dfb_list_runner::Worker &w, int wi, long idx, const VideoArgs &a, const Geometry &g, int f0, Window &win, Fetch &&fetch,
                      Deliver &&deliver) {
    const bool flow = a.step != 0;
    const int per = flow && a.save_type != DFB_SAVE_PNG ? 2 : 1;  // jpg and h5: an x and a y output per flow
    const int chunk = a.chunk_flows;
    std::vector<uint8_t *> out(2 * chunk), ox(chunk), oy(chunk);
    std::vector<size_t> lens(2 * chunk), lx(chunk), ly(chunk);
    ItemResult fr = fetch(f0, chunk + a.astep, win);
    if (fr.rc != DFB_OK) return fr;
    const int m = window_outputs(a, win);
    int rc = DFB_OK;
    if (m > 0) {
        const dfb_video &v = *win.v;
        const bool bgr = v.kind == DFB_VIDEO_BGR;
        const uint8_t *const *bf = bgr ? v.bgr + win.off : nullptr;
        const uint8_t *const *jf = bgr ? nullptr : v.jpeg + win.off;
        const size_t *jl = bgr ? nullptr : v.jpeg_len + win.off;
        const int dwa = g.resize ? g.dw : 0, dha = g.resize ? g.dh : 0;  // 0 / 0: no resize
        const size_t cap = !flow                         ? dfb_jpeg_max_bytes_bgr(g.dw, g.dh)
                           : a.save_type == DFB_SAVE_PNG ? dfb_png_max_bytes(g.dw, g.dh)
                           : a.save_type == DFB_SAVE_H5  ? (size_t)g.dw * g.dh * sizeof(float)
                                                         : dfb_jpeg_max_bytes(g.dw, g.dh);
        try {
            w.pinned.allocate((size_t)chunk * per * cap);
        } catch (const dfb::CudaError &) {
            return {DFB_ERR_CUDA, "worker " + std::to_string(wi) + ": pinned file ring allocation failed"};
        }
        for (int k = 0; k < per * chunk; ++k) out[k] = (uint8_t *)w.pinned + (size_t)k * cap;
        if (!flow) {
            rc = bgr ? dfb_extract_frames_host(w.h, bf, m, g.sw, g.sh, dwa, dha, a.quality, out.data(), cap, lens.data())
                     : dfb_extract_frames_jpeg_host(w.h, jf, jl, m, dwa, dha, a.quality, out.data(), cap, lens.data());
        } else if (a.save_type == DFB_SAVE_PNG) {
            rc = bgr ? dfb_process_bgr_batch_host_png(w.h, bf, m + a.astep, a.step, g.sw, g.sh, dwa, dha, out.data(), cap, lens.data())
                     : dfb_process_jpeg_batch_host_png(w.h, jf, jl, m + a.astep, a.step, dwa, dha, out.data(), cap, lens.data());
        } else if (a.save_type == DFB_SAVE_H5) {
            // the two float planes of flow i straight into files 2 i / 2 i + 1 (pinned: a direct DMA); every file is whole
            std::vector<float *> px(m), py(m);
            for (int i = 0; i < m; ++i) {
                px[i] = reinterpret_cast<float *>(out[2 * i]);
                py[i] = reinterpret_cast<float *>(out[2 * i + 1]);
                lens[2 * i] = lens[2 * i + 1] = cap;
            }
            rc = bgr ? dfb_process_bgr_batch_host_planes(w.h, bf, m + a.astep, a.step, g.sw, g.sh, dwa, dha, px.data(), py.data())
                     : dfb_process_jpeg_batch_host_planes(w.h, jf, jl, m + a.astep, a.step, dwa, dha, px.data(), py.data());
        } else {
            for (int i = 0; i < m; ++i) {
                ox[i] = out[2 * i];
                oy[i] = out[2 * i + 1];
            }
            rc = bgr ? dfb_process_bgr_batch_host(w.h, bf, m + a.astep, a.step, g.sw, g.sh, dwa, dha, a.bound, a.quality, ox.data(),
                                                  oy.data(), cap, lx.data(), ly.data())
                     : dfb_process_jpeg_batch_host(w.h, jf, jl, m + a.astep, a.step, dwa, dha, a.bound, a.quality, ox.data(), oy.data(),
                                                   cap, lx.data(), ly.data());
            for (int i = 0; i < m; ++i) {
                lens[2 * i] = lx[i];
                lens[2 * i + 1] = ly[i];
            }
        }
    }
    if (rc != DFB_OK) return {rc, video_error(idx, f0, dfb_last_error(w.h))};
    deliver(f0, m, win.ends, out.data(), lens.data());
    return {};
}

// run() over videos with the call's jpeg_exact: the runner owns the handles, so it is set on each of them and restored
// afterwards.
template <typename Run>
int with_jpeg_exact(dfb_list_runner *r, int jpeg_exact, Run &&run) {
    const int n_workers = (int)r->workers.size();
    std::vector<double> exact_before(n_workers, 0);
    for (int wi = 0; wi < n_workers; ++wi) {
        dfb_get_param(r->workers[wi].h, "jpeg_exact", &exact_before[wi]);
        dfb_set_param(r->workers[wi].h, "jpeg_exact", jpeg_exact);
    }
    const int rc = run();
    for (int wi = 0; wi < n_workers; ++wi) dfb_set_param(r->workers[wi].h, "jpeg_exact", exact_before[wi]);
    return rc;
}

// Worker w's handle for destination frames of dw x dh: a smaller handle is replaced by one at least that large in both
// dimensions, with the old one's jpeg_exact.  Its counters stay in the run's stats.  On failure the old handle stays.
int fit_worker(dfb_list_runner *r, dfb_list_runner::Worker &w, int dw, int dh, std::string &error) {
    if (dw <= w.max_w && dh <= w.max_h) return DFB_OK;
    const int mw = std::max(w.max_w, dw), mh = std::max(w.max_h, dh);
    dfb_handle *h = nullptr;
    if (int rc = dfb_create(r->algorithm.c_str(), w.device, mw, mh, &h)) {
        error = dfb_last_error(nullptr);
        return rc;
    }
    double exact = 0;
    dfb_get_param(w.h, "jpeg_exact", &exact);
    dfb_set_param(h, "jpeg_exact", exact);
    dfb_counters c{};
    if (dfb_get_counters(w.h, &c) == DFB_OK) {
        w.retired.kernel_launches += c.kernel_launches;
        w.retired.h2d_bytes += c.h2d_bytes;
        w.retired.d2h_bytes += c.d2h_bytes;
    }
    dfb_destroy(w.h);
    w.h = h;
    w.max_w = mw;
    w.max_h = mh;
    return DFB_OK;
}

// The caller's window of frames first .. first + max_n - 1 of video idx, into cur and win.  The video is sized by its first
// window with a frame; every later frame must have frame 0's size.
ItemResult fetch_stream_window(dfb_frames_fn source, const VideoArgs &a, long idx, int first, int max_n, dfb_video &cur, Window &win,
                               Geometry &g) {
    const std::string k = "video " + std::to_string(idx) + ": ";
    cur = dfb_video{};
    char msg[512] = "";
    if (source(a.user, (int)idx, first, max_n, &cur, msg, sizeof msg) != 0) return {DFB_ERR_INVALID_ARG, k + msg};
    if (malformed(cur) || cur.n_frames > max_n)
        return {DFB_ERR_INVALID_ARG, k + "the source returned a malformed window at frame " + std::to_string(first)};
    win = {&cur, 0, cur.n_frames, cur.n_frames < max_n};
    if (cur.n_frames == 0) return {};
    if (first == 0)
        if (int rc = size_video(cur, 0, a, g)) return {rc, k + dfb_last_error(nullptr)};
    // a BGR window has one size; a JPEG file that cannot be sized is left to the decoder, which names the fault
    const int n_check = cur.kind == DFB_VIDEO_BGR ? 1 : cur.n_frames;
    for (int i = 0; i < n_check; ++i) {
        int fw = cur.width, fh = cur.height;
        if (cur.kind == DFB_VIDEO_JPEG && dfb_jpeg_info(cur.jpeg[i], cur.jpeg_len[i], &fw, &fh) != DFB_OK) continue;
        if (fw != g.sw || fh != g.sh)
            return {DFB_ERR_SIZE, k + "frame " + std::to_string(first + i) + ": " + std::to_string(fw) + "x" + std::to_string(fh) +
                                      ", frame 0 is " + std::to_string(g.sw) + "x" + std::to_string(g.sh)};
    }
    return {};
}

// What the workers share about one video taken from the queue, under the run's mutex.
struct SharedVideo {
    long idx = 0;
    int next_first = 0;           // first frame of the next window to read
    bool reading = false;         // a source call for the video is in progress
    bool ended = false;           // no window is read any more: the final one has been, or the video was cut
    int next_deliver = 0;         // first_index of the next window to deliver
    int cut = INT_MAX;            // windows from this first frame on are not delivered (a failure, or the run stopping)
    int failed_first = INT_MAX;   // the earliest failed window, and its error
    ItemResult failure;
    uint64_t flows = 0;           // outputs of the windows delivered so far
    Geometry g;                   // set by window 0
};

// The dispatch of every list entry point (its policy is in the header, under dfb_list_run_windows).  Workers take videos from
// `queue` (or an in-process counter).  A worker holds at most one window: it claims a video's reader, reads the next window,
// releases the reader, computes the window and delivers it once every earlier window of the video has been delivered.  Reads
// of one video are in order and never overlap, so every window read is held by a worker that will deliver or drop it, and a
// worker waiting for its turn waits only on windows read before its own.
//   read(wi, idx, first, max_n, win, g)  fills win with frames first .. first + max_n - 1 of video idx, fewer when the video
//                                        ends there; the read of window 0 sizes the video into g.
//   body(w, wi, idx, g, f0, win, fetch, deliver)  runs window f0 on worker w: fetch(first, max_n, win) reads it (read, then
//                                        the scheduler's bookkeeping), and deliver(first, m, ends, call) runs call(), which
//                                        hands on the window's m outputs, in the video's order.
// share = false: a worker runs the video it took to its end, then takes the next one, and stops once the queue is empty; a
// failure cuts only the failed video, and every other worker finishes the video it holds and takes no new one.  share = true:
// once the queue is empty, an idle worker joins the earliest unfinished video whose reader is free, or waits for one; a
// failure cuts every video at its next unread window.
template <typename Read, typename Body>
int run_windows(dfb_list_runner *r, int n_videos, dfb_queue *queue, bool share, const VideoArgs &a, Read &&read, Body &&body,
                dfb_list_stats *stats, char *err, size_t err_len) {
    const int n_workers = (int)r->workers.size();
    dfb_list_stats st{};
    st.workers = n_workers;
    for (auto &w : r->workers) {  // the workers' engine counters from zero
        dfb_reset_counters(w.h);
        w.retired = dfb_counters{};
    }
    std::mutex mtx;
    std::condition_variable cv;
    std::list<SharedVideo> active;  // videos taken and not finished, in the order they were taken
    long local_next = 0;
    bool queue_empty = false;
    SharedVideo *failed = nullptr;  // the first video to fail; its error is its earliest failed window's

    // Under mtx: window `first` of v failed.  An earlier window's failure replaces a later one's.  The videos it cuts read no
    // other window, and deliver none that has not been read.
    auto fail = [&](SharedVideo &v, int first, ItemResult res) {
        if (first < v.failed_first) {
            v.failed_first = first;
            v.failure = std::move(res);
        }
        v.cut = std::min(v.cut, first);
        if (!failed) failed = &v;
        for (auto &s : active) {
            if (!share && &s != &v) continue;
            s.cut = std::min(s.cut, s.next_first);
            s.ended = true;
        }
        cv.notify_all();
    };
    const auto t_start = clk::now();

    auto worker = [&](int wi) {
        dfb_list_runner::Worker &w = r->workers[wi];
        cudaSetDevice(w.device);
        double busy = 0;
        long own = -1;  // the video this worker took from the queue
        std::unique_lock<std::mutex> lk(mtx);
        for (;;) {
            // A worker runs its own video to its end, then takes the next one.  With share, once the queue is empty, it joins
            // the earliest unfinished video whose reader is free, or waits for one.
            SharedVideo *v = nullptr;
            for (;;) {
                if (!share || !queue_empty) {
                    for (auto &s : active)
                        if (s.idx == own && !s.ended) v = &s;
                    if (v || failed) break;
                    const long idx = queue ? dfb_queue_next(queue) : local_next++;
                    if (idx < n_videos) {
                        v = &active.emplace_back();
                        v->idx = own = idx;
                        break;
                    }
                    queue_empty = true;
                    if (!share) break;
                }
                if (failed) break;
                bool readable = false;  // a window is left to read
                for (auto &s : active) {
                    if (s.ended) continue;
                    readable = true;
                    if (!s.reading) {
                        v = &s;
                        break;
                    }
                }
                if (v || !readable) break;
                cv.wait(lk);
            }
            if (!v) break;
            v->reading = true;
            const int f0 = v->next_first;
            lk.unlock();

            const auto t0 = clk::now();
            const std::string k = "video " + std::to_string(v->idx) + ": ";
            Window win;
            bool dropped = false;
            auto fetch = [&](int first, int max_n, Window &got) -> ItemResult {
                ItemResult fr = read(wi, v->idx, first, max_n, got, v->g);
                const int m = fr.rc == DFB_OK ? window_outputs(a, got) : 0;
                {
                    std::lock_guard<std::mutex> g(mtx);
                    v->reading = false;
                    if (first >= v->cut) {  // the run stopped while this window was read: neither a window nor a failure
                        dropped = true;
                        return {DFB_ERR_INVALID_ARG, {}};
                    }
                    if (fr.rc != DFB_OK) {
                        v->ended = true;
                        return fr;
                    }
                    v->next_first = first + m;
                    v->ended = got.ends;
                    cv.notify_all();
                }
                // every worker that computes a window of the video, its first included, fits its handle to it here
                std::string e;
                if (m > 0)
                    if (int rc = fit_worker(r, w, v->g.dw, v->g.dh, e)) return {rc, k + e};
                return fr;
            };
            // Everything this window adds to the video and to the stats is recorded under mtx before next_deliver moves
            // on: from then on the worker holding the video's next window may deliver it, and after the final window it
            // removes the video.  The worker does not touch v once its window is delivered.
            auto deliver = [&](int first, int m, bool ends, auto &&call) {
                std::unique_lock<std::mutex> dl(mtx);
                cv.wait(dl, [&] { return first >= v->cut || v->next_deliver == first; });
                if (first >= v->cut) {
                    dropped = true;
                    return;
                }
                dl.unlock();
                // every output of this window is in host memory now, and every earlier window of the video has been delivered;
                // `ends` is the reference's FlowBuffer::last_buffer, the only point at which a video may be marked done
                call();
                dl.lock();
                if (a.step != 0) {
                    st.flows_per_worker[wi] += m;
                    v->flows += m;
                }
                if (ends) {
                    ++st.clips;
                    ++st.clips_per_worker[wi];
                    st.flows += v->flows;
                    st.frames += (uint64_t)first + win.n;
                    active.remove_if([&](const SharedVideo &s) { return &s == v; });
                } else {
                    v->next_deliver = first + m;
                }
                cv.notify_all();
            };
            ItemResult res = body(w, wi, v->idx, v->g, f0, win, fetch, deliver);
            busy += seconds_since(t0);
            lk.lock();
            // a window that was delivered or dropped is done with; a failed one was never delivered, so v is still listed
            if (!dropped && res.rc != DFB_OK) fail(*v, f0, std::move(res));
        }
        st.busy_seconds_per_worker[wi] = busy;
        st.finish_seconds_per_worker[wi] = seconds_since(t_start);
    };

    if (n_videos > 0) {  // each worker on a host thread of its own, worker 0 on the caller's
        std::vector<std::thread> threads;
        for (int wi = 1; wi < n_workers; ++wi) threads.emplace_back(worker, wi);
        worker(0);
        for (auto &t : threads) t.join();
    }
    st.seconds = seconds_since(t_start);
    for (auto &w : r->workers) {  // the counters of every handle the workers used
        dfb_counters c{};
        if (dfb_get_counters(w.h, &c) == DFB_OK) {
            st.kernel_launches += c.kernel_launches;
            st.h2d_bytes += c.h2d_bytes;
            st.d2h_bytes += c.d2h_bytes;
        }
        st.kernel_launches += w.retired.kernel_launches;
        st.h2d_bytes += w.retired.h2d_bytes;
        st.d2h_bytes += w.retired.d2h_bytes;
    }
    if (stats) *stats = st;
    if (failed) {
        set_error(err, err_len, failed->failure.error);
        return failed->failure.rc;
    }
    return DFB_OK;
}

// Frames first .. first + max_n - 1 of a video whose n_frames frames are all in host memory.
Window slice(const dfb_video *v, int n_frames, int first, int max_n) {
    const int n = std::max(std::min(max_n, n_frames - first), 0);
    return {v, first, n, first + n >= n_frames};
}

// The entry points that hand out files: run_window computes each window, whose files go to a.done, under the call's jpeg_exact.
template <typename Read>
int run_files(dfb_list_runner *r, int n_videos, dfb_queue *queue, bool share, int jpeg_exact, const VideoArgs &a, Read &&read,
              dfb_list_stats *stats, char *err, size_t err_len) {
    auto body = [&](dfb_list_runner::Worker &w, int wi, long idx, const Geometry &g, int f0, Window &win, auto &fetch, auto &deliver) {
        return run_window(w, wi, idx, a, g, f0, win, fetch, [&](int first, int m, bool ends, uint8_t *const *files, const size_t *lens) {
            deliver(first, m, ends, [&] {
                if (a.done) a.done(a.user, (int)idx, w.device, first, m, ends, files, lens);
            });
        });
    };
    return with_jpeg_exact(r, jpeg_exact, [&] { return run_windows(r, n_videos, queue, share, a, read, body, stats, err, err_len); });
}

// dfb_list_run_stream and dfb_list_run_windows: windows from the caller's source.  A worker holds one window at a time, so the
// latest one it read, cur[wi], is all it keeps.
int run_source(dfb_list_runner *r, int n_videos, dfb_frames_fn source, dfb_queue *queue, bool share, int jpeg_exact, const VideoArgs &a,
               dfb_list_stats *stats, char *err, size_t err_len) {
    std::vector<dfb_video> cur(r->workers.size());
    auto read = [&](int wi, long idx, int first, int max_n, Window &win, Geometry &g) {
        return fetch_stream_window(source, a, idx, first, max_n, cur[wi], win, g);
    };
    return run_files(r, n_videos, queue, share, jpeg_exact, a, read, stats, err, err_len);
}

}  // namespace

extern "C" {

int dfb_list_run(dfb_list_runner *r, const dfb_clip *clips, int n_clips, int step, int bound, int chunk_flows, dfb_queue *queue,
                 dfb_chunk_done_fn done, void *user, dfb_list_stats *stats, char *err, size_t err_len) {
    if (!r || (!clips && n_clips > 0) || n_clips < 0 || step == 0 || bound < 0) {
        set_error(err, err_len, "dfb_list_run: bad arguments (step must be non-zero: step 0 is the frame-extraction mode)");
        return DFB_ERR_INVALID_ARG;
    }
    if (chunk_flows <= 0) chunk_flows = 64;
    const int astep = std::abs(step);
    for (int i = 0; i < n_clips; ++i) {
        if (clips[i].n_frames < 0 || clips[i].width <= 0 || clips[i].height <= 0 || (clips[i].n_frames > 0 && !clips[i].frames)) {
            set_error(err, err_len, "dfb_list_run: clip " + std::to_string(i) + " is malformed");
            return DFB_ERR_INVALID_ARG;
        }
        if (clips[i].width > r->max_w || clips[i].height > r->max_h) {
            set_error(err, err_len, "dfb_list_run: clip " + std::to_string(i) + " exceeds the size given to dfb_list_open");
            return DFB_ERR_SIZE;
        }
    }
    const size_t px_max = (size_t)r->max_w * r->max_h;
    const size_t out_bytes = (size_t)chunk_flows * px_max * (bound > 0 ? 2 : 8);
    VideoArgs a;  // the windows: flows [f0, f0 + m) of window f0 read frames f0 .. f0 + m - 1 + |step|
    a.step = step;
    a.astep = astep;
    a.chunk_flows = chunk_flows;

    auto read = [&](int, long idx, int first, int max_n, Window &win, Geometry &) {
        win = slice(nullptr, clips[idx].n_frames, first, max_n);
        return ItemResult{};
    };
    auto body = [&](dfb_list_runner::Worker &w, int wi, long idx, const Geometry &, int f0, Window &win, auto &fetch,
                    auto &deliver) -> ItemResult {
        ItemResult fr = fetch(f0, chunk_flows + astep, win);
        if (fr.rc != DFB_OK) return fr;
        try {
            w.pinned.allocate(out_bytes);
        } catch (const dfb::CudaError &) {
            return {DFB_ERR_CUDA, "worker " + std::to_string(wi) + ": pinned output allocation failed"};
        }
        uint8_t *qbuf = bound > 0 ? (uint8_t *)w.pinned : nullptr;
        float *fbuf = bound > 0 ? nullptr : reinterpret_cast<float *>((uint8_t *)w.pinned);
        std::vector<uint8_t *> qx(chunk_flows), qy(chunk_flows);
        std::vector<float *> fl(chunk_flows);
        const dfb_clip &c = clips[idx];
        const size_t px = (size_t)c.width * c.height;
        for (int i = 0; i < chunk_flows; ++i) {
            qx[i] = qbuf ? qbuf + (size_t)(2 * i) * px : nullptr;
            qy[i] = qbuf ? qbuf + (size_t)(2 * i + 1) * px : nullptr;
            fl[i] = fbuf ? fbuf + (size_t)i * px * 2 : nullptr;
        }
        const int m = window_outputs(a, win);  // a clip of n frames has max(n - |step|, 0) flows, src/denseflow_gpu.cpp:308
        int rc = DFB_OK;
        if (m > 0)
            rc = bound > 0 ? dfb_calc_batch_host_u8(w.h, c.frames + f0, m + astep, step, c.width, c.height, bound, qx.data(), qy.data())
                           : dfb_calc_batch_host(w.h, c.frames + f0, m + astep, step, c.width, c.height, fl.data());
        if (rc != DFB_OK) return {rc, "clip " + std::to_string(idx) + ": " + dfb_last_error(w.h)};
        deliver(f0, m, win.ends, [&] {
            if (done) done(user, (int)idx, w.device, f0, m, win.ends, bound > 0 ? qx.data() : nullptr, bound > 0 ? qy.data() : nullptr,
                           bound > 0 ? nullptr : fl.data());
        });
        return {};
    };
    return run_windows(r, n_clips, queue, false, a, read, body, stats, err, err_len);
}

int dfb_list_run_videos(dfb_list_runner *r, const dfb_video *videos, int n_videos, int step, int bound, int save_type, int quality,
                        int jpeg_exact, int new_width, int new_height, int new_short, int chunk_flows, dfb_queue *queue,
                        dfb_files_done_fn done, void *user, dfb_list_stats *stats, char *err, size_t err_len) {
    if (!r || (!videos && n_videos > 0) || n_videos < 0) {
        set_error(err, err_len, "dfb_list_run_videos: bad arguments (save_type is DFB_SAVE_JPG or DFB_SAVE_PNG, jpeg_exact 0 or 1)");
        return DFB_ERR_INVALID_ARG;
    }
    VideoArgs a;
    if (int rc = check_video_args("dfb_list_run_videos", step, bound, save_type, quality, jpeg_exact, new_width, new_height, new_short,
                                  chunk_flows, a, err, err_len))
        return rc;
    a.done = done;
    a.user = user;
    // every video's source and destination size, before any work
    std::vector<Geometry> geo(n_videos);
    for (int i = 0; i < n_videos; ++i) {
        const dfb_video &v = videos[i];
        if (malformed(v)) {
            set_error(err, err_len, "dfb_list_run_videos: video " + std::to_string(i) + " is malformed");
            return DFB_ERR_INVALID_ARG;
        }
        if (v.kind == DFB_VIDEO_JPEG && v.n_frames == 0) continue;  // an empty frame folder: nothing to size
        Geometry &g = geo[i];
        if (int rc = size_video(v, 0, a, g)) {
            set_error(err, err_len, "video " + std::to_string(i) + ": " + dfb_last_error(nullptr));
            return rc;
        }
        if (g.dw > r->max_w || g.dh > r->max_h) {
            set_error(err, err_len, "dfb_list_run_videos: video " + std::to_string(i) + " (" + std::to_string(g.dw) + "x" + std::to_string(g.dh) +
                                        " after resizing) exceeds the size given to dfb_list_open");
            return DFB_ERR_SIZE;
        }
    }
    auto read = [&](int, long idx, int first, int max_n, Window &win, Geometry &g) {
        win = slice(&videos[idx], videos[idx].n_frames, first, max_n);
        g = geo[idx];
        return ItemResult{};
    };
    return run_files(r, n_videos, queue, false, jpeg_exact, a, read, stats, err, err_len);
}

int dfb_list_run_stream(dfb_list_runner *r, int n_videos, dfb_frames_fn source, int step, int bound, int save_type, int quality,
                        int jpeg_exact, int new_width, int new_height, int new_short, int chunk_flows, dfb_queue *queue,
                        dfb_files_done_fn done, void *user, dfb_list_stats *stats, char *err, size_t err_len) {
    if (!r || !source || n_videos < 0) {
        set_error(err, err_len, "dfb_list_run_stream: bad arguments (save_type is DFB_SAVE_JPG or DFB_SAVE_PNG, jpeg_exact 0 or 1)");
        return DFB_ERR_INVALID_ARG;
    }
    VideoArgs a;
    if (int rc = check_video_args("dfb_list_run_stream", step, bound, save_type, quality, jpeg_exact, new_width, new_height, new_short,
                                  chunk_flows, a, err, err_len))
        return rc;
    a.done = done;
    a.user = user;
    return run_source(r, n_videos, source, queue, false, jpeg_exact, a, stats, err, err_len);
}

int dfb_list_run_windows(dfb_list_runner *r, int n_videos, dfb_frames_fn source, int step, int bound, int save_type, int quality,
                         int jpeg_exact, int new_width, int new_height, int new_short, int chunk_flows, dfb_queue *queue,
                         dfb_files_done_fn done, void *user, dfb_list_stats *stats, char *err, size_t err_len) {
    if (!source || n_videos < 0) {
        set_error(err, err_len, "dfb_list_run_windows: bad arguments (a source is required, n_videos >= 0)");
        return DFB_ERR_INVALID_ARG;
    }
    VideoArgs a;
    if (int rc = check_video_args("dfb_list_run_windows", step, bound, save_type, quality, jpeg_exact, new_width, new_height, new_short,
                                  chunk_flows, a, err, err_len))
        return rc;
    if (!r) {
        set_error(err, err_len, "dfb_list_run_windows: bad arguments (no runner)");
        return DFB_ERR_INVALID_ARG;
    }
    a.done = done;
    a.user = user;
    return run_source(r, n_videos, source, queue, true, jpeg_exact, a, stats, err, err_len);
}

int dfb_run_list(const char *algorithm, const int *devices, int n_workers, const dfb_clip *clips, int n_clips, int step, int bound,
                 int chunk_flows, dfb_queue *queue, dfb_chunk_done_fn done, void *user, dfb_list_stats *stats, char *err, size_t err_len) {
    if (!algorithm || !devices || n_workers < 1 || n_workers > DFB_LIST_MAX_WORKERS || (!clips && n_clips > 0) || n_clips < 0 || step == 0 ||
        bound < 0) {
        set_error(err, err_len, "dfb_run_list: bad arguments (step must be non-zero: step 0 is the frame-extraction mode)");
        return DFB_ERR_INVALID_ARG;
    }
    if (n_clips == 0) {  // tools/denseflow.cpp:86: nothing is created when every video of the list is already done
        dfb_list_stats st{};
        st.workers = n_workers;
        if (stats) *stats = st;
        return DFB_OK;
    }
    int max_w = 1, max_h = 1;
    for (int i = 0; i < n_clips; ++i) {
        max_w = std::max(max_w, clips[i].width);
        max_h = std::max(max_h, clips[i].height);
    }
    dfb_list_runner *r = nullptr;
    if (int rc = dfb_list_open(algorithm, devices, n_workers, max_w, max_h, &r, err, err_len)) return rc;
    const int rc = dfb_list_run(r, clips, n_clips, step, bound, chunk_flows, queue, done, user, stats, err, err_len);
    dfb_list_close(r);
    return rc;
}

}  // extern "C"
