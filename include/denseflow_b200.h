/*
 * denseflow_b200.h — C ABI of the H100-native (sm_90a) dense optical-flow engine.
 *
 * This is the drop-in boundary for the one hot path of open-mmlab/denseflow: the body of the
 * per-pair loop in DenseFlow::calc_optflows_imp (/root/reference/src/denseflow_gpu.cpp:313-342).
 * The reference has no FFI layer; what it binds there is the OpenCV algorithm-object interface.
 * Each entry point below names the reference call it replaces.
 *
 * Conventions: plain pointers and sizes, no C++/torch types; every function returns an int status
 * (0 = DFB_OK, negative = error) and never throws; dfb_last_error() gives the message the C++ host
 * rethrows as std::runtime_error (reference behaviour: message + exit 1, tools/denseflow.cpp:93-96).
 * A handle is single-threaded (reference: one thread calls create/calc/release,
 * include/dense_flow.h:78); handles on different threads/devices are independent.  Every call
 * selects the handle's device itself.  A handle owns ONE set of workspace (pyramid slots, lanes): successive calls that
 * take a stream must be stream-ordered with respect to each other (same stream, or the caller's events between them).
 */
#ifndef DENSEFLOW_B200_H
#define DENSEFLOW_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dfb_handle dfb_handle;

enum {
    DFB_OK = 0,
    DFB_ERR_INVALID_ARG = -1,
    DFB_ERR_UNKNOWN_ALGORITHM = -2, /* reference: std::runtime_error("unknown optical algorithm ...") src/denseflow_gpu.cpp:336 */
    DFB_ERR_CUDA = -3,              /* a CUDA call failed; the message carries the runtime's text and, when the tvl1 kernel's grid-barrier
                                       watchdog fired, "[k_tvl1_pair grid-barrier watchdog: CTA .. lane ..]".  The context is unusable after it */
    DFB_ERR_SIZE = -4,              /* frame larger than max_width x max_height given at create, or a/b mismatch */
    DFB_ERR_UNSUPPORTED = -5,       /* "nv" / "brox": outside this build (reference: "not enabled, pls recompile" :296) */
    DFB_ERR_NO_DEVICE = -6
};

/* Library / device probes (no reference equivalent; setDevice(0) is hard-wired at src/denseflow_gpu.cpp:482). */
const char *dfb_version(void);
int dfb_device_count(void);

/*
 * Factory.  Replaces  cuda::OpticalFlowDual_TVL1::create()   src/denseflow_gpu.cpp:299   (algorithm = "tvl1")
 *           and       cuda::FarnebackOpticalFlow::create()    src/denseflow_gpu.cpp:301   (algorithm = "farn")
 * with the argument-less upstream defaults (tvl1: tau .25, lambda .15, theta .3, nscales 5, warps 5,
 * epsilon .01, iterations 300, scaleStep .8; farn: numLevels 5, pyrScale .5, winSize 13, numIters 10,
 * polyN 5, polySigma 1.1, flags 0).  All device workspace for frames up to max_width x max_height is
 * allocated here, once (the reference re-creates the algorithm object per <=512-frame batch, :299-301,:349-352).
 */
int dfb_create(const char *algorithm, int device, int max_width, int max_height, dfb_handle **out);

/* Replaces alg.release()  src/denseflow_gpu.cpp:345-355. */
void dfb_destroy(dfb_handle *h);

/* Message of the last failing call on this handle (or of the last failing dfb_create when h == NULL). */
const char *dfb_last_error(const dfb_handle *h);

/*
 * Algorithm hyper-parameters.  The reference never sets any (always create() defaults); these exist
 * for tests and benchmarks.  tvl1: "tau" "lambda" "theta" "nscales" "warps" "epsilon" "iterations" "scale_step" (must not
 * exceed the default 0.8 the workspace is sized for); engine knobs: "fused" (1 = persistent fused primal+dual kernel
 * [default], 0 = one kernel per half-step, the reference's launch structure), "fused_k" (iterations kept on chip per tile
 * visit, default 8), "lanes" (pairs solved side by side per launch, 0 = auto [default], up to 64), "flag_sync" (1 =
 * neighbour-warp progress flags in the tile loop [default], 0 = CTA-wide barriers), "use_tma" (1 = TMA staging of the
 * shared-memory tiles [default]), "prefetch" (1 = L2 prefetch of a CTA's next tile during the iterations [default]),
 * "serial_launches" (1 = the fused launches of all handles on one device run strictly one after another; 0 [default] = a
 * second handle's launch fills the SMs the first one's finished lanes free), "time_kernels" (CUDA-event timing of the dominant kernel, see dfb_counters).  farn: "num_levels" "num_iters" "poly_sigma"
 * (winSize 13, polyN 5, pyrScale 0.5 are fixed), "use_tma" (1 = persistent TMA-staged iteration kernel [default], 0 = the
 * LDG-staged one), "time_kernels".  Every combination of the engine knobs produces bit-identical flows.
 */
int dfb_set_param(dfb_handle *h, const char *name, double value);
int dfb_get_param(const dfb_handle *h, const char *name, double *value);

/*
 * Compute, device buffers.  Replaces  alg->calc(gray_a, gray_b, flow_gpu, stream)  src/denseflow_gpu.cpp:327 / :329.
 *   a, b      : CV_8UC1 frames in device memory, row pitch in bytes (GpuMat pitch)
 *   flow_xy   : CV_32FC2 (u, v interleaved) in device memory, row pitch in bytes; u = x displacement
 *   stream    : cudaStream_t the work is enqueued on (the reference's DenseFlow::stream, include/dense_flow.h:33)
 * Asynchronous w.r.t. the host apart from the convergence read-back of the non-fused engine.
 */
int dfb_calc_device(dfb_handle *h, const uint8_t *a, size_t a_pitch, const uint8_t *b, size_t b_pitch, int width,
                    int height, float *flow_xy, size_t flow_pitch, void *stream);

/*
 * Compute, host buffers: upload a and b, calc, download the flow — the three statements
 * src/denseflow_gpu.cpp:317-318, :327/:329, :339 as one call.  Buffers are dense (pitch = width) and may be
 * pageable; the engine stages through its own pinned ring.  Blocks until flow_xy is complete.
 */
int dfb_calc_host(dfb_handle *h, const uint8_t *a, const uint8_t *b, int width, int height, float *flow_xy);

/*
 * The shape calc_optflows_imp really has (src/denseflow_gpu.cpp:307-342): N gray frames, step s,
 * M = max(N - |s|, 0) flows with pair (a, b) = (i, i+s) for s > 0 and (i-s, i) for s < 0 (:315-316).
 * Each frame is uploaded and pyramided once (the reference does both twice), and copies overlap compute.
 *   frames[n_frames] : host pointers, dense width*height uint8
 *   flows[M]         : host pointers, dense width*height*2 float (CV_32FC2)
 */
int dfb_calc_batch_host(dfb_handle *h, const uint8_t *const *frames, int n_frames, int step, int width, int height,
                        float *const *flows);

/*
 * Same batch, but the flow is bounded + quantised on the device and only the two uint8 planes come
 * back (SURVEY §8 f1): fuses convertFlowToImage (src/common.cpp:4-16, via encodeFlowMap :48-64 with
 * lowerBound = -bound, higherBound = +bound) into the epilogue.  Bit-exact to the CAST macro.
 *   qx[M], qy[M] : host pointers, dense width*height uint8
 */
int dfb_calc_batch_host_u8(dfb_handle *h, const uint8_t *const *frames, int n_frames, int step, int width, int height,
                           int bound, uint8_t *const *qx, uint8_t *const *qy);

/* Device-resident batch: frames is one device allocation [n_frames][height][width] uint8 (dense),
 * flows one device allocation [M][height][width][2] float.  Enqueued on `stream`. */
int dfb_calc_batch_device(dfb_handle *h, const uint8_t *frames, int n_frames, int step, int width, int height,
                          float *flows, void *stream);

/* Stand-alone quantiser on device buffers (src/common.cpp:4-16).  flow_xy pitch in bytes. */
int dfb_quantise_device(dfb_handle *h, const float *flow_xy, size_t flow_pitch, int width, int height, int bound,
                        uint8_t *qx, uint8_t *qy, size_t q_pitch, void *stream);

/*
 * The packed-PNG flow format on device buffers (SURVEY §8 f4).  Replaces convertFlowToPngImage (src/common.cpp:18-46), the
 * arithmetic behind `-st=png` (encodeFlowMapPng :66-71 then imencode(".png")s the result on the host): per-component
 * minMaxLoc, bound = min(1020, ceil(min(extent, max|v|) * 128/127 / 4) * 4) (+4 when divisible by 8), x and y as
 * convertTo(CV_8U, 128/bound, 128) [one float fused multiply-add, round-half-even, saturate — OpenCV's vector path], and a
 * third channel holding bound_x/4 in rows 0..h/2 and bound_y/4 below.  bgr: packed 3 bytes per pixel (x, y, bounds).
 * bounds_xy_host (optional, 2 doubles): receives bound_x, bound_y — passing it makes the call block on the stream.
 * -st=h5 stays what it is in a build without HDF5: "HDF5 support is not enabled, pls recompile" (:241) — a host writer.
 */
int dfb_flow_to_png_image_device(dfb_handle *h, const float *flow_xy, size_t flow_pitch, int width, int height, uint8_t *bgr,
                                  size_t bgr_pitch, double *bounds_xy_host, void *stream);

/*
 * Frame preparation on device buffers (SURVEY §8 f3) — what the reference's decode stage does on the CPU to every
 * frame before the hot path: cvtColor(frame, gray, COLOR_BGR2GRAY) src/denseflow_gpu.cpp:163 and
 * cv::resize(gray, gray, new_size) [INTER_LINEAR] :166-170.  Both are bit-exact to OpenCV's CPU fixed-point
 * arithmetic (the flow is computed on these pixels).  Pitches in bytes; bgr is packed 3 bytes per pixel.
 */
int dfb_bgr_to_gray_device(dfb_handle *h, const uint8_t *bgr, size_t bgr_pitch, int width, int height, uint8_t *gray,
                           size_t gray_pitch, void *stream);
int dfb_resize_gray_device(dfb_handle *h, const uint8_t *src, size_t src_pitch, int src_width, int src_height, uint8_t *dst,
                           size_t dst_pitch, int dst_width, int dst_height, void *stream);

/*
 * JPEG-encode one uint8 plane that lives in device memory (SURVEY §8 f2).  Replaces
 * imencode(".jpg", flow_img_x, encoded_x) / (..., flow_img_y, ...)  src/common.cpp:56-57 with OpenCV's defaults when
 * quality = 95 (baseline sequential, one gray component).  out is a host buffer of out_capacity bytes
 * (dfb_jpeg_max_bytes(width, height) is always enough); *out_len receives the length.  Blocks until
 * the bitstream is on the host.  Not byte-identical to libjpeg-turbo (lossy; the reference pins no bytes).
 */
size_t dfb_jpeg_max_bytes(int width, int height);
int dfb_encode_jpeg_gray_device(dfb_handle *h, const uint8_t *gray, size_t gray_pitch, int width, int height, int quality,
                                uint8_t *out, size_t out_capacity, size_t *out_len, void *stream);

/*
 * Decode one JPEG frame of an `-if` frame folder on the GPU (SURVEY §8 f3 remainder): replaces imread(path) [IMREAD_COLOR]
 * + cvtColor(BGR2GRAY) of the decode stage (src/denseflow_gpu.cpp:154-163) for JPEG inputs.  jpeg: the file's bytes in host
 * memory; gray: device buffer of at least max_width x max_height (row pitch in bytes); *width / *height receive the frame size.
 * nvJPEG decodes to BGR; the gray conversion is the bit-exact kernel of dfb_bgr_to_gray_device.  nvJPEG's IDCT and chroma
 * upsampling are NOT bit-identical to libjpeg-turbo's (the decoder behind imread): gray frames differ by a level or two
 * on a few percent of the pixels, which moves the flow by ~1e-2 px AEE at most on the synthetic clips (DESIGN.md) — use it
 * when throughput matters more than bit-reproducing the reference's decode.  Video files (VideoCapture, :118-151) stay on the host.
 */
int dfb_decode_jpeg_gray_device(dfb_handle *h, const uint8_t *jpeg, size_t jpeg_len, uint8_t *gray, size_t gray_pitch, int max_width,
                                int max_height, int *width, int *height, void *stream);

/*
 * Work counters of the most recent calc on this handle (for the roofline arithmetic, SURVEY §8(d)):
 *   iters[nscales*warps] executed inner iterations per (scale, warp), index s*warps + w, s = 0 finest
 *   level_w/level_h[nscales] pyramid sizes
 * dfb_get_counters: cumulative since create / last reset.
 */
typedef struct {
    int nscales, warps;
    int level_w[16], level_h[16];
    int iters[16 * 16];
} dfb_tvl1_stats;
int dfb_get_tvl1_stats(dfb_handle *h, dfb_tvl1_stats *out);
/* The same log for pair `pair_index` (0-based, in output order) of the most recent calc / batch call on this handle;
 * the engine keeps the last 256 pairs of a call.  Lets a test compare the executed schedule of every pair of a batch
 * with the oracle's. */
int dfb_get_tvl1_pair_stats(dfb_handle *h, int pair_index, dfb_tvl1_stats *out);

/*
 * The reference's per-batch chain minus decode and file IO, on the GPU, for decoded BGR frames:
 *   cvtColor(BGR2GRAY) src/denseflow_gpu.cpp:163 -> resize :166-170 -> flow :313-342 ->
 *   convertFlowToImage + imencode(".jpg") x2  src/common.cpp:48-64 (what writeFlowImages then writes, :84-100).
 * bgr[n_frames]: host pointers to packed 8-bit BGR frames (src_width x src_height, dense rows).  dst_width/dst_height:
 * the size get_new_size chose (src/denseflow_gpu.cpp:44-80), or 0/0 for no resize.  For each of the
 * M = max(n_frames - |step|, 0) pairs the two JPEG bitstreams are written to jpg_x[i] / jpg_y[i] (host buffers of
 * `capacity` bytes each, dfb_jpeg_max_bytes(dst) is enough) and their lengths to len_x[i] / len_y[i].
 */
int dfb_process_bgr_batch_host(dfb_handle *h, const uint8_t *const *bgr, int n_frames, int step, int src_width, int src_height,
                               int dst_width, int dst_height, int bound, int jpeg_quality, uint8_t *const *jpg_x,
                               uint8_t *const *jpg_y, size_t capacity, size_t *len_x, size_t *len_y);

/*
 * Test hook: run ONE stand-alone TV-L1 kernel on dense host planes (w*h floats each, uploaded into the engine's pitched
 * layout, downloaded after the launch) so each kernel can be checked against the oracle's building block:
 *   "gradient"      in {I}                                   out {Ix, Iy}
 *   "warp"          in {I0, I1, I1x, I1y, u1, u2}            out {I1wx, I1wy, grad, rho_c}
 *   "estimate_u"    in {I1wx,I1wy,grad,rho_c,p11,p12,p21,p22,u1,u2}  out {u1, u2}; scalars {l_t, theta, calc_error}; scalars_out[0] = sum(diff)
 *   "estimate_dual" in {u1,u2,p11,p12,p21,p22}               out {p11,p12,p21,p22}; scalars {taut}
 *   "resize"        in {src (w x h)}                         out {dst (scalars[0] x scalars[1])}; scalars {dw, dh, fx, fy, post_mul}
 * On a "farn" handle, single Farneback stages, launched by the engine's own launch code on its frame slots and lanes (w, h
 * at most the handle's maximum frame size):
 *   "farn_level_image"     in {frame (u8 values as floats)}  out {level image, level k size}; scalars {k}
 *   "farn_poly_exp"        in {level image}                  out {R0 .. R4}
 *   "farn_flow_init"       in {fx, fy of the coarser level}  out {fx, fy (scalars[0] x scalars[1])}; scalars {level w, level h}
 *   "farn_update_matrices" in {fx, fy, R0 x 5 (frame a), R1 x 5 (frame b)}  out {M0 .. M4}; scalars {pairs}
 *   "farn_iteration"       in {M x 5, R0 x 5, R1 x 5}        out {fx, fy, M'0 .. M'4}; scalars {use_tma, rebuild, pairs}
 *     (one box mean -> 2x2 solve -> rebuild of M iteration; M' is written only with rebuild = 1)
 *   The two pair stages run `pairs` (1..8, default 1) pairs in one launch: every plane then stacks the pairs' planes along
 *   its rows (height = pairs x the pair's height).
 * Not part of the reference's surface.
 */
int dfb_debug_run_kernel(dfb_handle *h, const char *kernel, const float *const *in, int n_in, float *const *out, int n_out,
                         int width, int height, const double *scalars, int n_scalars, double *scalars_out);

/*
 * Benchmark hook for the two stand-alone inner-loop kernels of the unfused schedule (the launches the reference makes
 * ~7 500 times per pair): "estimate_u" (48 B/px) or "estimate_dual" (40 B/px) at width x height.  `sets` independent
 * copies of the operand planes are rotated between launches so the working set exceeds the L2 (sets * 83 MB at 1080p);
 * `reps` launches are timed with CUDA events after 3 warm-up launches.  *ms_per_launch receives the mean.
 */
int dfb_debug_time_kernel(dfb_handle *h, const char *kernel, int width, int height, int sets, int reps, double *ms_per_launch);

typedef struct {
    uint64_t pairs;          /* flow fields computed */
    uint64_t kernel_launches; /* CUDA kernels launched by this handle */
    uint64_t pixel_iters;    /* sum over executed inner iterations of level pixels (tvl1) */
    uint64_t h2d_bytes, d2h_bytes;
    /* dominant-kernel timing, CUDA events on the launching stream around every launch of the fused tvl1
     * pair kernel (enabled with dfb_set_param(h, "time_kernels", 1)): */
    uint64_t timed_kernel_launches;
    uint64_t timed_kernel_ns;
    uint64_t timed_kernel_pairs;
    uint64_t pixel_chunks;   /* fused tvl1: sum over tile visits of level pixels (each visit moves 64 B/px and runs up to k iterations) */
} dfb_counters;
int dfb_get_counters(dfb_handle *h, dfb_counters *out);

/*
 * Where the most recent fused-tvl1 pair's device time went, in ns, as seen by CTA 0 of the persistent
 * kernel (%globaltimer): [0] level start (gradients, zeroing) [1] warps [2] tile iterations
 * [3] grid barriers (includes waiting for slower CTAs) [4] upsample + merge, [8+s] tile iterations at
 * scale s, [16+s] tile visits (chunks) at scale s.  Zeros for other engines.  (The reference has only the
 * wall-clock summary line, src/denseflow_gpu.cpp:492-496.)
 */
int dfb_get_tvl1_phase_ns(dfb_handle *h, uint64_t out[32]);
int dfb_reset_counters(dfb_handle *h);

/*
 * ---- video-list dispatch over several GPUs (SURVEY §8 e; BASELINE.json configs[4]) --------------------------------
 * The reference builds the list of videos from list.txt (tools/denseflow.cpp:54-81) and walks it on GPU 0
 * (src/denseflow_gpu.cpp:482-489); a video is marked done only after its last FlowBuffer has been written (:456-470).
 * dfb_run_list drains the same kind of list with n_workers host threads (worker i owns an engine handle on
 * devices[i]; a device may appear twice so one worker's copies overlap the other's compute) from ONE dynamic work
 * queue — no static i mod G assignment, no data-path collective, unit of work = one video.
 *   queue == NULL : in-process atomic counter (one process, one thread per GPU — the reference's process model)
 *   queue != NULL : a counter in POSIX shared memory shared by several processes (one process per GPU, e.g. torchrun):
 *                   every process passes the SAME clip list and its own device; each index is handed out exactly once.
 * Each video is solved in chunks of at most chunk_flows flows (0 = 64), frames overlapping by |step| between chunks as
 * the reference's own batches do (:182-189), and reported through `done` on the worker's thread once every output of
 * the chunk is in host memory:
 *   first_flow      global index of the chunk's first flow inside the video (FlowBuffer::base_start)
 *   last_chunk      1 for the final chunk of the video (FlowBuffer::last_buffer): the only point at which the host may
 *                   create the video's .done marker
 *   qx/qy           bound > 0: the convertFlowToImage planes (width*height uint8 each), flows == NULL
 *   flows           bound == 0: CV_32FC2 fields, qx == qy == NULL
 * The buffers belong to the worker and are reused after the callback returns.
 */
typedef struct dfb_queue dfb_queue;
int dfb_queue_open(const char *name, int create, dfb_queue **out); /* name: "/something" (shm_open); create = 1 also zeroes it */
long dfb_queue_next(dfb_queue *q);                                  /* atomic fetch-and-increment */
void dfb_queue_reset(dfb_queue *q);
void dfb_queue_close(dfb_queue *q, int unlink_name);

typedef struct {
    const uint8_t *const *frames; /* n_frames host pointers to dense width*height gray frames (pinned or pageable) */
    int n_frames, width, height;
} dfb_clip;
typedef void (*dfb_chunk_done_fn)(void *user, int clip_index, int device, int first_flow, int n_flows, int last_chunk,
                                  uint8_t *const *qx, uint8_t *const *qy, float *const *flows);
#define DFB_LIST_MAX_WORKERS 32
typedef struct {
    uint64_t clips, flows, frames; /* processed by THIS call (this process) */
    double seconds;                /* wall time of the call */
    int workers;
    uint64_t clips_per_worker[DFB_LIST_MAX_WORKERS], flows_per_worker[DFB_LIST_MAX_WORKERS];
    double busy_seconds_per_worker[DFB_LIST_MAX_WORKERS];   /* time spent inside clips */
    double finish_seconds_per_worker[DFB_LIST_MAX_WORKERS]; /* when the worker ran out of work (tail imbalance) */
    uint64_t kernel_launches, h2d_bytes, d2h_bytes;         /* summed over the workers' engine handles */
} dfb_list_stats;
int dfb_run_list(const char *algorithm, const int *devices, int n_workers, const dfb_clip *clips, int n_clips, int step, int bound,
                 int chunk_flows, dfb_queue *queue, dfb_chunk_done_fn done, void *user, dfb_list_stats *stats, char *err, size_t err_len);
/* The same with the workers (engine handles, pinned output rings) kept alive between lists: dfb_run_list is
 * dfb_list_open + dfb_list_run + dfb_list_close.  err/err_len: optional buffer for the failure message. */
typedef struct dfb_list_runner dfb_list_runner;
int dfb_list_open(const char *algorithm, const int *devices, int n_workers, int max_width, int max_height, dfb_list_runner **out, char *err,
                  size_t err_len);
int dfb_list_run(dfb_list_runner *r, const dfb_clip *clips, int n_clips, int step, int bound, int chunk_flows, dfb_queue *queue,
                 dfb_chunk_done_fn done, void *user, dfb_list_stats *stats, char *err, size_t err_len);
void dfb_list_close(dfb_list_runner *r);

#ifdef __cplusplus
}
#endif
#endif /* DENSEFLOW_B200_H */
