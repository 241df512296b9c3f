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
 * for tests and benchmarks.  tvl1: "tau" and "theta" (finite, > 0), "lambda" (finite, >= 0), "nscales" (1..16), "warps"
 * (1..16), "epsilon" (finite; <= 0 = no convergence checks), "iterations" (>= 1), "scale_step" (> 0 and not above the
 * default 0.8 the workspace is sized for), "median_filtering" (0 [default] or 1 = off; 3 or 5 = u1 and u2 are replaced by
 * their k x k median, replicate borders, before every iteration n of a warp with n % median_interval == 0, so every warp
 * starts with one; an optional extra of CPU DualTVL1's kind that the reference's CUDA TV-L1 does not have) and
 * "median_interval" (>= 1, default 30), "gamma" (finite, >= 0, default 0: OpenCV's setGamma, the weight of an illumination
 * field u3 solved beside the flow so that brightness changes between the frames are not read as motion; u3 starts at 0,
 * is resized between scales without the 1/scale_step factor and is discarded at the end; both schedules take it and give
 * the same bits, every flow call takes it, the list runner never sets it);
 * engine knobs: "fused" (1 = persistent fused primal+dual kernel
 * [default], 0 = one kernel per half-step, the reference's launch structure), "fused_k" (iterations kept on chip per tile
 * visit, 1..8, default 8), "lanes" (pairs solved side by side per launch, 0 = auto [default], up to 64), "use_tma"
 * (1 = TMA staging of the shared-memory tiles [default]), "time_kernels" (CUDA-event timing of the dominant kernel, see
 * dfb_counters).  farn: "num_levels" (0..5)
 * "num_iters" (>= 1) "poly_sigma" (finite, > 0) (winSize 13, polyN 5, pyrScale 0.5 are fixed), "time_kernels".  Every
 * combination of the engine knobs produces bit-identical flows.  Counts take whole numbers only, and on/off knobs 0 or 1.
 * A refused value (NaN, an infinity, a fraction or a value out of range) returns DFB_ERR_INVALID_ARG with "bad parameter
 * <name>" and leaves the parameter unchanged.
 * Both algorithms: "use_initial_flow" (0 [default] or 1; OpenCV's setUseInitialFlow(true) / OPTFLOW_USE_INITIAL_FLOW).  With
 * 1, the calls that take a float flow buffer (dfb_calc_device, dfb_calc_host, dfb_calc_batch_host, dfb_calc_batch_device and
 * the two _planes calls) read each pair's flow buffer as its initial flow before overwriting it.  TV-L1: level 0 of the flow
 * pyramid is that flow, level s the resize of level s - 1 with the frame pyramid's factors, times (float)scale_step, and the
 * coarsest level starts from it instead of 0.  Farneback: the coarsest level starts from the initial flow resized to it
 * (explicit size, CUDA convention) times (float)pyrScale^k instead of 0.  A null flow buffer, and every other flow call
 * (_u8, _png, the dfb_process_* chains), return DFB_ERR_INVALID_ARG with a message naming use_initial_flow before anything
 * is enqueued; the handle stays usable.  The list runner opens its own handles and never reads an initial flow.
 * farn: "gaussian_window" (0 [default] or 1; OpenCV's OPTFLOW_FARNEBACK_GAUSSIAN): every iteration averages M over a 13x13
 * Gaussian window (getGaussianKernel(13, 6 * 0.3f), replicate borders, vertical pass first) instead of the 13x13 box.
 * farn: "fast_pyramids" (0 [default] or 1; OpenCV's fastPyramids): level 0 is the unblurred frame and level k the pyrDown
 * (BORDER_REFLECT_101) of level k - 1, size ((w + 1) / 2, (h + 1) / 2), instead of B.1's blur and resize; the level count
 * is unchanged.  Both compose with each other, with use_initial_flow and with every accepted num_levels / num_iters /
 * poly_sigma, and every Farneback flow call takes them; the list runner never sets them.  A frame's pyramid lives only
 * within the call that prepares it, so a change applies from the next call on.
 * Both algorithms: "jpeg_exact" (0 [default] = JPEG files through nvJPEG; 1 = every JPEG this handle writes is exactly the
 * file cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, quality]) writes with OpenCV's other defaults, libjpeg-turbo 3.x:
 * baseline, standard Huffman tables, islow DCT, gray or YCbCr 4:2:0, no restart markers).  It covers
 * dfb_encode_jpeg_gray_device, dfb_encode_jpeg_bgr_device, dfb_process_bgr_batch_host, dfb_process_jpeg_batch_host and
 * dfb_extract_frames_host, dfb_extract_frames_jpeg_host and dfb_list_run_videos; the two settings give different bytes and
 * the same flows.  The exact encoder is the project's
 * own CUDA and never loads libnvjpeg.  Any other value is DFB_ERR_INVALID_ARG.
 */
int dfb_set_param(dfb_handle *h, const char *name, double value);
int dfb_get_param(const dfb_handle *h, const char *name, double *value);

/*
 * Compute, device buffers.  Replaces  alg->calc(gray_a, gray_b, flow_gpu, stream)  src/denseflow_gpu.cpp:327 / :329.
 *   a, b      : CV_8UC1 frames in device memory, row pitch in bytes (GpuMat pitch)
 *   flow_xy   : CV_32FC2 (u, v interleaved) in device memory, row pitch in bytes; u = x displacement
 *   stream    : cudaStream_t the work is enqueued on (the reference's DenseFlow::stream, include/dense_flow.h:33)
 * Asynchronous w.r.t. the host apart from the convergence read-back of the non-fused engine.
 * use_initial_flow = 1: flow_xy also holds the initial flow, read on `stream` before the result overwrites it.
 */
int dfb_calc_device(dfb_handle *h, const uint8_t *a, size_t a_pitch, const uint8_t *b, size_t b_pitch, int width,
                    int height, float *flow_xy, size_t flow_pitch, void *stream);

/*
 * Compute, host buffers: upload a and b, calc, download the flow — the three statements
 * src/denseflow_gpu.cpp:317-318, :327/:329, :339 as one call.  Buffers are dense (pitch = width) and may be
 * pageable; the engine stages through its own pinned ring.  Blocks until flow_xy is complete.
 * use_initial_flow = 1: flow_xy also holds the initial flow, uploaded through the same staging.
 */
int dfb_calc_host(dfb_handle *h, const uint8_t *a, const uint8_t *b, int width, int height, float *flow_xy);

/*
 * The shape calc_optflows_imp really has (src/denseflow_gpu.cpp:307-342): N gray frames, step s,
 * M = max(N - |s|, 0) flows with pair (a, b) = (i, i+s) for s > 0 and (i-s, i) for s < 0 (:315-316).
 * Each frame is uploaded and pyramided once (the reference does both twice), and copies overlap compute.
 *   frames[n_frames] : host pointers, dense width*height uint8
 *   flows[M]         : host pointers, dense width*height*2 float (CV_32FC2); with use_initial_flow = 1 flows[j] also holds
 *                      pair j's initial flow
 */
int dfb_calc_batch_host(dfb_handle *h, const uint8_t *const *frames, int n_frames, int step, int width, int height,
                        float *const *flows);

/*
 * Same batch, but the flow is bounded + quantised on the device and only the two uint8 planes come
 * back (SURVEY §8 f1): fuses convertFlowToImage (src/common.cpp:4-16, via encodeFlowMap :48-64 with
 * lowerBound = -bound, higherBound = +bound) into the epilogue.  Bit-exact to the CAST macro.
 *   qx[M], qy[M] : host pointers, dense width*height uint8
 * Refused while use_initial_flow = 1 (no float flow buffer to read it from).
 */
int dfb_calc_batch_host_u8(dfb_handle *h, const uint8_t *const *frames, int n_frames, int step, int width, int height,
                           int bound, uint8_t *const *qx, uint8_t *const *qy);

/* Device-resident batch: frames is one device allocation [n_frames][height][width] uint8 (dense),
 * flows one device allocation [M][height][width][2] float.  Enqueued on `stream`.  With use_initial_flow = 1 pair j's
 * field in flows also holds its initial flow. */
int dfb_calc_batch_device(dfb_handle *h, const uint8_t *frames, int n_frames, int step, int width, int height,
                          float *flows, void *stream);

/*
 * The same batches with the flow as two float planes per pair, the payloads of the flow_x / flow_y datasets the reference's
 * USE_HDF5 build writes (cv::split then H5LTmake_dataset_float, src/denseflow_gpu.cpp:223-239): the engines' merge epilogue
 * writes u1 and u2 as dense planes, so the values are bit for bit the x and y channels of dfb_calc_batch_host's fields.
 *   fx[M], fy[M] : host pointers, dense width*height float each (page-locked ones take a direct DMA)
 *   planes       : one device allocation [M][2][height][width] float (pair j's x plane, then its y plane); enqueued on `stream`
 * With use_initial_flow = 1 the two planes of pair j also hold its initial flow.
 */
int dfb_calc_batch_host_planes(dfb_handle *h, const uint8_t *const *frames, int n_frames, int step, int width, int height,
                               float *const *fx, float *const *fy);
int dfb_calc_batch_device_planes(dfb_handle *h, const uint8_t *frames, int n_frames, int step, int width, int height,
                                 float *planes, void *stream);

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
 * -st=h5 takes the flow unquantised: dfb_calc_batch_host_planes and the _planes chains below give its payloads, and
 * dfb_h5_create / dfb_h5_write_float / dfb_h5_close write the file (a build without DFB_USE_HDF5 refuses with the reference's
 * "HDF5 support is not enabled, pls recompile", :241).
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
 * (dfb_jpeg_max_bytes(width, height) holds i.i.d. noise at quality 100; a larger file fails cleanly with the needed
 * length in the message); *out_len receives the length.  Blocks until the bitstream is on the host.  With the handle's
 * "jpeg_exact" = 0 [default] nvJPEG encodes, not byte-identical to libjpeg-turbo; with 1 the file is imencode(".jpg")'s bytes.
 * Only the width x height plane is read: nvJPEG encodes a copy in handle scratch whose partial 8 x 8 blocks are padded
 * as libjpeg pads them (last column and row repeated), so the file depends on the plane alone.
 */
size_t dfb_jpeg_max_bytes(int width, int height);
int dfb_encode_jpeg_gray_device(dfb_handle *h, const uint8_t *gray, size_t gray_pitch, int width, int height, int quality,
                                uint8_t *out, size_t out_capacity, size_t *out_len, void *stream);
/*
 * n device planes of one size in one launch sequence, always with the exact encoder: file i is the bytes of
 * cv2.imencode(".jpg", plane_i, [IMWRITE_JPEG_QUALITY, quality]).  Plane i starts at planes + i * plane_stride, rows pitch
 * bytes apart (any alignment); out[i] are host buffers of `capacity` bytes each, len[i] receives file i's length.  The work
 * is enqueued on `stream` and the call blocks until the files are on the host; n == 0 is a no-op.  A file that does not
 * fit fails the call with the length it needs in the message ("jpeg output buffer too small: plane i (N > capacity)").
 */
int dfb_encode_jpeg_gray_batch_device(dfb_handle *h, const uint8_t *planes, size_t pitch, size_t plane_stride, int n,
                                      int width, int height, int quality, uint8_t *const *out, size_t capacity,
                                      size_t *len, void *stream);

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
 * ---- imdecode-exact JPEG decode of `-if` frame folders --------------------------------------------------------------
 * The decode stage reads each frame with imread(path, IMREAD_COLOR) and converts it with cvtColor(BGR2GRAY)
 * (src/denseflow_gpu.cpp:154-163).  These calls decode JPEG files on the GPU to EXACTLY the pixels of
 * cv2.imdecode(buf, IMREAD_COLOR) with libjpeg-turbo's default decompression as OpenCV sets it up (islow integer IDCT, fancy
 * upsampling, YCbCr -> BGR table arithmetic).  Integer-only: both builds give the same bytes.  Only the compressed bytes
 * cross PCIe; the host parses the markers, everything after (de-stuffing, entropy decode, IDCT, upsampling, colour) runs on
 * the device.  They work on either kind of handle.
 *
 * Accepted: baseline or extended sequential Huffman (SOF0 / SOF1), 8-bit samples, one scan holding every component;
 * 1 component, or 3 that libjpeg treats as YCbCr (JFIF marker, Adobe transform 1, or component ids 1-2-3); chroma sampled
 * 1x1 with luma h, v in {1, 2} (4:4:4, 4:2:2, 4:4:0, 4:2:0); 8- or 16-bit DQT tables; DRI / RST0-7; APPn and COM
 * segments are skipped.  DFB_ERR_UNSUPPORTED, with a message naming the feature, for progressive, arithmetic-coded,
 * lossless or 12-bit files, multi-scan files, other samplings (4:1:1, ...), RGB-coded or CMYK files and an EXIF
 * orientation other than 1 (imread would rotate the image).  DFB_ERR_INVALID_ARG, naming the frame, for a damaged header
 * and for corrupt data: an invalid Huffman code, data that ends before the last MCU, a wrong RST sequence or count (libjpeg
 * warns and makes up pixels there; these calls refuse instead), a scan not ended by a marker, and a dequantised
 * coefficient past 2048 or an IDCT output past -512..511 (no 8-bit encoder writes the first; past either, imdecode's
 * pixels depend on how libjpeg-turbo was built).  Progressive files still decode, approximately, through
 * dfb_decode_jpeg_gray_device.
 *
 * dfb_decode_jpeg_batch_device: n files (host buffers jpeg[i] of len[i] bytes; sizes and samplings may differ).
 * channels 3: imdecode(IMREAD_COLOR), packed BGR; channels 1: cvtColor(BGR2GRAY) of it (the frame the flow sees).  Frame i
 * goes to out + i * frame_stride (device memory, rows `pitch` bytes apart); width[i] / height[i] (optional arrays of n)
 * receive the sizes.  A frame larger than max_width x max_height or its pitch / stride: DFB_ERR_SIZE.  Enqueued on
 * `stream`; blocks until the device has reported every frame's status.  n == 0 is a no-op.
 */
int dfb_decode_jpeg_batch_device(dfb_handle *h, const uint8_t *const *jpeg, const size_t *len, int n, int channels, uint8_t *out,
                                 size_t pitch, size_t frame_stride, int max_width, int max_height, int *width, int *height, void *stream);
/*
 * The `-if` flow batch: dfb_process_bgr_batch_host with the frames given as JPEG files (every frame one size, else
 * DFB_ERR_SIZE naming the frame).  The outputs are byte for byte those of dfb_process_bgr_batch_host on the imdecoded
 * frames; the decode runs in groups of frames on the chain's input stream.
 */
int dfb_process_jpeg_batch_host(dfb_handle *h, const uint8_t *const *jpeg, const size_t *len, int n_frames, int step, int dst_width,
                                int dst_height, int bound, int jpeg_quality, uint8_t *const *jpg_x, uint8_t *const *jpg_y, size_t capacity,
                                size_t *len_x, size_t *len_y);
/*
 * Test hook: the entropy decode alone.  out (host, capacity_blocks x 64 int16) receives the quantised coefficients of every
 * block in decode (MCU) order, natural order, absolute DC; *n_blocks the block count; *sync_rounds (optional) how many
 * re-decode rounds the subsequence states took to converge.
 */
int dfb_debug_jpeg_coefficients(dfb_handle *h, const uint8_t *jpeg, size_t len, int16_t *out, size_t capacity_blocks, int *n_blocks,
                                int *sync_rounds);

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
 * Refused while use_initial_flow = 1, as are the other dfb_process_* chains.
 */
int dfb_process_bgr_batch_host(dfb_handle *h, const uint8_t *const *bgr, int n_frames, int step, int src_width, int src_height,
                               int dst_width, int dst_height, int bound, int jpeg_quality, uint8_t *const *jpg_x,
                               uint8_t *const *jpg_y, size_t capacity, size_t *len_x, size_t *len_y);

/*
 * ---- frame-extraction mode (`-s=0`, the reference CLI's default) ------------------------------------------------------
 * DenseFlow::extract_frames_video (src/denseflow_gpu.cpp:82-144) resizes each decoded colour frame with
 * cv::resize(frame, size) [INTER_LINEAR, CV_8UC3] (:146-177), encodes it with imencode(".jpg") [OpenCV defaults: quality
 * 95, libjpeg YCbCr 4:2:0] and writes img_%05d.jpg (src/common.cpp:73-82).  These calls do the resize and the encode on the
 * GPU and work on either kind of handle; the destination must fit the handle's max_width x max_height (DFB_ERR_SIZE),
 * dst 0 / 0 means no resize, and quality is 1..100.
 *
 * dfb_bgr_to_ycc420_device: the colour preparation alone, on device buffers.  bgr: packed 8-bit BGR (src_width x
 * src_height, row pitch in bytes).  Writes y (dst_width x dst_height) and cb, cr (ceil(dst_width / 2) x ceil(dst_height / 2),
 * sharing c_pitch): the resize is bit-exact to OpenCV's CPU fixed-point arithmetic per channel, the colour conversion is
 * libjpeg's rgb_ycc_convert and the 2 x 2 chroma downsampling libjpeg's h2v2_downsample with its alternating 1 / 2 bias and
 * last-column / last-row replication at odd sizes — exactly the samples libjpeg hands to its forward DCT.  Asynchronous.
 */
int dfb_bgr_to_ycc420_device(dfb_handle *h, const uint8_t *bgr, size_t bgr_pitch, int src_width, int src_height, int dst_width,
                             int dst_height, uint8_t *y, size_t y_pitch, uint8_t *cb, uint8_t *cr, size_t c_pitch, void *stream);
/*
 * Capacity for one colour JPEG of width x height: 2 bytes per sample of the image padded to 16 x 16 MCUs (1.5 samples per
 * pixel) + 4096.  It holds for i.i.d. noise at quality 100; content built to defeat the Huffman tables can exceed it, and a
 * bitstream larger than the capacity passed to the calls below fails cleanly with the needed length in the message.
 */
size_t dfb_jpeg_max_bytes_bgr(int width, int height);
/*
 * One frame: resize + imencode(".jpg", frame) of a BGR frame in device memory.  Baseline, standard Huffman tables, YCbCr
 * 4:2:0; out is a host buffer of out_capacity bytes, *out_len receives the length.  The work is enqueued on `stream` and
 * the call blocks until the bitstream is on the host.  With "jpeg_exact" = 0 [default] nvJPEG encodes, not byte-identical
 * to libjpeg; with 1 the file is imencode(".jpg", resized frame)'s bytes.  nvJPEG reads whole 16 x 16 MCUs of handle
 * scratch, padded as libjpeg pads them (luma: last column and row repeated; chroma columns downsampled from the repeated
 * last column, chroma rows repeating the last one), so only the DCT and the luma blocks wholly past the image (libjpeg's
 * DC-only dummy blocks) differ, and the file depends on the frame alone.  The same holds for every nvJPEG file of
 * dfb_extract_frames_host / dfb_extract_frames_jpeg_host, and for the flow chains' gray planes (8 x 8 blocks).
 */
int dfb_encode_jpeg_bgr_device(dfb_handle *h, const uint8_t *bgr, size_t bgr_pitch, int src_width, int src_height, int dst_width,
                               int dst_height, int quality, uint8_t *out, size_t out_capacity, size_t *out_len, void *stream);
/*
 * The batch of extract_frames_video: bgr[n_frames] host pointers (pageable or pinned) to dense packed BGR frames of
 * src_width x src_height.  Frame i's bitstream goes to jpg[i] (host buffers of `capacity` bytes each,
 * dfb_jpeg_max_bytes_bgr(dst) is the documented size) and its length to len[i], in order, for the host to write as
 * img_%05d.jpg.  Uploads, colour preparation, encodes and bitstream read-back of successive groups of frames overlap; the host
 * synchronises once per group.  Gives the bytes dfb_encode_jpeg_bgr_device gives frame by frame.  Blocks until every
 * bitstream is on the host; n_frames == 0 is a no-op.
 */
int dfb_extract_frames_host(dfb_handle *h, const uint8_t *const *bgr, int n_frames, int src_width, int src_height, int dst_width,
                            int dst_height, int quality, uint8_t *const *jpg, size_t capacity, size_t *len);

/*
 * ---- PNG flow images (-st=png) ---------------------------------------------------------------------------------------
 * encodeFlowMapPng (src/common.cpp:66-71) writes imencode(".png", img) of the packed image convertFlowToPngImage builds.
 * These calls run that encode on the GPU and return EXACTLY the bytes of cv2.imencode(".png", img) with OpenCV's default
 * PNG parameters: filter SUB on every row (NONE when the width is 1), zlib level 1 (Z_BEST_SPEED) with strategy Z_RLE, the
 * window libpng declares for the data size, and IDAT chunks of 8192 bytes of zlib stream.  An OpenCV built with other
 * defaults, or a caller that passes IMWRITE_PNG_* parameters, gets other (equally valid) bytes.  Integer-only: both builds
 * give the same bytes.  They work on either kind of handle; the image must fit the handle's max_width x max_height.
 *
 * dfb_png_max_bytes: an upper bound on the file size of a width x height image (every deflate block stored, plus the zlib
 * and PNG framing).  A pure function; needs no device.
 */
size_t dfb_png_max_bytes(int width, int height);
/*
 * imencode(".png", img) of one packed 8-bit BGR image in device memory (rows bgr_pitch bytes apart).  out: host buffer of
 * out_capacity bytes, *out_len receives the length.  Enqueued on `stream`; blocks until the file is on the host.  A file
 * larger than out_capacity fails with the needed length in the message and writes nothing.
 */
int dfb_encode_png_bgr_device(dfb_handle *h, const uint8_t *bgr, size_t bgr_pitch, int width, int height, uint8_t *out,
                              size_t out_capacity, size_t *out_len, void *stream);
/*
 * The -st=png branch of encode_save (src/denseflow_gpu.cpp:442-453) over host frames: for each of the M = max(n_frames -
 * |step|, 0) pairs, selected as dfb_calc_batch_host selects them, flow -> convertFlowToPngImage -> imencode(".png").
 * png[j] (host buffers of `capacity` bytes each, dfb_png_max_bytes is always enough) receives exactly what
 * writeFlowImagesPng writes for pair j, len[j] its length.  Flow and packing, the encodes and the read-back of successive
 * groups of pairs overlap; the host synchronises once per group.  Blocks until every file is on the host.
 * Refused while use_initial_flow = 1, as are all the dfb_process_* chains.
 */
int dfb_calc_batch_host_png(dfb_handle *h, const uint8_t *const *frames, int n_frames, int step, int width, int height,
                            uint8_t *const *png, size_t capacity, size_t *len);
/*
 * The -st=png branch behind the two colour frame sources: dfb_process_bgr_batch_host / dfb_process_jpeg_batch_host with
 * flow -> convertFlowToPngImage -> imencode(".png") per pair instead of the two quantised JPEGs.  Pair j's file goes to png[j]
 * (host buffers of `capacity` bytes each, dfb_png_max_bytes(dst) is always enough), its length to len[j]: byte for byte what
 * dfb_calc_batch_host_png gives for the gray, resized frames.  Arguments and refusals are those of the JPEG siblings.
 */
int dfb_process_bgr_batch_host_png(dfb_handle *h, const uint8_t *const *bgr, int n_frames, int step, int src_width, int src_height,
                                   int dst_width, int dst_height, uint8_t *const *png, size_t capacity, size_t *len);
int dfb_process_jpeg_batch_host_png(dfb_handle *h, const uint8_t *const *jpeg, const size_t *jpeg_len, int n_frames, int step,
                                    int dst_width, int dst_height, uint8_t *const *png, size_t capacity, size_t *len);
/*
 * The -st=h5 payloads behind the two colour frame sources: the _png chains with pair j's flow as two dense float planes
 * (dst_width x dst_height each) to fx[j] / fy[j] instead of a PNG file: bit for bit what dfb_calc_batch_host_planes gives for the
 * gray, resized frames.  Arguments and refusals are those of the _png siblings.
 */
int dfb_process_bgr_batch_host_planes(dfb_handle *h, const uint8_t *const *bgr, int n_frames, int step, int src_width, int src_height,
                                      int dst_width, int dst_height, float *const *fx, float *const *fy);
int dfb_process_jpeg_batch_host_planes(dfb_handle *h, const uint8_t *const *jpeg, const size_t *jpeg_len, int n_frames, int step,
                                       int dst_width, int dst_height, float *const *fx, float *const *fy);

/*
 * ---- HDF5 flow files (-st=h5; pure host functions, no device needed) ----------------------------------------------------
 * What the reference's USE_HDF5 build calls (src/utils.cpp:27-41, src/common.cpp:120-150), written by a self-contained
 * writer: dfb_h5_create is H5Fcreate(path, H5F_ACC_TRUNC), dfb_h5_write_float is H5LTmake_dataset_float(file, name, 2,
 * {rows, cols}, data) at the root group (a name already written is refused), dfb_h5_close writes the metadata and closes.
 * The file is the format libhdf5 writes by default (superblock 0, a symbol-table root group, contiguous IEEE f32 LE
 * datasets); payloads go to the file as they arrive, and the same calls give the same bytes (no timestamps).  Only a library
 * built with DFB_USE_HDF5 (build variant "hdf5") has the writer: elsewhere dfb_h5_create fails with DFB_ERR_UNSUPPORTED and
 * "HDF5 support is not enabled, pls recompile" (src/denseflow_gpu.cpp:241) in dfb_last_error(NULL).  Errors go to
 * dfb_last_error(NULL).  dfb_h5_close always frees the file object, and returns the first error of the file's writes.
 */
typedef struct dfb_h5_file dfb_h5_file;
int dfb_h5_create(const char *path, dfb_h5_file **out);
int dfb_h5_write_float(dfb_h5_file *f, const char *name, int rows, int cols, const float *data);
int dfb_h5_close(dfb_h5_file *f);
/*
 * `-if -s=0`: dfb_extract_frames_host with the frames given as JPEG files of one size (else DFB_ERR_SIZE naming the frame),
 * decoded on the device to imdecode's BGR pixels.  Frame i's file goes to jpg[i], its length to len[i]: byte for byte what
 * dfb_extract_frames_host gives for the imdecoded frames.  Refuses what dfb_process_jpeg_batch_host refuses in a file.
 */
int dfb_extract_frames_jpeg_host(dfb_handle *h, const uint8_t *const *jpeg, const size_t *jpeg_len, int n_frames, int dst_width,
                                 int dst_height, int quality, uint8_t *const *jpg, size_t capacity, size_t *len);

/*
 * ---- size rule and JPEG geometry (pure host functions; no device needed) -----------------------------------------------
 * dfb_new_size: DenseFlow::get_new_size (src/denseflow_gpu.cpp:44-80) for a w x h source and the -nw / -nh / -ns options:
 * *dw / *dh receive the destination size, which is the source size when no resize applies (-ns resizes only when
 * min(w, h) > new_short).  Refuses what check_param (:27-35) refuses, with its texts in dfb_last_error(NULL):
 * "height and width cannot < 0!" and "do not set height and width when set short!" (DFB_ERR_INVALID_ARG).
 * dfb_jpeg_info: the frame size of a JPEG file from its markers, so a caller can size a video before decoding it.  Fails as
 * the imdecode-exact decoder's header parse fails (DFB_ERR_UNSUPPORTED for progressive files, ...; DFB_ERR_INVALID_ARG for
 * corrupt headers), with the message in dfb_last_error(NULL).
 */
int dfb_new_size(int width, int height, int new_width, int new_height, int new_short, int *dw, int *dh);
int dfb_jpeg_info(const uint8_t *jpeg, size_t len, int *width, int *height);

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
 *   "farn_level_image"     in {frame (u8 values as floats)}  out {level image, level k size}; scalars {k} (B.1 / B.2's blur
 *     and resize whatever fast_pyramids says)
 *   "farn_pyr_down"        in {image}                        out {its pyrDown, (w + 1) / 2 x (h + 1) / 2} (fast_pyramids' level step)
 *   "farn_poly_exp"        in {level image}                  out {R0 .. R4}
 *   "farn_flow_init"       in {fx, fy of the coarser level}  out {fx, fy (scalars[0] x scalars[1])}; scalars {level w, level h}
 *   "farn_initial_flow"    in {x, y of the initial flow}     out {fx, fy of the coarsest level}; scalars {step, pitch, pairs}
 *     (use_initial_flow's level start: the start resized to the coarsest level of the handle's num_levels, times
 *     pyrScale^k; step 2 uploads the start as a float2 field, step 1 as two planes, rows `pitch` floats apart, 0 = dense)
 *   "farn_update_matrices" in {fx, fy, R0 x 5 (frame a), R1 x 5 (frame b)}  out {M0 .. M4}; scalars {pairs}
 *   "farn_iteration"       in {M x 5, R0 x 5, R1 x 5}        out {fx, fy, M'0 .. M'4}; scalars {rebuild, pairs}
 *     (one box mean -> 2x2 solve -> rebuild of M iteration, the Gaussian window instead of the box mean with
 *     gaussian_window = 1; M' is written only with rebuild = 1)
 *   The two pair stages run `pairs` (1..8, default 1) pairs in one launch: every plane then stacks the pairs' planes along
 *   its rows (height = pairs x the pair's height).
 * On a "tvl1" handle, single phases of the fused pair kernel, run by one cooperative launch of its own device code on the
 * engine's lanes, tensor maps and level geometry.  The last scalar is `lanes` (1..16, default 1 when fewer scalars than the
 * stage lists are given; scalars between the listed ones and the last are not read): every plane stacks one plane per lane
 * along its rows, and lane i runs on its own CTAs and workspace.  G (CTAs per lane) 0 means as many as fit.
 *   "tvl1_level_start" in {I1, u1, u2}                     out {I1x, I1y, p11, p12, p21, p22, u1, u2}; scalars {coarsest, lanes}
 *   "tvl1_warp"        in {I0, I1, I1x, I1y, u1, u2}       out {I1wx, I1wy, q, rho_c}; scalars {lanes}
 *   "tvl1_gq"          in {grad}                           out {q}; scalars {lanes}
 *     (q: the gradient plane as the inner loop reads it: grad in the strict build, -rcp(grad) or -1e30 in the default build)
 *   "tvl1_chunks"      in {I1wx, I1wy, grad, rho_c, u1, u2, p11, p12, p21, p22}  out {u1, u2, p11, p12, p21, p22};
 *                      scalars {kk, n, check, G, use_tma, lanes}; n chunks of kk iterations with the
 *                      handle's tau / lambda / theta; check: every chunk sums the convergence error, scalars_out[i] = lane i's
 *                      error of the last chunk (scalars_out must then hold `lanes` doubles)
 *   "tvl1_upsample"    in {u1, u2}                         out {u1, u2 (scalars[0] x scalars[1])}; scalars {dst w, dst h, lanes}
 *                      (resize to the finer level, times 1 / scale_step)
 *   "tvl1_merge"       in {u1, u2}                         out {flow x, flow y} (bound 0) or {qx, qy} as floats; scalars {bound, lanes}
 *   "tvl1_median"      in {u1, u2}                         out {u1, u2} (their k x k median); scalars {k (3 or 5), lanes}
 *   "tvl1_initial_flow" in {x, y of the initial flows}     out {u1, u2: every level, one after the other}; scalars {step,
 *                      pitch, lanes}; use_initial_flow's start pyramid (the batched copy into each lane's level 0, then the
 *                      resize x scale_step per level) at the handle's nscales / scale_step, on 1..64 lanes, with the start
 *                      uploaded as a float2 field (step 2) or two planes (step 1), rows `pitch` floats apart (0 = dense);
 *                      each level of an output holds the lanes' planes of that level stacked along the rows
 *   "jpeg_padded_gray" in {gray}                           out {the plane padded to round8(w) x round8(h)}
 *   "jpeg_padded_ycc420" in {B, G, R}                      out {Y round16(dw) x round16(dh), Cb, Cr round8(ceil(dw / 2)) x
 *                      round8(ceil(dh / 2))}; scalars {dst w, dst h} (0 / 0: no resize)
 *     (the planes the nvJPEG path (jpeg_exact = 0) hands the encoder, with libjpeg's edge padding; inputs hold uint8 values)
 *   "png_encode_batch" in {B, G, R}                        out {files: n rows of dfb_png_max_bytes(w, h / n)}; scalars {n}
 *                      (n = 1..16 images of h / n rows, stacked along the rows, encoded by one call of the batch PNG
 *                      encoder that -st=png uses; scalars_out[i] = file i's length, its bytes as floats in row i)
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
 * [3] grid barriers (includes waiting for slower CTAs) [4] upsample + merge, [24] median filtering, [8+s] tile iterations at
 * scale s, [16+s] tile visits (chunks) at scale s, for s = 0..7 only (the tile iterations of scales 8..15 count in [2] alone).
 * Zeros for other engines.  (The reference has only the
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
 * The buffers belong to the worker and are reused after the callback returns.  A failure ends the run with the first failed
 * video's code and message: the other workers finish the video they hold, every chunk and last_chunk included, and take no
 * new one.  The stats of a failed call count what was delivered: clips, flows and frames those of the videos whose last chunk
 * was delivered, flows_per_worker the flows of every delivered chunk.
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

/*
 * ---- the list over videos as the reference takes them: colour frames or `-if` JPEG folders in, files out ------------------
 * `denseflow list.txt -a=.. -s=S [-if] [-st=jpg|png] [-nw/-nh/-ns]` per video: decode -> get_new_size -> gray / resize -> flow
 * -> the files writeFlowImages / writeFlowImagesPng write, or with S = 0 extract_frames_video's img files.  Each worker
 * resolves a video's destination size with dfb_new_size and runs the matching single-handle chain:
 *   save_type DFB_SAVE_JPG  dfb_process_{bgr,jpeg}_batch_host        files 2 i / 2 i + 1: flow first_index + i's x / y
 *   save_type DFB_SAVE_PNG  dfb_process_{bgr,jpeg}_batch_host_png    file i: flow first_index + i
 *   save_type DFB_SAVE_H5   dfb_process_{bgr,jpeg}_batch_host_planes files 2 i / 2 i + 1: flow first_index + i's x / y plane as
 *                           raw little-endian float32, 4 * dw * dh bytes each (the payloads of writeHDF5's datasets; bound > 0
 *                           is still required, as check_param requires it, and unused)
 *   step 0                  dfb_extract_frames_host / dfb_extract_frames_jpeg_host   file i: frame first_index + i (img)
 * Chunks, queue and stats are those of dfb_list_run (stats: frames = decoded frames, flows = flow fields); max_width /
 * max_height of dfb_list_open bound the DESTINATION size.  jpeg_exact is set on every worker handle for the call and restored.
 * `done` runs on the worker's thread once every file of the chunk is in host memory; last_chunk (FlowBuffer::last_buffer) is 1
 * exactly once per video, after all its files (a video without outputs gets one call with n = 0).  The files live in the
 * worker's pinned ring and are reused after the callback returns.  bound <= 0 with a flow step is refused ("bound should >
 * 0!"); step 0 ignores bound.  A refused or corrupt JPEG fails the call with "video k: frame f: ..." (f: index in the video);
 * the runner stays usable.
 */
enum { DFB_VIDEO_BGR = 0, DFB_VIDEO_JPEG = 1 };
enum { DFB_SAVE_JPG = 0, DFB_SAVE_PNG = 1, DFB_SAVE_H5 = 2 };
typedef struct {
    int kind;                       /* DFB_VIDEO_BGR or DFB_VIDEO_JPEG */
    int n_frames;
    const uint8_t *const *bgr;      /* BGR: n_frames host pointers to dense packed BGR frames of width x height */
    int width, height;
    const uint8_t *const *jpeg;     /* JPEG: n_frames host pointers to the files' bytes, jpeg_len[i] bytes each */
    const size_t *jpeg_len;
} dfb_video;
typedef void (*dfb_files_done_fn)(void *user, int video, int device, int first_index, int n, int last_chunk, const uint8_t *const *files,
                                  const size_t *lens);
int dfb_list_run_videos(dfb_list_runner *r, const dfb_video *videos, int n_videos, int step, int bound, int save_type, int quality,
                        int jpeg_exact, int new_width, int new_height, int new_short, int chunk_flows, dfb_queue *queue,
                        dfb_files_done_fn done, void *user, dfb_list_stats *stats, char *err, size_t err_len);

/*
 * ---- the same list with frames pulled from the caller, one window at a time -------------------------------------------
 * dfb_list_run_stream is dfb_list_run_videos for videos the caller decodes while the list runs (a 10-minute 1080p video is
 * ~110 GB of BGR frames): only n_videos is known up front.  The worker that takes video k calls
 *   source(user, k, first, max_n, out, msg, msg_len)
 * for frames first .. first + max_n - 1 and runs them through the same chains.  The source fills *out (kind, n_frames, bgr +
 * width / height, or jpeg + jpeg_len); n_frames < max_n means the video ends there.  The pointers stay valid until that
 * window's `done` call returns, or until the call returns after a failure.  A nonzero return fails the run with "video k: <msg>".
 *   - max_n is at most chunk_flows + |step| (chunk_flows with step 0); consecutive windows overlap by |step| frames, the
 *     overlap the reference keeps between its batches.  The calls for one video come in order from the worker that owns it.
 *   - The video's size comes from its first window (BGR width / height, or dfb_jpeg_info of JPEG 0); a later frame of another
 *     size fails the run with "video k: frame f: ...".
 *   - A worker whose handle is smaller than a video's destination size replaces it with a large enough one (keeping the call's
 *     jpeg_exact), so max_width / max_height of dfb_list_open are only a starting size here.
 *   - For the same frames, the files and `done` calls equal dfb_list_run_videos', except that a video whose outputs end on a
 *     window boundary gets one more `done` call with n = 0 and last_chunk = 1.  last_chunk still comes once per video, after
 *     all its files.
 *   - A source error, or a refused or corrupt JPEG, ends the run; the runner stays usable.
 */
typedef int (*dfb_frames_fn)(void *user, int video, int first, int max_n, dfb_video *out, char *msg, size_t msg_len);
int dfb_list_run_stream(dfb_list_runner *r, int n_videos, dfb_frames_fn source, int step, int bound, int save_type, int quality,
                        int jpeg_exact, int new_width, int new_height, int new_short, int chunk_flows, dfb_queue *queue,
                        dfb_files_done_fn done, void *user, dfb_list_stats *stats, char *err, size_t err_len);

/*
 * ---- the same windows shared among the workers: one video on every GPU -------------------------------------------------
 * dfb_list_run_windows takes dfb_list_run_stream's arguments and writes the same files, but a video's windows, not the video,
 * are the unit of work once the queue is empty, so a single video (or the tail of a list) runs on every worker, and one worker
 * reads a video's next window while another computes the current one.
 *   - Windows: the sequence dfb_list_run_stream asks for (max_n = chunk_flows + |step|, chunk_flows at step 0; consecutive
 *     windows overlap by |step|; a short window ends the video).  The source calls for one video come in frame order and never
 *     overlap in time, but may come from different workers' threads.
 *   - Lifetime: dfb_list_run_stream's; what the source returns for a window stays valid until that window's `done` call
 *     returns, or until the call returns after a failure.
 *   - Delivery: the `done` calls for one video come in first_index order, each after the previous one has returned, on the
 *     thread of the worker that computed the window, with that worker's device.  last_chunk comes once per video, in its last
 *     call; the n = 0 trailing call follows dfb_list_run_stream's rule.  The files and every other argument equal
 *     dfb_list_run_stream's for the same source.
 *   - Scheduling: while the queue (the in-process counter or `queue`) holds videos, a worker runs the video it took and then
 *     takes the next one, in dfb_list_run_stream's order.  Once the queue is empty, an idle worker joins the earliest
 *     unfinished video whose reader is free (no source call in progress, final window not read yet), reads its next window and
 *     computes it; if no reader is free it waits until one is, and stops once no window is left to read.  A worker holds at
 *     most one window, so at most n_workers windows are alive.
 *   - Geometry: the video's first window sizes it; a worker that joins fits its handle to the video before it computes.  The
 *     frame-size checks are dfb_list_run_stream's.
 *   - Failures: the error reported for a video is the one a one-worker run reports: its earliest failed window's (source,
 *     size, decode or handle).  Windows before it are computed and delivered; it and every later window of the video get no
 *     `done` call.  Workers take no new windows, a window whose read completes after the failure is dropped, and the call
 *     returns once every worker has stopped.  The runner stays usable.
 *   - Stats: clips, flows and frames are dfb_list_run_stream's; flows_per_worker counts the flows each worker computed and
 *     clips_per_worker the videos whose last window it delivered.
 * Sharing one video among processes is not done: a dfb_queue still hands out whole videos.
 */
int dfb_list_run_windows(dfb_list_runner *r, int n_videos, dfb_frames_fn source, int step, int bound, int save_type, int quality,
                         int jpeg_exact, int new_width, int new_height, int new_short, int chunk_flows, dfb_queue *queue,
                         dfb_files_done_fn done, void *user, dfb_list_stats *stats, char *err, size_t err_len);

#ifdef __cplusplus
}
#endif
#endif /* DENSEFLOW_B200_H */
