"""Host-side mirror of the reference's algorithm-object interface for the hot path.

The reference (C++) creates `cuda::OpticalFlowDual_TVL1::create()` / `cuda::FarnebackOpticalFlow::create()`
(/root/reference/src/denseflow_gpu.cpp:299,301) and calls `alg->calc(gray_a, gray_b, flow, stream)` (:327,:329)
inside `DenseFlow::calc_optflows_imp` (:282-370).  The classes here keep those names, argument meaning and
error behaviour (unknown algorithm / unsupported size -> RuntimeError with the reference's message) on top of
the C ABI (include/denseflow_b200.h).  Everything numeric happens in the CUDA library.
"""
import ctypes as C

import numpy as np

from . import _lib


def _pairs(n, step):
    """M = max(N - |step|, 0): the flows of N frames at `step` (src/denseflow_gpu.cpp:308)"""
    return max(n - abs(step), 0)


def _sizes(new_size, w, h):
    """((dw, dh), (ow, oh)): the resize a call is asked for ((0, 0): none) and the size of its outputs, for w x h frames"""
    return (new_size or (0, 0)), (new_size or (w, h))


def _stream(device, stream=None):
    """The stream a device call is enqueued on: `stream`, or torch's current stream on `device`."""
    import torch
    return C.c_void_p(stream if stream is not None else torch.cuda.current_stream(device).cuda_stream)


def _ptrs(addrs):
    """A pointer array for the C side; an empty one still has one (null) entry."""
    return (C.c_void_p * max(len(addrs), 1))(*addrs)


def _frame_source(frames):
    """Host frames of one size as the frame source of a call: (frames, (their pointer array,), n, width, height)"""
    h, w = frames[0].shape[:2]
    return frames, (_ptrs([f.ctypes.data for f in frames]),), len(frames), w, h


def _check_out(a, shape, dtype, name):
    if not isinstance(a, np.ndarray) or a.dtype != dtype or a.shape[1:] != tuple(shape[1:]) or a.shape[0] < shape[0] \
            or not all(a[i].flags.c_contiguous for i in range(shape[0])):
        raise RuntimeError("%s: expected a C-contiguous %s array of shape %s" % (name, np.dtype(dtype).name, tuple(shape)))


# The outputs of a host batch call: each builder returns the call's output arguments and a collector of its result.
def _field(flows, m, h, w):
    """float32 [M,H,W,2]: `flows`, or a new array"""
    if flows is None:
        flows = np.empty((m, h, w, 2), np.float32)
    _check_out(flows, (m, h, w, 2), np.float32, "flows")
    return (_ptrs([flows[i].ctypes.data for i in range(m)]),), lambda: flows


def _u8_planes(qx, qy, m, h, w):
    """the quantised planes qx, qy, uint8 [M,H,W] each"""
    _check_out(qx, (m, h, w), np.uint8, "qx")
    _check_out(qy, (m, h, w), np.uint8, "qy")
    return tuple(_ptrs([q[i].ctypes.data for i in range(m)]) for q in (qx, qy)), lambda: (qx, qy)


def _float_planes(out, m, h, w):
    """float32 [M,2,H,W], out[j, 0] / out[j, 1] pair j's x / y plane: `out`, or a new array"""
    if out is None:
        out = np.empty((m, 2, h, w), np.float32)
    _check_out(out, (m, 2, h, w), np.float32, "out")
    return tuple(_ptrs([out[i, c].ctypes.data for i in range(m)]) for c in (0, 1)), lambda: out


def _files(k, m, cap, bufs=None):
    """k files for each of m items in host buffers of cap bytes (bufs: k lists of the caller's): the arguments (k pointer
    arrays, cap, k length arrays) and the files' bytes, one per item or a k-tuple per item."""
    if bufs is None:
        bufs = [[np.empty(max(cap, 1), np.uint8) for _ in range(m)] for _ in range(k)]
    lens = [(C.c_size_t * max(m, 1))() for _ in range(k)]

    def collect():
        files = [tuple(b[i][:ln[i]].tobytes() for b, ln in zip(bufs, lens)) for i in range(m)]
        return files if k > 1 else [f for f, in files]
    return (*[_ptrs([b.ctypes.data for b in bb]) for bb in bufs], cap, *lens), collect


class DenseOpticalFlow:
    """cv::cuda::DenseOpticalFlow look-alike bound to one GPU."""

    algorithm = None

    def __init__(self, algorithm, device=0, max_width=1920, max_height=1080, variant="default"):
        self._L = _lib.load(variant)
        self._h = C.c_void_p()
        self.algorithm = algorithm
        self.device = device
        self.max_width, self.max_height = max_width, max_height
        rc = self._L.dfb_create(algorithm.encode(), device, max_width, max_height, C.byref(self._h))
        if rc != _lib.DFB_OK:
            msg = self._L.dfb_last_error(None).decode()
            self._h = None
            raise RuntimeError(msg)  # reference: std::runtime_error -> what() + exit 1 (tools/denseflow.cpp:93-96)

    # -- lifetime (Ptr<>::release, src/denseflow_gpu.cpp:345-355) --
    def release(self):
        if getattr(self, "_h", None):
            self._L.dfb_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def _check(self, rc):
        if rc != _lib.DFB_OK:
            raise RuntimeError(self._L.dfb_last_error(self._h).decode() or "dfb error %d" % rc)

    def set(self, name, value):
        """dfb_set_param: one algorithm parameter or engine knob (include/denseflow_b200.h lists them).  TV-L1 also takes
        "median_filtering" (0 or 1 = off [default], 3 or 5 = the window of a median of the flow between iterations) and
        "median_interval" (>= 1, default 30: the median runs before iterations 0, I, 2I, ... of every warp) and "gamma"
        (finite, >= 0, default 0: OpenCV's setGamma, the weight of an illumination field that absorbs brightness changes
        between the two frames; both schedules take it and give the same bits).  Farneback also takes "gaussian_window"
        (0 [default] or 1: OPTFLOW_FARNEBACK_GAUSSIAN, a 13x13 Gaussian window instead of the box in every iteration) and
        "fast_pyramids" (0 [default] or 1: OpenCV's fastPyramids, level images by a chain of pyrDown).  Both algorithms
        take "use_initial_flow" (0 [default] or 1: OpenCV's useInitialFlow / OPTFLOW_USE_INITIAL_FLOW): with 1, the flow
        buffers of calc, calc_batch, calc_batch_device, calc_batch_planes and calc_batch_device_planes are read as each
        pair's starting flow before they are overwritten, so they must be passed, and every other flow call is refused.  A
        refused value raises RuntimeError("bad parameter <name>") and leaves the parameter as it was.  Returns self."""
        self._check(self._L.dfb_set_param(self._h, name.encode(), float(value)))
        return self

    def get(self, name):
        v = C.c_double()
        self._check(self._L.dfb_get_param(self._h, name.encode(), C.byref(v)))
        return v.value

    def _warm_start_probe(self, flow, call, *nulls, pairs=1):
        """With use_initial_flow set a call reads its flow buffer, so one without (flow None) must fail: call(*nulls), the
        call with null flow arguments, raises the library's refusal.  A call without pairs reads nothing."""
        if flow is None and self.get("use_initial_flow") != 0 and pairs:
            self._check(call(*nulls))

    # -- calc(I0, I1) -> flow (CV_32FC2), src/denseflow_gpu.cpp:327/:329 --
    def calc(self, a, b, flow=None, stream=None):
        """a, b: uint8 [H,W] numpy arrays (host path: upload, calc, download) or CUDA torch tensors
        (device path: enqueued on `stream` / torch's current stream, asynchronous).  With use_initial_flow set, `flow`
        ([H,W,2] float32, C-contiguous host array or CUDA tensor) is also the starting flow."""
        if isinstance(a, np.ndarray):
            a = np.ascontiguousarray(a, np.uint8)
            b = np.ascontiguousarray(b, np.uint8)
            if a.ndim != 2 or a.shape != b.shape:
                raise RuntimeError("calc: frames must be two CV_8UC1 images of the same size")
            h, w = a.shape
            call = lambda f: self._L.dfb_calc_host(self._h, a.ctypes.data, b.ctypes.data, w, h, f)  # noqa: E731
            self._warm_start_probe(flow, call, None)
            if flow is None:
                flow = np.empty((h, w, 2), np.float32)
            self._check(call(flow.ctypes.data))
            return flow
        import torch
        if a.dtype != torch.uint8 or b.dtype != torch.uint8 or a.dim() != 2 or a.shape != b.shape or not a.is_cuda or not b.is_cuda \
                or a.stride(1) != 1 or b.stride(1) != 1:
            raise RuntimeError("calc: frames must be two CV_8UC1 CUDA tensors of the same size with unit column stride")
        h, w = a.shape
        s = _stream(a.device, stream)
        call = lambda f, pitch: self._L.dfb_calc_device(self._h, a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), w, h,  # noqa: E731
                                                        f, pitch, s)
        self._warm_start_probe(flow, call, None, w * 8)
        if flow is None:
            flow = torch.empty((h, w, 2), dtype=torch.float32, device=a.device)
        self._check(call(flow.data_ptr(), flow.stride(0) * 4))
        return flow

    # -- the frame sources of the host batch calls: (keep-alive list, the call's frame arguments, n, width, height) --
    @staticmethod
    def _gray_frames(frames):
        """Every frame must be a CV_8UC1 image of the first frame's size (the C side reads width*height bytes of each)."""
        keep = []
        for i, f in enumerate(frames):
            f = np.asarray(f)
            if f.dtype != np.uint8 or f.ndim != 2 or (keep and f.shape != keep[0].shape):
                raise RuntimeError("frame %d: expected a uint8 [H,W] image of the same size as frame 0" % i)
            keep.append(np.ascontiguousarray(f))
        return _frame_source(keep)

    @staticmethod
    def _bgr_frames(frames_bgr, name):
        frames = [np.asarray(f) for f in frames_bgr]
        if any(f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] != 3 or f.shape != frames[0].shape for f in frames):
            raise RuntimeError("%s: frames must be uint8 [H,W,3] images of one size" % name)
        return _frame_source([np.ascontiguousarray(f) for f in frames])

    def _jpeg_frames(self, jpegs):
        """JPEG files of one size (the call checks it): their size is bounded by the handle's maximum."""
        keep, ptrs, lens = self._jpeg_buffers(jpegs)
        return keep, (ptrs, lens), len(keep), self.max_width, self.max_height

    # -- the batch shape of calc_optflows_imp (src/denseflow_gpu.cpp:307-342) --
    def calc_batch(self, frames, step=1, flows=None, bound=None):
        """frames: sequence of uint8 [H,W] host arrays (or one [N,H,W] array).  Returns M = max(N-|step|,0)
        flows [M,H,W,2] float32, or with bound=B the quantised (qx, qy) uint8 [M,H,W] planes
        (convertFlowToImage, src/common.cpp:4-16, done on the GPU).  With use_initial_flow set, flows[j] is also pair j's
        starting flow."""
        if len(frames) == 0:
            return np.empty((0, 0, 0, 2), np.float32)
        keep, src, n, w, h = self._gray_frames(frames)
        m = _pairs(n, step)
        if bound is not None:
            return self.calc_batch_u8_into(keep, step, bound, np.empty((m, h, w), np.uint8), np.empty((m, h, w), np.uint8))
        call = lambda op: self._L.dfb_calc_batch_host(self._h, *src, n, step, w, h, op)  # noqa: E731
        self._warm_start_probe(flows, call, None, pairs=m)
        out, collect = _field(flows, m, h, w)
        self._check(call(*out))
        return collect()

    def calc_batch_u8_into(self, frames, step, bound, qx, qy):
        """calc_batch(..., bound=B) writing into caller-provided (e.g. pinned) uint8 arrays qx, qy of shape [M,H,W]."""
        keep, src, n, w, h = self._gray_frames(frames)
        out, collect = _u8_planes(qx, qy, _pairs(n, step), h, w)
        self._check(self._L.dfb_calc_batch_host_u8(self._h, *src, n, step, w, h, int(bound), *out))
        return collect()

    def calc_batch_device(self, frames, step=1, flows=None, stream=None):
        """frames: CUDA uint8 tensor [N,H,W] (contiguous); flows: CUDA float32 [M,H,W,2] (contiguous), with use_initial_flow
        set also the pairs' starting flows."""
        import torch
        n, h, w = frames.shape
        s = _stream(frames.device, stream)
        call = lambda f: self._L.dfb_calc_batch_device(self._h, frames.data_ptr(), n, step, w, h, f, s)  # noqa: E731
        self._warm_start_probe(flows, call, None)
        if flows is None:
            flows = torch.empty((_pairs(n, step), h, w, 2), dtype=torch.float32, device=frames.device)
        self._check(call(flows.data_ptr()))
        return flows

    # -- the flow as two float planes per pair: the payloads of -st=h5's flow_x / flow_y datasets --
    def calc_batch_planes(self, frames, step=1, out=None):
        """calc_batch with the flow channels first: float32 [M,2,H,W], out[j,0] / out[j,1] bit for bit flows[j,...,0] /
        flows[j,...,1].  The engines' merge epilogue writes the planes; out may be a caller (e.g. page-locked) array, with
        use_initial_flow set also the pairs' starting flows."""
        if len(frames) == 0:
            return np.empty((0, 2, 0, 0), np.float32)
        keep, src, n, w, h = self._gray_frames(frames)
        m = _pairs(n, step)
        call = lambda xp, yp: self._L.dfb_calc_batch_host_planes(self._h, *src, n, step, w, h, xp, yp)  # noqa: E731
        self._warm_start_probe(out, call, None, None, pairs=m)
        args, collect = _float_planes(out, m, h, w)
        self._check(call(*args))
        return collect()

    def calc_batch_device_planes(self, frames, step=1, planes=None, stream=None):
        """frames: CUDA uint8 tensor [N,H,W] (contiguous); planes: CUDA float32 [M,2,H,W] (contiguous), with use_initial_flow
        set also the pairs' starting flows."""
        import torch
        n, h, w = frames.shape
        m = _pairs(n, step)
        s = _stream(frames.device, stream)
        call = lambda p: self._L.dfb_calc_batch_device_planes(self._h, frames.data_ptr(), n, step, w, h, p, s)  # noqa: E731
        self._warm_start_probe(planes, call, None)
        if planes is None:
            planes = torch.empty((m, 2, h, w), dtype=torch.float32, device=frames.device)
        if planes.dtype != torch.float32 or tuple(planes.shape) != (m, 2, h, w) or not planes.is_contiguous():
            raise RuntimeError("planes: expected a contiguous float32 CUDA tensor of shape %s" % ((m, 2, h, w),))
        self._check(call(planes.data_ptr()))
        return planes

    def process_bgr_batch_planes(self, frames_bgr, step=1, new_size=None):
        """-st=h5 payloads for decoded BGR frames: gray -> resize -> flow -> float32 [M,2,dh,dw], bit for bit calc_batch_planes of
        the gray, resized frames."""
        if len(frames_bgr) == 0:
            return np.empty((0, 2, 0, 0), np.float32)
        keep, src, n, sw, sh = self._bgr_frames(frames_bgr, "process_bgr_batch_planes")
        (dw, dh), (ow, oh) = _sizes(new_size, sw, sh)
        out, collect = _float_planes(None, _pairs(n, step), oh, ow)
        self._check(self._L.dfb_process_bgr_batch_host_planes(self._h, *src, n, step, sw, sh, dw, dh, *out))
        return collect()

    def process_jpeg_batch_planes(self, jpegs, step=1, new_size=None):
        """-if -st=h5 payloads: process_bgr_batch_planes with the frames given as JPEG files of one size, decoded on the GPU to
        imdecode's pixels."""
        keep, (ptrs, lens), n, _, _ = self._jpeg_frames(jpegs)
        m = _pairs(n, step)
        if m == 0:
            return np.empty((0, 2, 0, 0), np.float32)
        w, h = C.c_int(), C.c_int()  # without a resize, the outputs have frame 0's size (the call checks that all have it)
        if not new_size and self._L.dfb_jpeg_info(ptrs[0], lens[0], C.byref(w), C.byref(h)) != _lib.DFB_OK:
            raise RuntimeError(self._L.dfb_last_error(None).decode())
        (dw, dh), (ow, oh) = _sizes(new_size, w.value, h.value)
        out, collect = _float_planes(None, m, oh, ow)
        self._check(self._L.dfb_process_jpeg_batch_host_planes(self._h, ptrs, lens, n, step, dw, dh, *out))
        return collect()

    def quantise_device(self, flow, bound):
        import torch
        h, w = flow.shape[:2]
        qx = torch.empty((h, w), dtype=torch.uint8, device=flow.device)
        qy = torch.empty((h, w), dtype=torch.uint8, device=flow.device)
        self._check(self._L.dfb_quantise_device(self._h, flow.data_ptr(), flow.stride(0) * 4, w, h, int(bound),
                                                qx.data_ptr(), qy.data_ptr(), w, _stream(flow.device)))
        return qx, qy

    # -- convertFlowToPngImage (src/common.cpp:18-46): the CV_8UC3 image `-st=png` encodes --
    def flow_to_png_image_device(self, flow, return_bounds=True):
        """flow: CUDA float32 [H,W,2].  Returns (bgr uint8 [H,W,3] CUDA tensor, (bound_x, bound_y) or None)."""
        import torch
        h, w = flow.shape[:2]
        bgr = torch.empty((h, w, 3), dtype=torch.uint8, device=flow.device)
        b = (C.c_double * 2)()
        self._check(self._L.dfb_flow_to_png_image_device(self._h, flow.data_ptr(), flow.stride(0) * 4, w, h, bgr.data_ptr(), w * 3,
                                                         b if return_bounds else None, _stream(flow.device)))
        return bgr, ((b[0], b[1]) if return_bounds else None)

    # -- frame preparation (cvtColor BGR2GRAY + resize INTER_LINEAR, src/denseflow_gpu.cpp:163-170), bit-exact to OpenCV CPU --
    def bgr_to_gray_device(self, bgr):
        import torch
        h, w = bgr.shape[:2]
        gray = torch.empty((h, w), dtype=torch.uint8, device=bgr.device)
        self._check(self._L.dfb_bgr_to_gray_device(self._h, bgr.data_ptr(), bgr.stride(0), w, h, gray.data_ptr(), w, _stream(bgr.device)))
        return gray

    def resize_gray_device(self, gray, dst_width, dst_height):
        import torch
        h, w = gray.shape
        out = torch.empty((dst_height, dst_width), dtype=torch.uint8, device=gray.device)
        self._check(self._L.dfb_resize_gray_device(self._h, gray.data_ptr(), gray.stride(0), w, h, out.data_ptr(), dst_width,
                                                   dst_width, dst_height, _stream(gray.device)))
        return out

    # -- imencode(".jpg", plane) on the GPU (src/common.cpp:56-57), OpenCV default quality 95 --
    def encode_jpeg_gray_device(self, gray, quality=95):
        h, w = gray.shape
        cap = self._L.dfb_jpeg_max_bytes(w, h)
        buf = np.empty(cap, np.uint8)
        n = C.c_size_t()
        self._check(self._L.dfb_encode_jpeg_gray_device(self._h, gray.data_ptr(), gray.stride(0), w, h, int(quality), buf.ctypes.data,
                                                        cap, C.byref(n), _stream(gray.device)))
        return buf[:n.value].tobytes()

    def encode_jpeg_gray_batch_device(self, planes, quality=95, capacity=None):
        """planes: CUDA uint8 [n, H, W] (rows contiguous; any row and plane stride).  One launch sequence; always the exact
        encoder: returns [bytes of cv2.imencode(".jpg", planes[i], [IMWRITE_JPEG_QUALITY, quality])]."""
        import torch
        n, h, w = planes.shape
        if n == 0:
            return []
        if planes.dtype != torch.uint8 or not planes.is_cuda or planes.stride(2) != 1:
            raise ValueError("planes must be a CUDA uint8 tensor [n, H, W] with contiguous rows")
        cap = int(capacity) if capacity is not None else self._L.dfb_jpeg_max_bytes(w, h)
        out, collect = _files(1, n, cap)
        self._check(self._L.dfb_encode_jpeg_gray_batch_device(self._h, planes.data_ptr(), planes.stride(1), planes.stride(0), n, w, h,
                                                              int(quality), *out, _stream(planes.device)))
        return collect()

    # -- imread(".jpg") + cvtColor(BGR2GRAY) of an `-if` frame folder on the GPU (nvJPEG decode; not bit-identical to libjpeg-turbo) --
    def decode_jpeg_gray_device(self, jpeg_bytes, max_width, max_height, device=None):
        import torch
        dev = device if device is not None else torch.device("cuda", self.device)
        buf = np.frombuffer(jpeg_bytes, np.uint8)
        out = torch.empty((max_height, max_width), dtype=torch.uint8, device=dev)
        w, h = C.c_int(), C.c_int()
        self._check(self._L.dfb_decode_jpeg_gray_device(self._h, buf.ctypes.data, buf.size, out.data_ptr(), max_width, max_width, max_height,
                                                        C.byref(w), C.byref(h), _stream(dev)))
        return out[:h.value, :w.value]

    # -- imread(IMREAD_COLOR) [+ cvtColor(BGR2GRAY)] of `-if` frame folders on the GPU, exactly cv2.imdecode's pixels --
    @staticmethod
    def _jpeg_buffers(jpegs):
        """bytes / uint8 numpy arrays / CPU uint8 torch tensors (e.g. page-locked) -> (keep-alive list, pointers, lengths)"""
        keep, ptrs, lens = [], [], []
        for j in jpegs:
            if isinstance(j, (bytes, bytearray, memoryview)):
                j = np.frombuffer(j, np.uint8)
            if isinstance(j, np.ndarray):
                j = np.ascontiguousarray(j.reshape(-1), np.uint8)
                ptrs.append(j.ctypes.data)
                lens.append(j.size)
            else:  # a CPU torch tensor
                if j.dtype.itemsize != 1 or j.is_cuda or not j.is_contiguous():
                    raise RuntimeError("JPEG buffers must be contiguous uint8 host memory")
                ptrs.append(j.data_ptr())
                lens.append(j.numel())
            keep.append(j)
        return keep, _ptrs(ptrs), (C.c_size_t * max(len(lens), 1))(*lens)

    def decode_jpeg_batch(self, jpegs, channels=3, max_width=None, max_height=None, pitch=None, stream=None, device=None):
        """Decodes JPEG files (bytes, numpy or CPU torch uint8 buffers; sizes and samplings may differ) on the GPU to exactly
        cv2.imdecode(buf, IMREAD_COLOR) (channels 3: uint8 [h,w,3] BGR CUDA tensors) or its cvtColor(BGR2GRAY) (channels 1:
        uint8 [h,w]).  max_width / max_height bound the frames (default: the handle's maximum); pitch: output row pitch in
        bytes (default max_width * channels).  Returns one tensor per file, views into one [n, max_height, pitch] buffer."""
        import torch
        dev = device if device is not None else torch.device("cuda", self.device)
        mw = max_width or self.max_width
        mh = max_height or self.max_height
        pitch = pitch or mw * channels
        keep, ptrs, lens = self._jpeg_buffers(jpegs)
        n = len(keep)
        out = torch.empty((max(n, 1), mh, pitch), dtype=torch.uint8, device=dev)
        ws, hs = (C.c_int * max(n, 1))(), (C.c_int * max(n, 1))()
        self._check(self._L.dfb_decode_jpeg_batch_device(self._h, ptrs, lens, n, int(channels), out.data_ptr(), pitch, mh * pitch, mw, mh,
                                                         ws, hs, _stream(dev, stream)))
        res = []
        for i in range(n):
            v = out[i, :hs[i], :ws[i] * channels]
            res.append(v.unflatten(1, (ws[i], 3)) if channels == 3 else v)
        return res

    def process_jpeg_batch(self, jpegs, step=1, bound=20, new_size=None, quality=95):
        """The `-if` flow batch: process_bgr_batch with the frames given as JPEG files of one size, decoded on the GPU to
        imdecode's pixels.  Returns [(jpg_x bytes, jpg_y bytes)] per pair, byte for byte process_bgr_batch's."""
        keep, src, n, w, h = self._jpeg_frames(jpegs)
        (dw, dh), (ow, oh) = _sizes(new_size, w, h)
        out, collect = _files(2, _pairs(n, step), self._L.dfb_jpeg_max_bytes(ow, oh))
        self._check(self._L.dfb_process_jpeg_batch_host(self._h, *src, n, step, dw, dh, int(bound), int(quality), *out))
        return collect()

    def debug_jpeg_coefficients(self, jpeg):
        """Test hook: (int16 [blocks, 64] quantised coefficients in decode order, natural order, absolute DC; sync rounds)."""
        keep, ptrs, lens = self._jpeg_buffers([jpeg])
        cap = 1 << 20
        while True:
            out = np.empty((cap, 64), np.int16)
            nb, rounds = C.c_int(), C.c_int()
            rc = self._L.dfb_debug_jpeg_coefficients(self._h, ptrs[0], lens[0], out.ctypes.data, cap, C.byref(nb), C.byref(rounds))
            if rc == _lib.DFB_ERR_SIZE and nb.value > cap:
                cap = nb.value
                continue
            self._check(rc)
            return out[:nb.value], rounds.value

    # -- gray -> resize -> flow -> quantise -> JPEG for decoded BGR frames (the reference's chain minus decode / file IO) --
    def process_bgr_batch(self, frames_bgr, step=1, bound=20, new_size=None, quality=95):
        """frames_bgr: list of uint8 [H,W,3]; new_size: (w, h) or None.  Returns [(jpg_x bytes, jpg_y bytes)] per pair."""
        frames = [np.ascontiguousarray(f, np.uint8) for f in frames_bgr]  # any dtype is converted, unlike the other BGR entries
        keep, src, n, sw, sh = self._bgr_frames(frames, "process_bgr_batch")
        (dw, dh), (ow, oh) = _sizes(new_size, sw, sh)
        out, collect = _files(2, _pairs(n, step), self._L.dfb_jpeg_max_bytes(ow, oh))
        self._check(self._L.dfb_process_bgr_batch_host(self._h, *src, n, step, sw, sh, dw, dh, int(bound), int(quality), *out))
        return collect()

    # -- frame-extraction mode (-s=0, extract_frames_video, src/denseflow_gpu.cpp:82-144): resize + imencode(".jpg") per frame --
    @staticmethod
    def _bgr_device(bgr):
        if bgr.dtype.itemsize != 1 or bgr.dim() != 3 or bgr.shape[2] != 3 or not bgr.is_cuda or bgr.stride(2) != 1 or bgr.stride(1) != 3:
            raise RuntimeError("expected a packed uint8 [H,W,3] BGR CUDA tensor (rows may be pitched)")
        return bgr.shape[1], bgr.shape[0]

    def bgr_to_ycc420_device(self, bgr, new_size=None):
        """bgr: uint8 [H,W,3] CUDA tensor; new_size: (w, h) or None.  Returns the planes libjpeg would DCT for
        imencode(".jpg", cv::resize(bgr, new_size)): (y [h,w], cb [ceil(h/2),ceil(w/2)], cr [ceil(h/2),ceil(w/2)])."""
        import torch
        sw, sh = self._bgr_device(bgr)
        dw, dh = new_size if new_size else (sw, sh)
        y = torch.empty((dh, dw), dtype=torch.uint8, device=bgr.device)
        cb = torch.empty(((dh + 1) // 2, (dw + 1) // 2), dtype=torch.uint8, device=bgr.device)
        cr = torch.empty_like(cb)
        self._check(self._L.dfb_bgr_to_ycc420_device(self._h, bgr.data_ptr(), bgr.stride(0), sw, sh, dw, dh, y.data_ptr(), dw,
                                                     cb.data_ptr(), cr.data_ptr(), cb.stride(0), _stream(bgr.device)))
        return y, cb, cr

    def encode_jpeg_bgr_device(self, bgr, new_size=None, quality=95):
        """imencode(".jpg", cv::resize(bgr, new_size)) of a uint8 [H,W,3] BGR CUDA tensor, on the GPU.  Returns the bytes."""
        sw, sh = self._bgr_device(bgr)
        (dw, dh), (ow, oh) = _sizes(new_size, sw, sh)
        cap = self._L.dfb_jpeg_max_bytes_bgr(ow, oh)
        buf = np.empty(cap, np.uint8)
        n = C.c_size_t()
        self._check(self._L.dfb_encode_jpeg_bgr_device(self._h, bgr.data_ptr(), bgr.stride(0), sw, sh, dw, dh, int(quality), buf.ctypes.data,
                                                       cap, C.byref(n), _stream(bgr.device)))
        return buf[:n.value].tobytes()

    def extract_frames(self, frames_bgr, new_size=None, quality=95):
        """frames_bgr: uint8 [H,W,3] host images of one size (pageable or page-locked), or one [N,H,W,3] array.
        Returns one JPEG bitstream per frame, in order (what extract_frames_video writes as img_%05d.jpg)."""
        if len(frames_bgr) == 0:
            return []
        keep, src, n, sw, sh = self._bgr_frames(frames_bgr, "extract_frames")
        (dw, dh), (ow, oh) = _sizes(new_size, sw, sh)
        out, collect = _files(1, n, self._L.dfb_jpeg_max_bytes_bgr(ow, oh))
        self._check(self._L.dfb_extract_frames_host(self._h, *src, n, sw, sh, dw, dh, int(quality), *out))
        return collect()

    # -- -st=png: imencode(".png") on the GPU, byte-identical to OpenCV's default PNG parameters (src/common.cpp:66-71) --
    def encode_png_bgr_device(self, bgr, capacity=None):
        """imencode(".png", bgr) of a uint8 [H,W,3] BGR CUDA tensor (rows may be pitched), on the GPU.  Returns the bytes."""
        w, h = self._bgr_device(bgr)
        cap = self._L.dfb_png_max_bytes(w, h) if capacity is None else int(capacity)
        buf = np.empty(max(cap, 1), np.uint8)
        n = C.c_size_t()
        self._check(self._L.dfb_encode_png_bgr_device(self._h, bgr.data_ptr(), bgr.stride(0), w, h, buf.ctypes.data, cap, C.byref(n),
                                                      _stream(bgr.device)))
        return buf[:n.value].tobytes()

    def process_bgr_batch_png(self, frames_bgr, step=1, new_size=None):
        """-st=png for decoded BGR frames: gray -> resize -> flow -> convertFlowToPngImage -> imencode(".png") on the GPU.
        frames_bgr: list of uint8 [H,W,3]; new_size: (w, h) or None.  Returns one PNG file (bytes) per pair, byte for byte
        calc_batch_png of the gray, resized frames."""
        if len(frames_bgr) == 0:
            return []
        keep, src, n, sw, sh = self._bgr_frames(frames_bgr, "process_bgr_batch_png")
        (dw, dh), (ow, oh) = _sizes(new_size, sw, sh)
        out, collect = _files(1, _pairs(n, step), self._L.dfb_png_max_bytes(ow, oh))
        self._check(self._L.dfb_process_bgr_batch_host_png(self._h, *src, n, step, sw, sh, dw, dh, *out))
        return collect()

    def process_jpeg_batch_png(self, jpegs, step=1, new_size=None):
        """-if -st=png: process_bgr_batch_png with the frames given as JPEG files of one size, decoded on the GPU to imdecode's
        pixels.  Returns one PNG file (bytes) per pair."""
        keep, src, n, w, h = self._jpeg_frames(jpegs)
        (dw, dh), (ow, oh) = _sizes(new_size, w, h)
        out, collect = _files(1, _pairs(n, step), self._L.dfb_png_max_bytes(ow, oh))
        self._check(self._L.dfb_process_jpeg_batch_host_png(self._h, *src, n, step, dw, dh, *out))
        return collect()

    def extract_frames_jpeg(self, jpegs, new_size=None, quality=95):
        """-if -s=0: extract_frames with the frames given as JPEG files of one size, decoded on the GPU to imdecode's pixels.
        Returns one JPEG bitstream per frame, in order (img_%05d.jpg)."""
        keep, src, n, w, h = self._jpeg_frames(jpegs)
        if n == 0:
            return []
        (dw, dh), (ow, oh) = _sizes(new_size, w, h)
        out, collect = _files(1, n, self._L.dfb_jpeg_max_bytes_bgr(ow, oh))
        self._check(self._L.dfb_extract_frames_jpeg_host(self._h, *src, n, dw, dh, int(quality), *out))
        return collect()

    def calc_batch_png(self, frames, step=1, out=None):
        """frames: sequence of uint8 [H,W] host arrays (or one [N,H,W] array).  Returns, for each of the M = max(N-|step|,0)
        pairs, the PNG file writeFlowImagesPng writes: imencode(".png", convertFlowToPngImage(flow)).  out: optional list of
        M uint8 host buffers (e.g. page-locked) of dfb_png_max_bytes(W, H) bytes or more to encode into."""
        if len(frames) == 0:
            return []
        keep, src, n, w, h = self._gray_frames(frames)
        m = _pairs(n, step)
        cap = self._L.dfb_png_max_bytes(w, h)
        if out is not None and (len(out) < m or any(not isinstance(b, np.ndarray) or b.dtype != np.uint8 or b.ndim != 1 or b.size < cap
                                                    or not b.flags.c_contiguous for b in out[:m])):
            raise RuntimeError("out: expected %d C-contiguous uint8 buffers of at least %d bytes" % (m, cap))
        args, collect = _files(1, m, cap, None if out is None else [out[:m]])
        self._check(self._L.dfb_calc_batch_host_png(self._h, *src, n, step, w, h, *args))
        return collect()

    # -- test hook: one stand-alone kernel on host planes --
    def debug_run_kernel(self, kernel, inputs, n_out, scalars=(), out_shape=None, all_scalars=False):
        """returns (output planes, scalars_out[0]), or with all_scalars (output planes, scalars_out[:16]); out_shape: the shape of
        every output, or a list of one shape per output (default: the inputs')"""
        inputs = [np.ascontiguousarray(a, np.float32) for a in inputs]
        h, w = inputs[0].shape
        oshapes = out_shape if isinstance(out_shape, list) else [out_shape or (h, w)] * n_out
        outs = [np.empty(s, np.float32) for s in oshapes]
        ip = (C.c_void_p * len(inputs))(*[a.ctypes.data for a in inputs])
        op = (C.c_void_p * n_out)(*[a.ctypes.data for a in outs])
        sc = (C.c_double * max(len(scalars), 1))(*[float(x) for x in scalars])
        so = (C.c_double * 16)()
        self._check(self._L.dfb_debug_run_kernel(self._h, kernel.encode(), ip, len(inputs), op, n_out, w, h, sc, len(scalars), so))
        return outs, (list(so) if all_scalars else so[0])

    def debug_time_kernel(self, kernel, width, height, sets=6, reps=60):
        """Mean ms per launch of a stand-alone inner-loop kernel on an L2-busting rotation of operand sets."""
        ms = C.c_double()
        self._check(self._L.dfb_debug_time_kernel(self._h, kernel.encode(), width, height, sets, reps, C.byref(ms)))
        return ms.value

    # -- counters for the roofline arithmetic --
    def tvl1_stats(self):
        st = _lib.Tvl1Stats()
        self._check(self._L.dfb_get_tvl1_stats(self._h, C.byref(st)))
        # rows of the C array are indexed s*warps + w
        flat = np.array(st.iters[:], np.int64)
        iters = flat[:st.nscales * st.warps].reshape(st.nscales, st.warps)
        sizes = [(st.level_w[i], st.level_h[i]) for i in range(st.nscales)]
        return iters, sizes

    def tvl1_pair_stats(self, pair_index):
        """Executed inner iterations [nscales, warps] of pair `pair_index` of the most recent calc / batch call."""
        st = _lib.Tvl1Stats()
        self._check(self._L.dfb_get_tvl1_pair_stats(self._h, int(pair_index), C.byref(st)))
        return np.array(st.iters[:], np.int64)[:st.nscales * st.warps].reshape(st.nscales, st.warps)

    def counters(self):
        c = _lib.Counters()
        self._check(self._L.dfb_get_counters(self._h, C.byref(c)))
        return {k: getattr(c, k) for k, _ in c._fields_}

    def phase_ns(self):
        buf = (C.c_uint64 * 32)()
        self._check(self._L.dfb_get_tvl1_phase_ns(self._h, buf))
        v = list(buf)
        return {"level_start": v[0], "warp": v[1], "tiles": v[2], "barrier": v[3], "upsample_merge": v[4],
                "tile_load": v[5], "tile_iter": v[6], "tile_store": v[7],
                "tiles_per_scale": v[8:16], "chunks_per_scale": v[16:24], "median": v[24]}

    def reset_counters(self):
        self._check(self._L.dfb_reset_counters(self._h))


def new_size(width, height, new_width=0, new_height=0, new_short=0, variant="default"):
    """DenseFlow::get_new_size (src/denseflow_gpu.cpp:44-80) with the -nw / -nh / -ns options: the (w, h) a width x height
    video is resized to, or its own size when no resize applies.  Raises RuntimeError with check_param's texts."""
    L = _lib.load(variant)
    dw, dh = C.c_int(), C.c_int()
    if L.dfb_new_size(int(width), int(height), int(new_width), int(new_height), int(new_short), C.byref(dw), C.byref(dh)) != _lib.DFB_OK:
        raise RuntimeError(L.dfb_last_error(None).decode())
    return dw.value, dh.value


def jpeg_info(jpeg, variant="default"):
    """(width, height) of a JPEG file from its markers; raises RuntimeError for files the GPU decoder refuses."""
    L = _lib.load(variant)
    buf = np.frombuffer(jpeg, np.uint8)
    w, h = C.c_int(), C.c_int()
    rc = L.dfb_jpeg_info(buf.ctypes.data if buf.size else None, buf.size, C.byref(w), C.byref(h))
    if rc != _lib.DFB_OK:
        raise RuntimeError(L.dfb_last_error(None).decode())
    return w.value, h.value


class OpticalFlowDual_TVL1(DenseOpticalFlow):
    @classmethod
    def create(cls, device=0, max_width=1920, max_height=1080, variant="default"):
        """cuda::OpticalFlowDual_TVL1::create() with upstream defaults (src/denseflow_gpu.cpp:299)."""
        return cls("tvl1", device, max_width, max_height, variant)


class FarnebackOpticalFlow(DenseOpticalFlow):
    @classmethod
    def create(cls, device=0, max_width=1920, max_height=1080, variant="default"):
        """cuda::FarnebackOpticalFlow::create() with upstream defaults (src/denseflow_gpu.cpp:301)."""
        return cls("farn", device, max_width, max_height, variant)


def create(algorithm, device=0, max_width=1920, max_height=1080, variant="default"):
    """The algorithm switch of calc_optflows_imp (src/denseflow_gpu.cpp:291-304, error text of :296 / :336)."""
    if algorithm == "tvl1":
        return OpticalFlowDual_TVL1.create(device, max_width, max_height, variant)
    if algorithm == "farn":
        return FarnebackOpticalFlow.create(device, max_width, max_height, variant)
    return DenseOpticalFlow(algorithm, device, max_width, max_height, variant)  # raises with the reference's message
