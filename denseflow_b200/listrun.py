"""Video-list dispatch (SURVEY §8 e, BASELINE.json configs[4]): host-side mirror of dfb_run_list / dfb_queue_*.

The reference reads list.txt into a vector of videos (/root/reference/tools/denseflow.cpp:54-81), walks it on one GPU and marks
each video done after its last buffer is written (src/denseflow_gpu.cpp:456-470).  `run_list` hands the same kind of list to W
workers (one engine handle per entry of `devices`) that pull videos from one dynamic queue; with `queue=WorkQueue(name)` the
queue lives in POSIX shared memory and is shared by several processes (one process per GPU).
"""
import ctypes as C

import numpy as np

from . import _lib


class WorkQueue:
    """Cross-process fetch-and-increment counter (dfb_queue_*)."""

    def __init__(self, name, create, variant="default"):
        self._L = _lib.load(variant)
        self._q = C.c_void_p()
        self.name = name
        self.owner = bool(create)
        if self._L.dfb_queue_open(name.encode(), int(bool(create)), C.byref(self._q)) != _lib.DFB_OK:
            raise RuntimeError("cannot open work queue %s" % name)

    def next(self):
        return self._L.dfb_queue_next(self._q)

    def reset(self):
        self._L.dfb_queue_reset(self._q)

    def close(self):
        if self._q:
            self._L.dfb_queue_close(self._q, int(self.owner))
            self._q = C.c_void_p()


def _pack_clips(clips):
    keep = []
    arr = (_lib.Clip * max(len(clips), 1))()
    for i, frames in enumerate(clips):
        fr = []
        for f in frames:
            f = np.asarray(f)
            if f.dtype != np.uint8 or f.ndim != 2 or not f.flags.c_contiguous or (fr and f.shape != fr[0].shape):
                raise RuntimeError("clip %d: frames must be C-contiguous uint8 [H,W] images of one size" % i)
            fr.append(f)
        ptrs = (C.c_void_p * max(len(fr), 1))(*[f.ctypes.data for f in fr])
        keep.append((fr, ptrs))
        arr[i].frames = ptrs
        arr[i].n_frames = len(fr)
        arr[i].height, arr[i].width = (fr[0].shape if fr else (1, 1))
    shapes = [(arr[i].height, arr[i].width) for i in range(len(clips))]
    return arr, shapes, keep


def _pack_video(frames):
    """One video as a dfb_video, and what keeps its memory alive (the structure holds its pointer tables)."""
    v = _lib.Video()
    v.n_frames = len(frames)
    if frames and isinstance(frames[0], (bytes, bytearray, memoryview)):
        bufs = [np.frombuffer(f, np.uint8) for f in frames]
        v.kind = _lib.VIDEO_JPEG
        v.jpeg = (C.c_void_p * len(bufs))(*[b.ctypes.data for b in bufs])
        v.jpeg_len = (C.c_size_t * len(bufs))(*[b.size for b in bufs])
        return v, (v, bufs)
    fr = [np.ascontiguousarray(f) for f in frames]
    if any(f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] != 3 or f.shape != fr[0].shape for f in fr):
        raise RuntimeError("frames must be uint8 [H,W,3] BGR images of one size, or JPEG files (bytes)")
    v.kind = _lib.VIDEO_BGR
    v.bgr = (C.c_void_p * max(len(fr), 1))(*[f.ctypes.data for f in fr])
    v.height, v.width = fr[0].shape[:2] if fr else (1, 1)
    return v, (v, fr)


def _pack_videos(videos):
    keep = []
    arr = (_lib.Video * max(len(videos), 1))()
    for i, frames in enumerate(videos):
        try:
            v, k = _pack_video(frames)
        except RuntimeError as ex:
            raise RuntimeError("video %d: %s" % (i, ex)) from None
        arr[i] = v
        keep.append(k)
    return arr, keep


def output_names(step, first_index, n, save_type="jpg"):
    """The file names the reference gives a chunk's files (src/common.cpp:73-118), in the order run_videos hands them out:
    writeFlowImages (flow_x_%05d.jpg / flow_y_%05d.jpg per flow), writeFlowImagesPng (flow_%05d.png) and, with step 0,
    writeImages (img_%05d.jpg).  Steps > 1 add _p<step>, steps < 0 add _m<|step|> and offset the index by |step|."""
    if step == 0:
        return ["img_%05d.jpg" % (first_index + i) for i in range(n)]
    base = -step if step < 0 else 0
    tag = "_p%d" % step if step > 1 else "_m%d" % -step if step < 0 else ""
    names = []
    for i in range(n):
        k = first_index + i + base
        if save_type == "png":
            names.append("flow%s_%05d.png" % (tag, k))
        else:
            names += ["flow_x%s_%05d.jpg" % (tag, k), "flow_y%s_%05d.jpg" % (tag, k)]
    return names


def h5_names(step, first_index, n):
    """The dataset names writeHDF5 gives a chunk's flows (src/common.cpp:120-150), in the order run_videos hands out their
    h5 files: every flow_x of the chunk, then every flow_y.  Steps > 1 add _p<step>, steps < 0 add _m<|step|> and offset the
    index by |step|, as output_names does."""
    base = -step if step < 0 else 0
    tag = "_p%d" % step if step > 1 else "_m%d" % -step if step < 0 else ""
    return (["/flow_x%s_%05d" % (tag, first_index + i + base) for i in range(n)] +
            ["/flow_y%s_%05d" % (tag, first_index + i + base) for i in range(n)])


def h5_path(outdir, step):
    """The file writeHDF5 writes a video's flows to: <outdir>.h5 (step 1), <outdir>_p<s>.h5 (s > 1), <outdir>_m<|s|>.h5 (s < 0)."""
    outdir = str(outdir).rstrip("/")
    tag = "_p%d" % step if step > 1 else "_m%d" % -step if step < 0 else ""
    return outdir + tag + ".h5"


_SAVE_TYPES = {"jpg": _lib.SAVE_JPG, "png": _lib.SAVE_PNG, "h5": _lib.SAVE_H5}


def _callback(on_chunk, shapes):
    if on_chunk is None:
        return None

    def _cb(user, clip, dev, first, n, last, qx, qy, flows):
        h, w = shapes[clip]
        if qx:
            vx = [np.ctypeslib.as_array(C.cast(qx[i], C.POINTER(C.c_uint8)), (h, w)) for i in range(n)]
            vy = [np.ctypeslib.as_array(C.cast(qy[i], C.POINTER(C.c_uint8)), (h, w)) for i in range(n)]
            on_chunk(clip, dev, first, bool(last), vx, vy, None)
        else:
            vf = [np.ctypeslib.as_array(C.cast(flows[i], C.POINTER(C.c_float)), (h, w, 2)) for i in range(n)]
            on_chunk(clip, dev, first, bool(last), None, None, vf)

    return _lib.CHUNK_DONE_FN(_cb)


def _stats(st):
    W = st.workers
    return {"clips": st.clips, "flows": st.flows, "frames": st.frames, "seconds": st.seconds, "workers": W,
            "clips_per_worker": list(st.clips_per_worker[:W]), "flows_per_worker": list(st.flows_per_worker[:W]),
            "busy_seconds_per_worker": list(st.busy_seconds_per_worker[:W]),
            "finish_seconds_per_worker": list(st.finish_seconds_per_worker[:W]),
            "kernel_launches": st.kernel_launches, "h2d_bytes": st.h2d_bytes, "d2h_bytes": st.d2h_bytes}


def _call(L, fn, *args, stats=True):
    """L.<fn>(*args, [&stats,] err, 512): raises the runner's message, or "<fn> failed (<rc>)" when it leaves none; returns the
    dict of dfb_list_stats."""
    st = _lib.ListStats()
    err = C.create_string_buffer(512)
    rc = getattr(L, fn)(*args, *([C.byref(st)] if stats else []), err, 512)
    if rc != _lib.DFB_OK:
        raise RuntimeError(err.value.decode() or "%s failed (%d)" % (fn, rc))
    return _stats(st)


def _files_per_flow(step, save_type):
    """The files of one output in an on_chunk call: a flow's x and y (jpg, h5) or its PNG, or a frame's JPEG with step 0."""
    if save_type not in _SAVE_TYPES:
        raise RuntimeError("only jpg/png/h5 are supported (no %s) for output" % save_type)
    return 2 if step != 0 and save_type != "png" else 1


def _on_files(on_chunk, per):
    """A FILES_DONE_FN body: hands on_chunk(video, device, first_index, last_chunk, files) the chunk's files as bytes."""
    def done(user, video, dev, first, n, last, files, lens):
        on_chunk(video, dev, first, bool(last), [C.string_at(files[i], lens[i]) for i in range(per * n)])
    return done


class ListRunner:
    """Workers kept alive between lists (dfb_list_open / dfb_list_run / dfb_list_close): worker i owns an engine handle on
    devices[i]; a device may appear more than once."""

    def __init__(self, algorithm, devices, max_width, max_height, variant="default"):
        self._L = _lib.load(variant)
        self._r = C.c_void_p()
        devs = (C.c_int * len(devices))(*devices)
        _call(self._L, "dfb_list_open", algorithm.encode(), devs, len(devices), int(max_width), int(max_height), C.byref(self._r),
              stats=False)  # a refused open leaves the runner null

    def run(self, clips, step=1, bound=32, chunk_flows=0, queue=None, on_chunk=None, packed=None):
        """packed: the result of a previous pack(clips) (building the pointer tables of a long list takes a while)."""
        arr, shapes, keep = packed if packed is not None else _pack_clips(clips)
        cb = _callback(on_chunk, shapes)
        return _call(self._L, "dfb_list_run", self._r, arr, len(shapes), int(step), int(bound), int(chunk_flows),
                     queue._q if queue is not None else None, C.cast(cb, C.c_void_p) if cb else None, None)

    def run_videos(self, videos, step=1, bound=20, save_type="jpg", quality=95, jpeg_exact=0, new_width=0, new_height=0, new_short=0,
                   chunk_flows=0, queue=None, on_chunk=None):
        """The list as the reference takes it (`denseflow list.txt -s=step -b=bound -st=save_type [-if] [-nw/-nh/-ns]`).
        videos: one entry per video, a list of uint8 [H,W,3] BGR frames or a list of JPEG files (bytes).  Each video is resized
        as get_new_size decides and turned into files on the GPU.  on_chunk(video, device, first_index, last_chunk, files) is
        called on the worker's thread once every file of a chunk is in host memory; files is a list of bytes-like views that
        die when the callback returns, named as output_names(step, first_index, n, save_type) names them.  With save_type "h5"
        files 2 i / 2 i + 1 are flow first_index + i's x / y plane as raw float32 [dh, dw] (writeHDF5's datasets, named by
        h5_names).  last_chunk is the
        reference's FlowBuffer::last_buffer.  Returns a dict of dfb_list_stats."""
        per = _files_per_flow(step, save_type)
        arr, keep = _pack_videos(videos)
        cb = _lib.FILES_DONE_FN(_on_files(on_chunk, per)) if on_chunk is not None else None
        return _call(self._L, "dfb_list_run_videos", self._r, arr, len(videos), int(step), int(bound), _SAVE_TYPES[save_type],
                     int(quality), int(jpeg_exact), int(new_width), int(new_height), int(new_short), int(chunk_flows),
                     queue._q if queue is not None else None, C.cast(cb, C.c_void_p) if cb else None, None)

    def run_stream(self, n_videos, source, on_chunk=None, step=1, bound=20, save_type="jpg", quality=95, jpeg_exact=0, new_width=0,
                   new_height=0, new_short=0, chunk_flows=0, queue=None):
        """run_videos with the frames pulled from `source` one window at a time (dfb_list_run_stream), so a list of long videos
        runs in bounded memory.  source(video, first, max_n) returns frames first .. first + max_n - 1 of the video, fewer when
        the video ends there, as uint8 [H,W,3] BGR frames or JPEG files (bytes).  It runs on the worker's thread, in frame order
        for each video; consecutive windows overlap by |step| frames.  A window is kept alive until its on_chunk call returns
        (or until the run ends after a failure).  An exception in source ends the run with "video k: <message>"; one in
        on_chunk ends it too and is raised again here.  on_chunk and the result are those of run_videos, except that a video
        whose outputs end on a window boundary gets one more on_chunk call with no files and last_chunk True."""
        return self._run_source("dfb_list_run_stream", n_videos, source, on_chunk, step, bound, save_type, quality, jpeg_exact,
                                new_width, new_height, new_short, chunk_flows, queue)

    def run_windows(self, n_videos, source, on_chunk=None, step=1, bound=20, save_type="jpg", quality=95, jpeg_exact=0, new_width=0,
                    new_height=0, new_short=0, chunk_flows=0, queue=None):
        """run_stream with a video's windows shared among the workers (dfb_list_run_windows): once the queue is empty, idle
        workers join the unfinished videos, so a single video runs on every worker.  source is called for one video in frame
        order, one call at a time, but possibly from different workers' threads.  A window is kept alive until its on_chunk
        call returns (or until the run ends after a failure).  on_chunk calls for one video come in first_index order, one at
        a time, on the thread of the worker that computed the window.  Arguments, files, errors and the result are
        run_stream's; flows_per_worker counts the flows each worker computed."""
        return self._run_source("dfb_list_run_windows", n_videos, source, on_chunk, step, bound, save_type, quality, jpeg_exact,
                                new_width, new_height, new_short, chunk_flows, queue)

    def _run_source(self, fn, n_videos, source, on_chunk, step, bound, save_type, quality, jpeg_exact, new_width, new_height, new_short,
                    chunk_flows, queue):
        """run_stream and run_windows: the runner is done with each window once its on_chunk call has returned."""
        per = _files_per_flow(step, save_type)
        deliver = _on_files(on_chunk, per) if on_chunk is not None else None
        windows = {}  # (video, first) -> a live window and the memory behind it
        failures = []

        def _source(user, video, first, max_n, out, msg, msg_len):
            try:
                if failures:
                    raise RuntimeError("stopped after an on_chunk call failed")
                v, keep = _pack_video(list(source(video, first, max_n)))
            except Exception as ex:
                text = (str(ex) or type(ex).__name__).encode()[:msg_len - 1]
                C.memmove(msg, text + b"\0", len(text) + 1)
                return 1
            out[0] = v
            windows[(video, first)] = keep
            return 0

        def _done(user, video, dev, first, n, last, files, lens):
            try:
                if deliver is not None and not failures:
                    deliver(user, video, dev, first, n, last, files, lens)
            except BaseException as ex:
                failures.append(ex)
            windows.pop((video, first), None)

        src = _lib.FRAMES_FN(_source)
        cb = _lib.FILES_DONE_FN(_done)
        try:
            return _call(self._L, fn, self._r, int(n_videos), C.cast(src, C.c_void_p), int(step), int(bound), _SAVE_TYPES[save_type],
                         int(quality), int(jpeg_exact), int(new_width), int(new_height), int(new_short), int(chunk_flows),
                         queue._q if queue is not None else None, C.cast(cb, C.c_void_p), None)
        finally:
            windows.clear()
            if failures:  # an on_chunk failure is the cause of any refusal that followed it, and is raised instead
                raise failures[0]

    @staticmethod
    def pack(clips):
        return _pack_clips(clips)

    def close(self):
        if getattr(self, "_r", None):
            self._L.dfb_list_close(self._r)
            self._r = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def run_list(algorithm, devices, clips, step=1, bound=32, chunk_flows=0, queue=None, on_chunk=None, variant="default"):
    """clips: list of sequences of uint8 [H,W] frames (one sequence per video; frames of one video share a size).
    on_chunk(clip_index, device, first_flow, last_chunk, qx, qy, flows): called on the worker's thread when every output of
    a chunk is in host memory (qx/qy: lists of uint8 [H,W] views when bound > 0, flows: list of float32 [H,W,2] views otherwise;
    the views die when the callback returns).  `last_chunk` is the reference's FlowBuffer::last_buffer.
    Returns a dict of dfb_list_stats."""
    L = _lib.load(variant)
    arr, shapes, keep = _pack_clips(clips)
    cb = _callback(on_chunk, shapes)
    devs = (C.c_int * len(devices))(*devices)
    return _call(L, "dfb_run_list", algorithm.encode(), devs, len(devices), arr, len(clips), int(step), int(bound), int(chunk_flows),
                 queue._q if queue is not None else None, C.cast(cb, C.c_void_p) if cb else None, None)
