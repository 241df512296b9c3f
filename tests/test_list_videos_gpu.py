"""The -st=png chains behind the colour frame sources, `-if -s=0`, and the video list over them: every file equals the
single-handle chain's (and, for the strict build, the reference pipeline's own code path run through the oracle), chunks
carry global indices, last_chunk fires once per video after all its files, and a refused JPEG names the video and the
frame without spoiling the runner."""
import threading
import time

import cv2
import numpy as np
import pytest

import jpeg_cases as J

pytestmark = pytest.mark.gpu
_handles = {}


def handle(alg, size=(128, 96), variant="default", exact=0):
    import denseflow_b200 as d
    key = (alg, size, variant)
    if key not in _handles:
        _handles[key] = d.create(alg, 0, size[0], size[1], variant=variant)
    return _handles[key].set("jpeg_exact", exact)


def bgr_frames(n, h, w, seed=0):
    from denseflow_b200 import synth
    gray = synth.stream(h, w, max(n, 1), seed=seed)[:n]
    return [np.stack([np.roll(g, 2, 1), g, 255 - np.roll(g, 3, 0)], -1).astype(np.uint8) for g in gray]


def jpegs(frames):
    return [J.encode(f, "420", 95) for f in frames]


def imdecode(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)


def gray_resized(frames, new_size):
    g = [cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in frames]
    return [cv2.resize(x, new_size, interpolation=cv2.INTER_LINEAR) for x in g] if new_size else g


# ---- the -st=png chains ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("alg", ["tvl1", "farn"])
@pytest.mark.parametrize("step", [1, -1, 3, -3])
@pytest.mark.parametrize("n_frames", [0, 1, 2, 9, 19])
@pytest.mark.parametrize("new_size", [None, (72, 50)])
def test_png_chains_equal_calc_batch_png(alg, step, n_frames, new_size):
    e = handle(alg)
    frames = bgr_frames(n_frames, 64, 96, seed=n_frames)
    files = jpegs(frames)
    decoded = [imdecode(b) for b in files]
    got = e.process_bgr_batch_png(decoded, step, new_size)
    want = e.calc_batch_png(gray_resized(decoded, new_size), step) if n_frames else []
    assert len(got) == max(n_frames - abs(step), 0)
    assert got == want
    assert e.process_jpeg_batch_png(files, step, new_size) == got


def test_png_chains_1080p_groups_and_flows_afterwards():
    from denseflow_b200 import synth
    e = handle("tvl1", (1920, 1080))
    a, b, _ = synth.pair(64, 96, 0)
    f1 = e.calc(a, b)
    frames = bgr_frames(11, 1080, 1920, seed=5)
    files = jpegs(frames)
    decoded = [imdecode(x) for x in files]
    got = e.process_jpeg_batch_png(files, 1)
    assert got == e.process_bgr_batch_png(decoded, 1) == e.calc_batch_png(gray_resized(decoded, None), 1)
    assert e.process_jpeg_batch_png(files[:6], -1, (340, 256)) == e.calc_batch_png(gray_resized(decoded[:6], (340, 256)), -1)
    assert np.array_equal(e.calc(a, b), f1)
    png = got[0]
    assert cv2.imdecode(np.frombuffer(png, np.uint8), cv2.IMREAD_UNCHANGED).shape == (1080, 1920, 3)


def test_png_chains_refuse_what_their_siblings_refuse():
    e = handle("farn")
    frames = bgr_frames(3, 64, 96)
    with pytest.raises(RuntimeError, match="step must be non-zero"):
        e.process_bgr_batch_png(frames, 0)
    with pytest.raises(RuntimeError, match="exceeds"):
        e.process_bgr_batch_png(frames, 1, (256, 64))
    with pytest.raises(RuntimeError, match="frame 2"):
        e.process_jpeg_batch_png(jpegs(frames[:2]) + [J.encode(J.image("smooth", 48, 96), "420", 95)], 1)
    with pytest.raises(RuntimeError, match="progressive"):
        e.process_jpeg_batch_png([J.encode(f, "420", 90, progressive=True) for f in frames], 1)
    # too small: the needed length comes back in the message, and the handle keeps working
    from denseflow_b200 import _lib
    import ctypes as C
    f = [np.ascontiguousarray(x) for x in frames]
    fp = (C.c_void_p * 3)(*[x.ctypes.data for x in f])
    bufs = [np.empty(64, np.uint8) for _ in range(2)]
    op = (C.c_void_p * 2)(*[x.ctypes.data for x in bufs])
    lens = (C.c_size_t * 2)()
    assert e._L.dfb_process_bgr_batch_host_png(e._h, fp, 3, 1, 96, 64, 0, 0, op, 64, lens) == _lib.DFB_ERR_INVALID_ARG
    assert b"needs" in e._L.dfb_last_error(e._h)
    assert e.process_bgr_batch_png(frames, 1) == e.calc_batch_png(gray_resized(frames, None), 1)


# ---- -if -s=0 ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("exact", [0, 1])
@pytest.mark.parametrize("n_frames,new_size", [(1, None), (19, None), (19, (72, 50)), (9, (150, 111))])
def test_extract_frames_jpeg_equals_extract_frames(exact, n_frames, new_size):
    e = handle("tvl1", (160, 120), exact=exact)
    files = jpegs(bgr_frames(n_frames, 64, 96, seed=n_frames))
    decoded = [imdecode(b) for b in files]
    got = e.extract_frames_jpeg(files, new_size)
    assert got == e.extract_frames(decoded, new_size)
    if exact:
        want = [cv2.imencode(".jpg", cv2.resize(d, new_size, interpolation=cv2.INTER_LINEAR) if new_size else d)[1].tobytes()
                for d in decoded]
        assert got == want
    # a corrupt frame in the second group of eight is named in the call
    with pytest.raises(RuntimeError, match="frame 9: .*ends before the last MCU"):
        e.extract_frames_jpeg((files * 10)[:9] + [J.truncated(64, 96)], new_size)
    assert e.extract_frames_jpeg(files, new_size) == got


# ---- the list over videos ---------------------------------------------------------------------------------------------

def _videos():
    """BGR and JPEG videos of different source sizes; -ns 80 resizes the 128x96 ones (short side 96) and not the 96x64 ones;
    a one-frame video and an empty one."""
    return [bgr_frames(9, 64, 96, seed=1), jpegs(bgr_frames(7, 96, 128, seed=2)), bgr_frames(1, 64, 96, seed=3), [],
            jpegs(bgr_frames(10, 64, 96, seed=4)), bgr_frames(6, 96, 128, seed=5)]


def _devices():
    import torch
    return [0, 0, 0] + list(range(1, torch.cuda.device_count()))


def _single(e, video, step, save_type, new_size, bound=20):
    """the single-handle chain's files for one video, in run_videos' order"""
    if not video:
        return []
    is_jpeg = isinstance(video[0], bytes)
    if step == 0:
        return e.extract_frames_jpeg(video, new_size) if is_jpeg else e.extract_frames(video, new_size)
    if save_type == "png":
        return e.process_jpeg_batch_png(video, step, new_size) if is_jpeg else e.process_bgr_batch_png(video, step, new_size)
    pairs = e.process_jpeg_batch(video, step, bound, new_size) if is_jpeg else e.process_bgr_batch(video, step, bound, new_size)
    return [f for p in pairs for f in p]


def _run(r, videos, step, save_type, **kw):
    got = {i: {} for i in range(len(videos))}
    events = []
    lock = threading.Lock()
    per = 2 if step != 0 and save_type == "jpg" else 1

    def on_chunk(video, dev, first, last, files):
        with lock:
            assert len(files) % per == 0
            for k, f in enumerate(files):
                got[video][per * first + k] = bytes(f)
            events.append((video, first, len(files) // per, last, threading.get_ident()))

    st = r.run_videos(videos, step=step, save_type=save_type, chunk_flows=4, on_chunk=on_chunk, **kw)
    for i in range(len(videos)):
        mine = [ev for ev in events if ev[0] == i]
        lasts = [ev for ev in mine if ev[3]]
        assert len(lasts) == 1 and mine[-1] is lasts[0], (i, mine)  # once, after every other chunk of the video
        firsts = [ev[1] for ev in mine]
        assert firsts == sorted(firsts)
        assert len({ev[4] for ev in mine}) == 1, (i, mine)  # every chunk from the worker that took the video
    return [[got[i][k] for k in range(len(got[i]))] for i in range(len(videos))], st


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
def test_run_videos_equals_single_handle_chains(alg):
    from denseflow_b200 import api, listrun
    videos = _videos()
    r = listrun.ListRunner(alg, _devices(), 128, 96)
    try:
        for step, save_type, exact in [(1, "jpg", 1), (-1, "jpg", 1), (3, "png", 0), (1, "png", 0), (-1, "png", 0), (3, "jpg", 0),
                                       (0, "jpg", 1), (0, "jpg", 0)]:
            e = handle(alg, exact=exact)
            files, st = _run(r, videos, step, save_type, jpeg_exact=exact, new_short=80)
            for i, v in enumerate(videos):
                src = (imdecode(v[0]).shape if isinstance(v[0], bytes) else v[0].shape) if v else (1, 1)
                dw, dh = api.new_size(src[1], src[0], new_short=80)
                want = _single(e, v, step, save_type, (dw, dh) if (dw, dh) != (src[1], src[0]) else None)
                assert files[i] == want, (step, save_type, i)
            n_out = [max(len(v) - abs(step), 0) if step else len(v) for v in videos]
            assert st["clips"] == len(videos) and st["frames"] == sum(len(v) for v in videos)
            assert st["flows"] == (sum(n_out) if step else 0)
            assert sum(st["clips_per_worker"]) == len(videos)
        # a following run_list on the same runner gives its normal results
        _check_run_list(r, alg)
    finally:
        r.close()


def _check_run_list(r, alg):
    from denseflow_b200 import synth
    clips = [list(synth.stream(64, 96, n, seed=40 + n)) for n in (6, 3)]
    e = handle(alg)
    got = {}

    def on_chunk(clip, dev, first, last, qx, qy, flows):
        for k in range(len(qx)):
            got[(clip, first + k)] = (qx[k].copy(), qy[k].copy())

    r.run(clips, step=1, bound=20, chunk_flows=4, on_chunk=on_chunk)
    for i, c in enumerate(clips):
        qx, qy = e.calc_batch(c, step=1, bound=20)
        for j in range(len(qx)):
            assert np.array_equal(got[(i, j)][0], qx[j]) and np.array_equal(got[(i, j)][1], qy[j])


def test_run_videos_refusals_name_the_video_and_frame():
    from denseflow_b200 import listrun
    videos = _videos()
    r = listrun.ListRunner("farn", [0, 0, 0], 128, 96)
    try:
        with pytest.raises(RuntimeError, match="bound should > 0!"):
            r.run_videos(videos, step=1, bound=0)
        with pytest.raises(RuntimeError, match="do not set height and width when set short!"):
            r.run_videos(videos, step=1, new_width=64, new_short=64)
        frames = bgr_frames(10, 64, 96, seed=4)
        prog = list(videos[4])
        prog[6] = J.encode(frames[6], "420", 90, progressive=True)  # second chunk (frames 4..8): named in the video
        trunc = list(videos[4])
        whole = trunc[5]
        trunc[5] = whole[:int(len(whole) * 0.6)] + b"\xff\xd9"
        for bad, msg in [(prog, "video 4: frame 6: .*progressive"), (trunc, "video 4: frame 5: .*ends before the last MCU")]:
            vs = videos[:4] + [bad] + videos[5:]
            for step, st in [(1, "jpg"), (1, "png"), (0, "jpg")]:
                with pytest.raises(RuntimeError, match=msg):
                    r.run_videos(vs, step=step, save_type=st, chunk_flows=4)
        first_bad = [J.encode(frames[0], "420", 90, progressive=True)] + list(videos[4][1:])
        with pytest.raises(RuntimeError, match="video 1: frame 0: .*progressive"):
            r.run_videos([videos[0], first_bad], step=1)
        # the runner stays usable: run_videos and run_list give their normal results
        files, _ = _run(r, videos, 1, "png", new_short=80)
        e = handle("farn")
        assert files[4] == e.process_jpeg_batch_png(videos[4], 1)
        assert files[5] == e.process_bgr_batch_png(videos[5], 1, (107, 80))
        _check_run_list(r, "farn")
    finally:
        r.close()


def test_a_failure_lets_the_other_workers_finish_their_videos():
    """Video 1 fails at its second chunk (a corrupt frame 6) while video 0, longer, runs on another worker: video 0 still gets
    every chunk, its last_chunk included, with a clean run's bytes, and the run reports video 1's error."""
    from denseflow_b200 import listrun
    frames = bgr_frames(10, 64, 96, seed=4)
    bad = jpegs(frames)
    bad[6] = bad[6][:int(len(bad[6]) * 0.6)] + b"\xff\xd9"
    videos = [jpegs(bgr_frames(4 * 12 + 1, 64, 96, seed=7)), bad]
    started = threading.Event()
    threads = {0: set(), 1: set()}
    chunks = []

    def on_chunk(video, dev, first, last, files):
        threads[video].add(threading.get_ident())
        if video == 1:
            started.set()
            return
        if first == 0:
            started.wait(60)  # video 1 runs on another worker
            time.sleep(0.5)   # and fails at its next chunk meanwhile
        chunks.append((first, last, [bytes(f) for f in files]))

    r = listrun.ListRunner("farn", [0, 0, 0], 96, 64)
    try:
        with pytest.raises(RuntimeError, match="^video 1: frame 6: .*ends before the last MCU"):
            r.run_videos(videos, step=1, chunk_flows=4, jpeg_exact=1, on_chunk=on_chunk)
        clean = []
        r.run_videos(videos[:1], step=1, chunk_flows=4, jpeg_exact=1,
                     on_chunk=lambda v, d, f, last, fs: clean.append((f, last, [bytes(x) for x in fs])))
    finally:
        r.close()
    assert started.is_set() and len(threads[0]) == len(threads[1]) == 1 and threads[0] != threads[1], threads
    assert chunks == clean and [c[0] for c in clean] == list(range(0, 48, 4)) and [c[1] for c in clean] == [False] * 11 + [True]


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
def test_run_videos_strict_equals_the_reference_pipeline(alg, oracle):
    """One 64x48 `-if` video of 5 frames: the strict build's files are the bytes the reference's own code path writes, with
    the oracle's flows in place of the GPU ones: imencode(".jpg", convertFlowToImage(flow)) and
    imencode(".png", convertFlowToPngImage(flow))."""
    from denseflow_b200 import listrun
    from oracle import cv_restate
    video = jpegs(bgr_frames(5, 48, 64, seed=9))
    gray = [cv2.cvtColor(imdecode(b), cv2.COLOR_BGR2GRAY) for b in video]
    calc = oracle.tvl1_calc if alg == "tvl1" else oracle.farn_calc
    flows = [calc(gray[j], gray[j + 1]) for j in range(4)]
    r = listrun.ListRunner(alg, [0], 64, 48, variant="strict")
    try:
        jpg, _ = _run(r, [video], 1, "jpg", jpeg_exact=1, bound=20)
        png, _ = _run(r, [video], 1, "png", jpeg_exact=1)
    finally:
        r.close()
    want_jpg = []
    for f in flows:
        qx, qy = oracle.quantise(f, 20)
        want_jpg += [cv2.imencode(".jpg", qx)[1].tobytes(), cv2.imencode(".jpg", qy)[1].tobytes()]
    assert jpg[0] == want_jpg
    assert png[0] == [cv2.imencode(".png", cv_restate.flow_to_png_image(f)[0])[1].tobytes() for f in flows]
