"""ListRunner.run_windows (dfb_list_run_windows) on the GPU: a video's windows shared among the workers give run_stream's files,
chunks and counts for every mode, one video runs on several workers with its reads in order and its chunks delivered in
order, windows live until their chunk is delivered and no longer, failures report the earliest failed window and leave the
runner usable, joining workers grow their handles, and the command writes the same tree from a single input on every
worker."""
import os
import threading
import time
import weakref

import numpy as np
import pytest

import h5_read
from test_cli_gpu import _videos, bgr_frames, jpegs, read_video, tree, window_source, write_ffv1

pytestmark = pytest.mark.gpu


def run_collect(run, n_videos, step, save_type):
    """Run `run(on_chunk)`; per video its files in index order and its (first, n, last) sequence, after checking that the
    chunks of a video never overlap in time."""
    per = 2 if step != 0 and save_type != "png" else 1
    files = {i: {} for i in range(n_videos)}
    seq = {i: [] for i in range(n_videos)}
    busy = set()
    lock = threading.Lock()

    def on_chunk(video, dev, first, last, fs):
        with lock:
            assert video not in busy
            busy.add(video)
        try:
            for k, f in enumerate(fs):
                files[video][per * first + k] = bytes(f)
            seq[video].append((first, len(fs) // per, last))
        finally:
            with lock:
                busy.discard(video)

    st = run(on_chunk)
    return [[files[i][k] for k in range(len(files[i]))] for i in range(n_videos)], [seq[i] for i in range(n_videos)], st


def assert_same_run(got, want):
    (gf, gs, gst), (wf, ws, wst) = got, want
    assert gf == wf
    assert gs == ws
    for k in ("clips", "flows", "frames"):
        assert gst[k] == wst[k], k
    assert sum(gst["flows_per_worker"]) == gst["flows"]
    assert sum(gst["clips_per_worker"]) == gst["clips"]


# (step, save type, -ns): every step with two save types, h5 included, with and without a resize
CONFIGS = [(1, "jpg", 0), (1, "h5", 80), (-1, "png", 80), (-1, "h5", 0), (3, "jpg", 80), (3, "png", 0), (-3, "jpg", 0),
           (-3, "h5", 80), (0, "jpg", 0), (0, "jpg", 80)]


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
def test_run_windows_equals_run_stream(alg):
    from denseflow_b200 import listrun
    one = listrun.ListRunner(alg, [0], 128, 96)
    shared = listrun.ListRunner(alg, [0, 0, 0, 0], 32, 32)  # every worker grows its handle
    try:
        for step, save_type, ns in CONFIGS:
            videos = _videos(step)
            kw = dict(step=step, save_type=save_type, jpeg_exact=1, new_short=ns, chunk_flows=4, bound=20)
            want = run_collect(lambda cb: one.run_stream(len(videos), window_source(videos), cb, **kw), len(videos), step, save_type)
            calls = []
            got = run_collect(lambda cb: shared.run_windows(len(videos), window_source(videos, calls), cb, **kw), len(videos), step,
                              save_type)
            assert_same_run(got, want)
            # the windows run_stream asks for, once each and in order per video
            for i in range(len(videos)):
                firsts = [c[1] for c in calls if c[0] == i]
                assert firsts[0] == 0 and all(b - a == 4 for a, b in zip(firsts, firsts[1:])), (step, save_type, i)
                assert all(c[2] == 4 + abs(step) for c in calls if c[0] == i)
    finally:
        one.close()
        shared.close()


def test_one_video_runs_on_several_workers():
    from denseflow_b200 import listrun
    frames = bgr_frames(4 * 40 + 1, 96, 128, seed=21)  # 40 windows at chunk 4
    lock = threading.Lock()
    reading, reads, chunks = [False], [], []

    def source(video, first, max_n):
        with lock:
            assert not reading[0], first  # one call at a time for the video
            reading[0] = True
            reads.append(first)
        time.sleep(0.004)
        with lock:
            reading[0] = False
        return frames[first:first + max_n]

    def on_chunk(video, dev, first, last, files):
        chunks.append((first, len(files) // 2, last))

    r = listrun.ListRunner("tvl1", [0, 0, 0], 128, 96)
    try:
        st = r.run_windows(1, source, on_chunk, step=1, chunk_flows=4, jpeg_exact=1)
        want = run_collect(lambda cb: r.run_stream(1, window_source([frames]), cb, step=1, chunk_flows=4, jpeg_exact=1), 1, 1, "jpg")
    finally:
        r.close()
    assert reads == [4 * j for j in range(41)]
    assert chunks == want[1][0] and [c[0] for c in chunks] == sorted(c[0] for c in chunks)
    assert st["flows"] == 160 and st["clips"] == 1 and st["frames"] == 161
    assert sum(1 for f in st["flows_per_worker"] if f > 0) >= 2, st["flows_per_worker"]


def test_live_frames_stay_within_the_window_bound():
    from denseflow_b200 import listrun
    live = [0, 0]
    lock = threading.Lock()

    def gone():
        with lock:
            live[0] -= 1

    def source(video, first, max_n):
        n = max(min(max_n, 120 - first), 0)
        out = []
        for k in range(n):
            f = np.full((48, 64, 3), (first + k + 40 * video) % 256, np.uint8)
            with lock:
                live[0] += 1
                live[1] = max(live[1], live[0])
            weakref.finalize(f, gone)
            out.append(f)
        return out

    r = listrun.ListRunner("farn", [0, 0, 0], 64, 48)
    try:
        st = r.run_windows(2, source, None, step=2, chunk_flows=8)
    finally:
        r.close()
    assert st["frames"] == 2 * 120 and st["flows"] == 2 * 118
    assert live[1] <= 3 * (8 + 2), live
    assert live[0] == 0


def test_a_window_is_not_read_after_its_chunk():
    """A source that overwrites each window's frames as soon as its chunk is delivered still gives run_stream's bytes."""
    from denseflow_b200 import listrun
    videos = [bgr_frames(4 * 12 + 1, 48, 64, seed=31), jpegs(bgr_frames(4 * 9 + 3, 48, 64, seed=32))]
    held = {}
    lock = threading.Lock()

    def source(video, first, max_n):
        win = [bytearray(f) if isinstance(f, bytes) else f.copy() for f in videos[video][first:first + max_n]]
        with lock:
            held[(video, first)] = win
        return win

    def overwrite(video, first):
        with lock:
            win = held.pop((video, first))
        for f in win:
            if isinstance(f, bytearray):
                f[:] = b"\0" * len(f)
            else:
                f[...] = 0

    r = listrun.ListRunner("tvl1", [0, 0, 0], 64, 48)
    try:
        for step, save_type in [(1, "jpg"), (-3, "png"), (0, "jpg")]:
            got = {}

            def on_chunk(video, dev, first, last, files):
                got[(video, first)] = [bytes(f) for f in files]
                overwrite(video, first)

            r.run_windows(2, source, on_chunk, step=step, save_type=save_type, chunk_flows=4, jpeg_exact=1)
            want = {}
            r.run_stream(2, window_source(videos), lambda v, d, f, last, fs: want.__setitem__((v, f), [bytes(x) for x in fs]),
                         step=step, save_type=save_type, chunk_flows=4, jpeg_exact=1)
            assert got == want, (step, save_type)
    finally:
        r.close()


def test_windows_are_shared_only_after_the_last_video_started():
    from denseflow_b200 import listrun
    lengths = [41, 5, 9, 30, 13, 7, 50, 3, 21, 11, 60, 2]
    videos = [bgr_frames(n, 48, 64, seed=40 + i) for i, n in enumerate(lengths)]
    lock = threading.Lock()
    events = []  # ("read" | "chunk", video, first, thread)

    def source(video, first, max_n):
        with lock:
            events.append(("read", video, first, threading.get_ident()))
        return videos[video][first:first + max_n]

    def on_chunk(video, dev, first, last, files):
        with lock:
            events.append(("chunk", video, first, threading.get_ident()))

    r = listrun.ListRunner("farn", [0, 0, 0], 64, 48)
    try:
        st = r.run_windows(len(videos), source, on_chunk, step=1, chunk_flows=4)
    finally:
        r.close()
    assert st["clips"] == len(videos) and st["flows"] == sum(n - 1 for n in lengths)
    last_start = next(k for k, e in enumerate(events) if e[:3] == ("read", len(videos) - 1, 0))
    owner = {e[1]: e[3] for e in events if e[0] == "chunk" and e[2] == 0}
    for k, e in enumerate(events):
        if e[0] == "chunk" and e[3] != owner[e[1]]:
            assert k > last_start, (e, last_start)


def _corrupt(blob):
    return blob[:int(len(blob) * 0.6)] + b"\xff\xd9"


def test_failures_report_the_earliest_window():
    from denseflow_b200 import listrun
    good = bgr_frames(4 * 20 + 1, 48, 64, seed=50)  # 20 windows at chunk 4: window j reads frames 4 j .. 4 j + 4
    files = jpegs(good)
    bad5 = list(files)
    bad5[22] = _corrupt(files[22])  # window 5 only
    bad57 = list(bad5)
    bad57[30] = _corrupt(files[30])  # and window 7
    other = list(files[:30]) + jpegs(bgr_frames(51, 64, 96, seed=51))  # frame 30 on: 96x64

    def failing(video, first, max_n):
        if first >= 40:
            raise ValueError("cannot read frame %d" % first)
        return good[first:first + max_n]

    def broken(video, dev, first, last, fl):
        raise KeyError("on_chunk")

    r = listrun.ListRunner("tvl1", [0, 0, 0, 0], 64, 48)
    want = run_collect(lambda cb: r.run_stream(1, window_source([files]), cb, step=1, chunk_flows=4, jpeg_exact=1), 1, 1, "jpg")
    try:
        for source, text, first_failed in [(window_source([bad5]), "^video 0: frame 22: .*ends before the last MCU", 20),
                                           (window_source([bad57]), "^video 0: frame 22: .*ends before the last MCU", 20),
                                           (failing, "^video 0: cannot read frame 40$", 40),
                                           (window_source([other]), "^video 0: frame 30: 96x64, frame 0 is 64x48$", 28)]:
            chunks = []
            with pytest.raises(RuntimeError, match=text):
                r.run_windows(1, source, lambda v, d, f, last, fs: chunks.append(f), step=1, chunk_flows=4, jpeg_exact=1)
            # every window before the failed one is delivered, in order, and none from it on
            assert chunks == list(range(0, first_failed, 4)), (text, chunks)
            got = run_collect(lambda cb: r.run_windows(1, window_source([files]), cb, step=1, chunk_flows=4, jpeg_exact=1), 1, 1,
                              "jpg")
            assert_same_run(got, want)
        with pytest.raises(KeyError):
            r.run_windows(1, window_source([good]), broken, step=1, chunk_flows=4)
        got = run_collect(lambda cb: r.run_windows(1, window_source([files]), cb, step=1, chunk_flows=4, jpeg_exact=1), 1, 1, "jpg")
        assert_same_run(got, want)
    finally:
        r.close()


def test_joining_workers_grow_their_handles():
    from denseflow_b200 import listrun
    small, large = bgr_frames(6, 48, 64, seed=60), bgr_frames(4 * 16 + 1, 240, 320, seed=61)
    one = listrun.ListRunner("tvl1", [0], 64, 48)
    shared = listrun.ListRunner("tvl1", [0, 0, 0], 64, 48)

    def slow(video, first, max_n):
        time.sleep(0.002)
        return [small, large][video][first:first + max_n]

    try:
        kw = dict(step=1, chunk_flows=4, jpeg_exact=1)
        want = run_collect(lambda cb: one.run_stream(2, window_source([small, large]), cb, **kw), 2, 1, "jpg")
        got = run_collect(lambda cb: shared.run_windows(2, slow, cb, **kw), 2, 1, "jpg")
        assert_same_run(got, want)
        assert sum(1 for f in got[2]["flows_per_worker"] if f > 0) >= 2, got[2]
        # the grown handles still run a small video
        again = run_collect(lambda cb: shared.run_windows(1, window_source([small]), cb, **kw), 1, 1, "jpg")
        assert again[0][0] == want[0][0]
    finally:
        one.close()
        shared.close()


# ---- the command ---------------------------------------------------------------------------------------------------------

def cli_run(args, monkeypatch=None, variant="default"):
    """cli.run; with monkeypatch, through run_stream on one worker per device (what the command ran before it shared a video's
    windows).  Returns the stats and the printed lines."""
    from denseflow_b200 import cli, listrun
    lines = []
    with pytest.MonkeyPatch.context() as mp:
        if monkeypatch:
            mp.setattr(cli, "WORKERS_PER_DEVICE", 1)
            mp.setattr(listrun.ListRunner, "run_windows", listrun.ListRunner.run_stream)
        st = cli.run(cli.parse_args(args), lines.append, variant=variant)
    return st, lines


def _same_summary(a, b):
    head = lambda s: s.split(" processed")[0]
    assert head(a) == head(b), (a, b)


def test_cli_single_inputs_on_every_worker(tmp_path):
    frames = bgr_frames(150, 96, 128, seed=70)
    write_ffv1(tmp_path / "clip.avi", frames)
    assert len(read_video(tmp_path / "clip.avi")) == 150
    (tmp_path / "data" / "f").mkdir(parents=True)
    for i, blob in enumerate(jpegs(bgr_frames(151, 96, 128, seed=71))):
        (tmp_path / "data" / "f" / ("img_%05d.jpg" % i)).write_bytes(blob)
    (tmp_path / "list.txt").write_text(str(tmp_path / "data" / "f") + "\n")
    cases = [([str(tmp_path / "clip.avi"), "-s=1", "-b=20"], "clip"),
             ([str(tmp_path / "data" / "f"), "-if", "-s=-2", "-st=png", "-ns=64"], "f"),
             ([str(tmp_path / "list.txt"), "-if", "-s=3", "-b=20"], "."),  # a list of one: the .done marker too
             ([str(tmp_path / "clip.avi"), "-s=0"], "clip")]
    for k, (args, sub) in enumerate(cases):
        st, lines = cli_run(args + ["-o=" + str(tmp_path / ("w%d" % k))])
        st1, lines1 = cli_run(args + ["-o=" + str(tmp_path / ("s%d" % k))], monkeypatch=True)
        got, want = tree(tmp_path / ("w%d" % k) / sub), tree(tmp_path / ("s%d" % k) / sub)
        assert got == want and len(got) > 100, args
        assert lines[:-1] == lines1[:-1]
        _same_summary(lines[-1], lines1[-1])
        for key in ("clips", "flows", "frames"):
            assert st[key] == st1[key]
        assert sum(1 for f in st["flows_per_worker"] if f > 0) >= 2 or args[1] == "-s=0", st
    assert os.path.isfile(tmp_path / "w2" / ".done" / "f")


def test_cli_h5_single_video_on_every_worker(tmp_path):
    frames = bgr_frames(150, 96, 128, seed=72)
    write_ffv1(tmp_path / "clip.avi", frames)
    args = [str(tmp_path / "clip.avi"), "-s=1", "-b=20", "-st=h5"]
    st, _ = cli_run(args + ["-o=" + str(tmp_path / "w")], variant="hdf5")
    cli_run(args + ["-o=" + str(tmp_path / "s")], monkeypatch=True, variant="hdf5")
    got, want = open(tmp_path / "w" / "clip.h5", "rb").read(), open(tmp_path / "s" / "clip.h5", "rb").read()
    assert got == want
    names = h5_read.H5File(str(tmp_path / "w" / "clip.h5")).names
    assert len(names) == 2 * 149 and "flow_x_00000" in names and "flow_y_00148" in names
    assert sum(1 for f in st["flows_per_worker"] if f > 0) >= 2, st


@pytest.mark.parametrize("step,chunk", [(1, 2), (-2, 3), (0, 2)])
def test_counts_without_a_done_callback(step, chunk):
    """dfb_list_run_windows through the C ABI with done = NULL: the workers sharing a video deliver with nothing to call, so
    the worker of a video's final window can reach it right behind the previous window's.  Every window's flows still
    count, once, and the video leaves the run only after all of them."""
    import ctypes as C
    from denseflow_b200 import _lib, listrun
    lengths = [97, 61]
    videos = [bgr_frames(n, 48, 64, seed=80 + i) for i, n in enumerate(lengths)]
    keep = []

    def source(user, video, first, max_n, out, msg, msg_len):
        v, k = listrun._pack_video(videos[video][first:first + max_n])
        keep.append(k)  # every window stays alive until the call returns
        out[0] = v
        return 0

    src = _lib.FRAMES_FN(source)
    r = listrun.ListRunner("farn", [0] * 6, 64, 48)
    try:
        st = _lib.ListStats()
        err = C.create_string_buffer(512)
        rc = r._L.dfb_list_run_windows(r._r, len(videos), C.cast(src, C.c_void_p), step, 20, _lib.SAVE_JPG, 95, 0, 0, 0, 0, chunk,
                                       None, None, None, C.byref(st), err, 512)
    finally:
        r.close()
    assert rc == _lib.DFB_OK, err.value
    s = listrun._stats(st)
    flows = sum(max(n - abs(step), 0) for n in lengths) if step else 0
    assert s["flows"] == flows and sum(s["flows_per_worker"]) == flows, s
    assert s["clips"] == len(videos) == sum(s["clips_per_worker"]) and s["frames"] == sum(lengths), s
    assert sum(1 for f in s["flows_per_worker"] if f > 0) >= 2 or step == 0, s
