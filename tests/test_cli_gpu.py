"""ListRunner.run_stream (dfb_list_run_stream) and `python -m denseflow_b200` on the GPU: streamed windows give run_videos'
bytes for every mode, the frames a source has to keep alive stay within the window bound, handles grow to a larger video,
failures name the video and frame and leave the runner usable, and the command writes the reference's tree."""
import os
import threading
import weakref

import cv2
import numpy as np
import pytest

import jpeg_cases as J

pytestmark = pytest.mark.gpu


def bgr_frames(n, h, w, seed=0):
    from denseflow_b200 import synth
    gray = synth.stream(h, w, max(n, 1), seed=seed)[:n]
    return [np.stack([np.roll(g, 2, 1), g, 255 - np.roll(g, 3, 0)], -1).astype(np.uint8) for g in gray]


def jpegs(frames):
    return [J.encode(f, "420", 95) for f in frames]


def collect(run, n_videos, step, save_type, calls=None):
    """Run `run(on_chunk)`; the files per video in index order, after checking that last_chunk comes once per video after
    all its files, that chunks arrive in order, and that every chunk of a video (and every source call in `calls`, as
    window_source records them) comes from one thread."""
    per = 2 if step != 0 and save_type == "jpg" else 1
    got = {i: {} for i in range(n_videos)}
    events = []
    lock = threading.Lock()

    def on_chunk(video, dev, first, last, files):
        with lock:
            for k, f in enumerate(files):
                got[video][per * first + k] = bytes(f)
            events.append((video, first, len(files) // per, last, threading.get_ident()))

    st = run(on_chunk)
    for i in range(n_videos):
        mine = [ev for ev in events if ev[0] == i]
        assert [ev[3] for ev in mine].count(True) == 1 and mine[-1][3], (i, mine)
        assert [ev[1] for ev in mine] == sorted(ev[1] for ev in mine)
        threads = {ev[4] for ev in mine} | {c[3] for c in calls or [] if c[0] == i}
        assert len(threads) == 1, (i, threads)
    return [[got[i][k] for k in range(len(got[i]))] for i in range(n_videos)], st


def window_source(videos, calls=None):
    """source(video, first, max_n) over whole videos in memory; with `calls`, records (video, first, max_n, thread) per call."""
    def source(video, first, max_n):
        if calls is not None:
            calls.append((video, first, max_n, threading.get_ident()))
        return videos[video][first:first + max_n]
    return source


def _videos(step):
    """BGR and JPEG videos of two sizes whose lengths are 0, 1, |step|, exactly one window (chunk 4 + |step|) and several."""
    a = max(abs(step), 1)
    win = 4 + abs(step)
    lens = [0, 1, a, win, 3 * win + 2, 2 * 4 + abs(step)]
    out = []
    for i, n in enumerate(lens):
        h, w = (64, 96) if i % 2 == 0 else (96, 128)
        f = bgr_frames(n, h, w, seed=10 + i)
        out.append(jpegs(f) if i % 3 == 1 else f)
    return out


CONFIGS = [(1, "jpg", 0), (-1, "png", 80), (3, "jpg", 80), (3, "png", 0), (-3, "jpg", 0), (0, "jpg", 0), (0, "jpg", 80)]


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
def test_run_stream_equals_run_videos(alg):
    from denseflow_b200 import listrun
    whole = listrun.ListRunner(alg, [0, 0, 0], 128, 96)
    stream = listrun.ListRunner(alg, [0, 0, 0], 32, 32)  # every worker grows its handle
    try:
        for step, save_type, ns in CONFIGS:
            videos = _videos(step)
            kw = dict(step=step, save_type=save_type, jpeg_exact=1, new_short=ns, chunk_flows=4, bound=20)
            want, st_w = collect(lambda cb: whole.run_videos(videos, on_chunk=cb, **kw), len(videos), step, save_type)
            calls = []
            got, st_s = collect(lambda cb: stream.run_stream(len(videos), window_source(videos, calls), cb, **kw), len(videos), step,
                                save_type, calls)
            assert got == want, (step, save_type, ns)
            for k in ("clips", "flows", "frames"):
                assert st_s[k] == st_w[k], (k, step, save_type)
            # windows of at most chunk + |step| frames, overlapping by |step|, asked in order per video
            for i in range(len(videos)):
                firsts = [c[1] for c in calls if c[0] == i]
                assert firsts == sorted(firsts) and firsts[0] == 0
                assert all(c[2] == 4 + abs(step) for c in calls if c[0] == i)
                assert all(b - a == 4 for a, b in zip(firsts, firsts[1:]))
    finally:
        whole.close()
        stream.close()


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
        st = r.run_stream(4, source, None, step=2, chunk_flows=8)
    finally:
        r.close()
    assert st["frames"] == 4 * 120 and st["flows"] == 4 * 118
    assert live[1] <= 3 * (8 + 2), live
    assert live[0] == 0


def test_handle_grows_for_a_larger_video():
    from denseflow_b200 import api, listrun
    small, large = bgr_frames(6, 48, 64, seed=1), bgr_frames(6, 240, 320, seed=2)
    r = listrun.ListRunner("tvl1", [0], 64, 48)
    try:
        got, st = collect(lambda cb: r.run_stream(2, window_source([small, large]), cb, step=1, chunk_flows=4, jpeg_exact=1),
                          2, 1, "jpg")
        again, _ = collect(lambda cb: r.run_stream(1, window_source([small]), cb, step=1, chunk_flows=4, jpeg_exact=1), 1, 1, "jpg")
    finally:
        r.close()
    e = api.create("tvl1", 0, 320, 240).set("jpeg_exact", 1)
    for v, files in zip([small, large], got):
        assert files == [f for p in e.process_bgr_batch(v, 1, 20) for f in p]
    assert again[0] == got[0]
    assert st["kernel_launches"] > 0


def test_failures_name_the_video_and_frame():
    from denseflow_b200 import listrun
    good = bgr_frames(10, 48, 64, seed=3)
    files = jpegs(good)
    corrupt = list(files)
    corrupt[6] = files[6][:int(len(files[6]) * 0.6)] + b"\xff\xd9"
    resized = list(good[:4]) + bgr_frames(5, 64, 96, seed=4)

    def failing(video, first, max_n):
        if video == 1 and first >= 4:
            raise ValueError("cannot read frame %d" % first)
        return good[first:first + max_n]

    r = listrun.ListRunner("farn", [0, 0], 64, 48)
    try:
        with pytest.raises(RuntimeError, match="^video 1: cannot read frame 4$"):
            r.run_stream(2, failing, None, step=1, chunk_flows=4)
        with pytest.raises(RuntimeError, match="video 1: frame 6: .*ends before the last MCU"):
            r.run_stream(2, window_source([files, corrupt]), None, step=1, chunk_flows=4)
        with pytest.raises(RuntimeError, match="video 0: frame 4: 96x64, frame 0 is 64x48"):
            r.run_stream(1, window_source([resized]), None, step=0, chunk_flows=4)
        with pytest.raises(RuntimeError, match="video 0: .*frames must be uint8"):
            r.run_stream(1, lambda v, f, n: [np.zeros((4, 4), np.float32)], None, step=1)

        def broken(video, dev, first, last, fl):
            raise KeyError("on_chunk")

        with pytest.raises(KeyError):
            r.run_stream(1, window_source([good]), broken, step=1, chunk_flows=4)
        # the runner keeps working
        got, _ = collect(lambda cb: r.run_stream(2, window_source([good, files]), cb, step=1, chunk_flows=4, save_type="png"), 2, 1,
                         "png")
        want, _ = collect(lambda cb: r.run_videos([good, files], step=1, chunk_flows=4, save_type="png", on_chunk=cb), 2, 1, "png")
        assert got == want and len(got[0]) == 9
    finally:
        r.close()


def test_a_failure_lets_the_other_workers_finish_their_videos():
    """Video 1 fails at its second window while video 0, longer, runs on another worker: video 0 still gets every chunk, its
    last_chunk included, with a clean run's bytes, and the run reports video 1's error."""
    from denseflow_b200 import listrun
    videos = [bgr_frames(4 * 12 + 1, 48, 64, seed=5), bgr_frames(10, 48, 64, seed=6)]
    failed = threading.Event()
    threads = {0: set(), 1: set()}
    chunks = []

    def source(video, first, max_n):
        threads[video].add(threading.get_ident())
        if video == 1 and first >= 4:
            failed.set()
            raise ValueError("cannot read frame %d" % first)
        if video == 0 and first == 8:
            failed.wait(60)  # video 0 is mid-way when video 1 fails
        return videos[video][first:first + max_n]

    def on_chunk(video, dev, first, last, files):
        threads[video].add(threading.get_ident())
        if video == 0:
            chunks.append((first, last, [bytes(f) for f in files]))

    r = listrun.ListRunner("farn", [0, 0, 0], 64, 48)
    try:
        with pytest.raises(RuntimeError, match="^video 1: cannot read frame 4$"):
            r.run_stream(2, source, on_chunk, step=1, chunk_flows=4, jpeg_exact=1)
        clean = []
        r.run_stream(1, window_source(videos), lambda v, d, f, last, fs: clean.append((f, last, [bytes(x) for x in fs])), step=1,
                     chunk_flows=4, jpeg_exact=1)
    finally:
        r.close()
    assert failed.is_set() and len(threads[0]) == len(threads[1]) == 1 and threads[0] != threads[1], threads
    assert chunks == clean and clean[-1][1] and sum(len(c[2]) for c in clean) == 2 * 48


# ---- the command ---------------------------------------------------------------------------------------------------------

def write_ffv1(path, frames):
    h, w = frames[0].shape[:2]
    vw = cv2.VideoWriter(str(path), cv2.VideoWriter_fourcc(*"FFV1"), 25, (w, h))
    assert vw.isOpened()
    for f in frames:
        vw.write(f)
    vw.release()


def read_video(path):
    cap = cv2.VideoCapture(str(path))
    out = []
    while True:
        ok, f = cap.read()
        if not ok:
            return out
        out.append(f)


def tree(root):
    out = {}
    for d, _, fs in os.walk(root):
        for f in fs:
            p = os.path.join(d, f)
            out[os.path.relpath(p, root)] = open(p, "rb").read()
    return out


def cli_main(args, **kw):
    from denseflow_b200 import cli
    lines = []
    if not kw:
        return cli.main(args, out=lines.append), lines
    cli.run(cli.parse_args(args), lines.append, **kw)
    return 0, lines


def expected_files(frames, step, save_type, bound=20, new_short=0):
    """run_videos of the decoded frames, named as the reference names them"""
    from denseflow_b200 import listrun
    r = listrun.ListRunner("tvl1", [0], 128, 96)
    try:
        files, _ = collect(lambda cb: r.run_videos([frames], step=step, bound=bound, save_type=save_type, jpeg_exact=1, new_short=new_short,
                                                   on_chunk=cb), 1, step, save_type)
    finally:
        r.close()
    n = max(len(frames) - abs(step), 0) if step else len(frames)
    return dict(zip(listrun.output_names(step, 0, n, save_type), files[0]))


def test_cli_ffv1_video_equals_run_videos(tmp_path):
    frames = bgr_frames(75, 96, 128, seed=7)  # two windows of 64 flows
    write_ffv1(tmp_path / "clip.avi", frames)
    decoded = read_video(tmp_path / "clip.avi")
    assert len(decoded) == 75 and all(np.array_equal(a, b) for a, b in zip(decoded, frames))
    rc, lines = cli_main([str(tmp_path / "clip.avi"), "-o=" + str(tmp_path / "o"), "-s=1", "-b=20"])
    assert rc == 0 and lines[-1].startswith("1 videos (75 frames, 74 tvl1 flows) processed, using "), lines
    assert tree(tmp_path / "o" / "clip") == expected_files(decoded, 1, "jpg")
    rc, _ = cli_main([str(tmp_path / "clip.avi"), "-o=" + str(tmp_path / "p"), "-s=-2", "-st=png", "-ns=64"])
    assert rc == 0 and tree(tmp_path / "p" / "clip") == expected_files(decoded, -2, "png", new_short=64)


def test_cli_list_tree_markers_skip_and_force(tmp_path):
    a, b, c = bgr_frames(9, 48, 64, seed=1), bgr_frames(5, 96, 128, seed=2), bgr_frames(7, 48, 64, seed=3)
    (tmp_path / "data" / "jump").mkdir(parents=True)
    (tmp_path / "data" / "run" / "c").mkdir(parents=True)
    (tmp_path / "data" / "run" / "empty").mkdir(parents=True)
    write_ffv1(tmp_path / "data" / "jump" / "a.avi", a)
    write_ffv1(tmp_path / "data" / "run" / "b.avi", b)
    for i, blob in enumerate(jpegs(c)):
        (tmp_path / "data" / "run" / "c" / ("img_%05d.jpg" % i)).write_bytes(blob)
    lst = tmp_path / "list.txt"
    lst.write_text("".join(str(tmp_path / "data" / p) + "\n" for p in ["jump/a.avi", "run/b.avi"]))
    lst_if = tmp_path / "frames.txt"
    lst_if.write_text("".join(str(tmp_path / "data" / p) + "\n" for p in ["run/c", "run/empty"]))
    out = tmp_path / "o"
    rc, lines = cli_main([str(lst), "-a=tvl1", "-s=1", "-b=20", "-cf", "-o=" + str(out)])
    assert rc == 0 and sorted(lines[:-1]) == ['done video "jump/a"', 'done video "run/b"'], lines
    assert lines[-1].startswith("2 videos (14 frames, 12 tvl1 flows) processed")
    rc, lines = cli_main([str(lst_if), "-a=tvl1", "-s=1", "-b=20", "-cf", "-if", "-v", "-o=" + str(out)])
    assert rc == 0 and lines[0] == '"%s" is empty!' % (tmp_path / "data" / "run" / "empty") and lines[1] == 'done video "run/c"'
    got = tree(out)
    want = {}
    for cls, stem, frames in [("jump", "a", read_video(tmp_path / "data" / "jump" / "a.avi")),
                              ("run", "b", read_video(tmp_path / "data" / "run" / "b.avi")),
                              ("run", "c", [cv2.imdecode(np.frombuffer(x, np.uint8), cv2.IMREAD_COLOR) for x in jpegs(c)])]:
        want.update({"%s/%s/%s" % (cls, stem, k): v for k, v in expected_files(frames, 1, "jpg").items()})
        want[".done/%s/%s" % (cls, stem)] = b""
    assert got == want
    assert os.path.isdir(out / "run" / "empty") and not os.path.exists(out / ".done" / "run" / "empty")
    # a second run skips every video; -f redoes them
    rc, lines = cli_main([str(lst), "-s=1", "-b=20", "-cf", "-v", "-o=" + str(out)])
    assert rc == 0 and lines == ['skip "jump/a"', 'skip "run/b"']
    os.remove(out / "jump" / "a" / "flow_x_00000.jpg")
    rc, lines = cli_main([str(lst), "-s=1", "-b=20", "-cf", "-f", "-o=" + str(out)])
    assert rc == 0 and lines[-1].startswith("2 videos") and tree(out) == got


def test_cli_extract_frames_writes_no_markers(tmp_path):
    frames = bgr_frames(70, 48, 64, seed=5)
    write_ffv1(tmp_path / "v.avi", frames)
    decoded = read_video(tmp_path / "v.avi")
    lst = tmp_path / "l.txt"
    lst.write_text(str(tmp_path / "v.avi") + "\n")
    rc, lines = cli_main([str(lst), "-o=" + str(tmp_path / "o")])
    assert rc == 0 and lines == [lines[-1]] and lines[-1].startswith("1 videos (70 frames, 0 tvl1 flows) processed")
    want = {"v/img_%05d.jpg" % i: cv2.imencode(".jpg", f, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes() for i, f in enumerate(decoded)}
    assert tree(tmp_path / "o") == want and os.listdir(tmp_path / "o" / ".done") == []


def test_cli_cannot_open_a_video(tmp_path):
    (tmp_path / "bad.avi").write_bytes(b"not a video")
    rc, lines = cli_main([str(tmp_path / "bad.avi"), "-s=1", "-o=" + str(tmp_path / "o")])
    assert rc == 1 and lines == ["cannot open video_path stream:" + str(tmp_path / "bad.avi")]


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
def test_cli_strict_equals_the_reference_pipeline(tmp_path, alg, oracle):
    """A 64x48 `-if` video in the strict build: imencode of the oracle's quantised flows (jpg) or packed flows (png)."""
    from oracle import cv_restate
    video = jpegs(bgr_frames(5, 48, 64, seed=9))
    (tmp_path / "v").mkdir()
    for i, blob in enumerate(video):
        (tmp_path / "v" / ("f%d.jpg" % i)).write_bytes(blob)
    gray = [cv2.cvtColor(cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2GRAY) for b in video]
    calc = oracle.tvl1_calc if alg == "tvl1" else oracle.farn_calc
    flows = [calc(gray[j], gray[j + 1]) for j in range(4)]
    for st in ("jpg", "png"):
        out = tmp_path / ("o_" + st)
        cli_main([str(tmp_path / "v"), "-if", "-s=1", "-b=20", "-a=" + alg, "-st=" + st, "-o=" + str(out)], variant="strict")
        got = tree(out / "v")
        if st == "jpg":
            want = {}
            for i, f in enumerate(flows):
                qx, qy = oracle.quantise(f, 20)
                want["flow_x_%05d.jpg" % i] = cv2.imencode(".jpg", qx)[1].tobytes()
                want["flow_y_%05d.jpg" % i] = cv2.imencode(".jpg", qy)[1].tobytes()
        else:
            want = {"flow_%05d.png" % i: cv2.imencode(".png", cv_restate.flow_to_png_image(f)[0])[1].tobytes() for i, f in enumerate(flows)}
        assert got == want, (alg, st)
