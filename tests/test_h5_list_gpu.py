"""-st=h5 through the list runner and the command on the GPU: DFB_SAVE_H5 hands every video the single-handle chain's float
planes, and `python -m denseflow_b200 ... -st=h5` with the hdf5 library writes writeHDF5's file, read back with tests/h5_read.py."""
import os
import threading

import cv2
import numpy as np
import pytest

import h5_read
import jpeg_cases as J
from test_cli_gpu import bgr_frames, cli_main, read_video, write_ffv1

pytestmark = pytest.mark.gpu


def _planes_single(frames, step, new_short=0, alg="tvl1", variant="default"):
    """the single-handle chain: process_{bgr,jpeg}_batch_planes of the whole video"""
    import denseflow_b200 as d
    e = d.create(alg, 0, 128, 96, variant=variant)
    try:
        if not frames:
            return np.empty((0, 2, 0, 0), np.float32)
        jpeg = isinstance(frames[0], (bytes, bytearray))
        from denseflow_b200 import api
        if jpeg:
            w, h = api.jpeg_info(frames[0])
        else:
            h, w = frames[0].shape[:2]
        dw, dh = api.new_size(w, h, 0, 0, new_short)
        ns = (dw, dh) if (dw, dh) != (w, h) else None
        return e.process_jpeg_batch_planes(frames, step, ns) if jpeg else e.process_bgr_batch_planes(frames, step, ns)
    finally:
        e.release()


def _videos():
    jp = [J.encode(f, "420", 95) for f in bgr_frames(9, 48, 64, seed=4)]
    return [bgr_frames(11, 96, 128, seed=1), jp, bgr_frames(1, 48, 64, seed=2), [], bgr_frames(7, 48, 64, seed=3), jp[:6]]


@pytest.mark.parametrize("stream", [False, True])
@pytest.mark.parametrize("step,new_short", [(1, 0), (-3, 0), (3, 40)])
def test_list_runner_h5_equals_the_single_handle_chain(stream, step, new_short):
    from denseflow_b200 import listrun
    videos = _videos()
    got = {i: {} for i in range(len(videos))}
    last = {i: 0 for i in range(len(videos))}
    lock = threading.Lock()

    def on_chunk(video, dev, first, is_last, files):
        with lock:
            assert len(files) % 2 == 0
            for k, f in enumerate(files):
                got[video][2 * first + k] = bytes(f)
            last[video] += bool(is_last)

    r = listrun.ListRunner("tvl1", [0, 0, 0], 128, 96)
    try:
        if stream:
            r.run_stream(len(videos), lambda v, first, n: videos[v][first:first + n], on_chunk, step=step, bound=20, save_type="h5",
                         new_short=new_short, chunk_flows=4)
        else:
            r.run_videos(videos, step=step, bound=20, save_type="h5", new_short=new_short, chunk_flows=4, on_chunk=on_chunk)
    finally:
        r.close()
    assert all(last[i] == 1 for i in range(len(videos))), last
    for i, v in enumerate(videos):
        want = _planes_single(v, step, new_short)
        files = [got[i][k] for k in range(len(got[i]))]
        assert len(files) == 2 * want.shape[0]
        for j in range(want.shape[0]):
            assert files[2 * j] == want[j, 0].tobytes() and files[2 * j + 1] == want[j, 1].tobytes(), (i, j)
            assert len(files[2 * j]) == 4 * want.shape[2] * want.shape[3]


def _datasets(path):
    r = h5_read.H5File(str(path))
    assert r.eof == os.path.getsize(path)
    return {n: r.read(n) for n in r.names}


def _want(planes, step):
    from denseflow_b200 import listrun
    names = listrun.h5_names(step, 0, planes.shape[0])
    m = planes.shape[0]
    return {names[j].lstrip("/"): planes[j, 0] for j in range(m)} | {names[m + j].lstrip("/"): planes[j, 1] for j in range(m)}


def _same(got, want):
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].dtype == np.float32 and got[k].tobytes() == want[k].tobytes(), k


@pytest.mark.parametrize("step", [1, 3, -1])
def test_cli_h5_files(tmp_path, step):
    a = bgr_frames(75, 96, 128, seed=7)  # two windows of 64 flows
    c = [J.encode(f, "420", 95) for f in bgr_frames(7, 48, 64, seed=3)]
    (tmp_path / "data" / "jump").mkdir(parents=True)
    (tmp_path / "data" / "run" / "c").mkdir(parents=True)
    (tmp_path / "data" / "run" / "empty").mkdir(parents=True)
    write_ffv1(tmp_path / "data" / "jump" / "a.avi", a)
    for i, blob in enumerate(c):
        (tmp_path / "data" / "run" / "c" / ("img_%05d.jpg" % i)).write_bytes(blob)
    (tmp_path / "v.txt").write_text(str(tmp_path / "data" / "jump" / "a.avi") + "\n")
    (tmp_path / "f.txt").write_text("".join(str(tmp_path / "data" / p) + "\n" for p in ["run/c", "run/empty"]))
    out = tmp_path / "o"
    from denseflow_b200 import listrun
    rc, lines = cli_main([str(tmp_path / "v.txt"), "-s=%d" % step, "-b=20", "-st=h5", "-cf", "-o=" + str(out)], variant="hdf5")
    assert lines[0] == 'done video "jump/a"' and lines[-1].startswith("1 videos (75 frames, %d tvl1 flows)" % (75 - abs(step)))
    rc, lines = cli_main([str(tmp_path / "f.txt"), "-s=%d" % step, "-b=20", "-st=h5", "-cf", "-if", "-o=" + str(out)], variant="hdf5")
    assert lines[0] == 'done video "run/c"'
    pa, pc, pe = (listrun.h5_path(str(out / p), step) for p in ("jump/a", "run/c", "run/empty"))
    _same(_datasets(pa), _want(_planes_single(read_video(tmp_path / "data" / "jump" / "a.avi"), step), step))
    _same(_datasets(pc), _want(_planes_single(c, step), step))
    assert _datasets(pe) == {} and not os.path.exists(out / ".done" / "run" / "empty")
    assert os.path.isfile(out / ".done" / "jump" / "a") and os.path.isfile(out / ".done" / "run" / "c")
    assert os.listdir(out / "jump" / "a") == [] and os.listdir(out / "run" / "c") == []
    # .done: a second run skips the video and does not touch its file; -f writes it again
    before = open(pa, "rb").read()
    rc, lines = cli_main([str(tmp_path / "v.txt"), "-s=%d" % step, "-st=h5", "-cf", "-v", "-o=" + str(out)], variant="hdf5")
    assert lines == ['skip "jump/a"'] and open(pa, "rb").read() == before
    rc, lines = cli_main([str(tmp_path / "v.txt"), "-s=%d" % step, "-st=h5", "-cf", "-f", "-b=20", "-o=" + str(out)], variant="hdf5")
    assert open(pa, "rb").read() == before


def test_cli_h5_single_video_and_the_default_library(tmp_path):
    frames = bgr_frames(5, 48, 64, seed=5)
    write_ffv1(tmp_path / "clip.avi", frames)
    rc, lines = cli_main([str(tmp_path / "clip.avi"), "-s=1", "-st=h5", "-o=" + str(tmp_path / "o")], variant="hdf5")
    _same(_datasets(tmp_path / "o" / "clip.h5"), _want(_planes_single(read_video(tmp_path / "clip.avi"), 1), 1))
    assert os.listdir(tmp_path / "o" / "clip") == []
    rc, lines = cli_main([str(tmp_path / "clip.avi"), "-s=1", "-st=h5", "-o=" + str(tmp_path / "p")])
    assert rc == 1 and lines == ["HDF5 support is not enabled, pls recompile"]


@pytest.mark.parametrize("alg", ["tvl1", "farn"])
def test_cli_h5_strict_against_the_oracle(tmp_path, alg, oracle):
    from denseflow_b200 import synth
    video = [J.encode(f, "420", 95) for f in bgr_frames(5, 48, 64, seed=9)]
    (tmp_path / "v").mkdir()
    for i, blob in enumerate(video):
        (tmp_path / "v" / ("f%d.jpg" % i)).write_bytes(blob)
    gray = [cv2.cvtColor(cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2GRAY) for b in video]
    calc = oracle.tvl1_calc if alg == "tvl1" else oracle.farn_calc
    cli_main([str(tmp_path / "v"), "-if", "-s=1", "-b=20", "-a=" + alg, "-st=h5", "-o=" + str(tmp_path / "o")], variant="strict_hdf5")
    got = _datasets(tmp_path / "o" / "v.h5")
    assert sorted(got) == ["flow_x_%05d" % j for j in range(4)] + ["flow_y_%05d" % j for j in range(4)]
    planes = _planes_single(video, 1, alg=alg, variant="strict_hdf5")
    for j in range(4):
        assert got["flow_x_%05d" % j].tobytes() == planes[j, 0].tobytes()
        assert got["flow_y_%05d" % j].tobytes() == planes[j, 1].tobytes()
        ref = calc(gray[j], gray[j + 1])
        assert synth.aee(np.stack([got["flow_x_%05d" % j], got["flow_y_%05d" % j]], -1), ref) <= (1e-3 if alg == "tvl1" else 1e-4)
