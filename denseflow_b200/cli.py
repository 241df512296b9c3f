"""`python -m denseflow_b200`: the reference's `denseflow` command (tools/denseflow.cpp, SURVEY §3.4) on the GPU list runner.

    python -m denseflow_b200 videolist.txt -b=20 -a=tvl1 -s=1 -cf -v

takes the reference's flags and writes its file tree: `<o>/[<class>/]<stem>/flow_x_00000.jpg ...` (or `flow_*.png`, or with
-s=0 `img_*.jpg`), and for a list in flow mode one `<o>/.done/[<class>/]<stem>` marker per finished video, which a later run
skips unless -f is given.  Videos are decoded with cv2.VideoCapture on the worker threads, one window of frames at a time,
so a list of long videos runs in bounded memory; `-if` folders go to the GPU as JPEG bytes and are decoded there.  Every
visible GPU runs two workers.  Each takes whole videos while the list lasts; then idle workers join the unfinished videos
window by window, so a single video or `-if` folder runs on every worker, one reading its next window while another
computes.  Errors print their message and exit 1, as the reference's main() does.

`-st=h5` in flow mode needs the library built with HDF5 support, the counterpart of the reference's -DUSE_HDF5=yes build:
`DFB_LIBRARY=hdf5 python -m denseflow_b200 ...` writes each video's flows as float32 datasets /flow_x_%05d and /flow_y_%05d to
`<output dir>.h5` (`_p<s>` / `_m<|s|>` before `.h5` for other steps).  The default library refuses it with the reference's
"HDF5 support is not enabled, pls recompile".
"""
import os
import re
import sys
import threading
import time

# tools/denseflow.cpp's keys: (names, default, help); a switch has no default
KEYS = [
    (("h", "help"), None, "print help message"),
    (("o", "outputDir"), ".", "root dir of output"),
    (("a", "algorithm"), "tvl1", "optical flow algorithm (nv/tvl1/farn/brox)"),
    (("s", "step"), "0", "right - left (0 for img, non-0 for flow)"),
    (("b", "bound"), "32", "maximum of optical flow"),
    (("nw", "newWidth"), "0", "new width"),
    (("nh", "newHeight"), "0", "new height"),
    (("ns", "newShort"), "0", "short side length"),
    (("cf", "classFolder"), None, "outputDir/class/video/flow.jpg"),
    (("if", "inputFrames"), None, "inputs are frames"),
    (("st", "saveType"), "jpg", "save format type (png/h5/jpg)"),
    (("f", "force"), None, "regardless of the marked .done file"),
    (("v", "verbose"), None, "verbose"),
]
INPUT_HELP = "filename of video or folder of frames or a list.txt of those"
WORKERS_PER_DEVICE = 2
CHUNK_FLOWS = 64


class CliError(Exception):
    """A failure the command reports as its message and exit code 1."""


def _print(text):
    print(text, flush=True)


# ---- cv::CommandLineParser ---------------------------------------------------------------------------------------------

def _cpp_int(text):
    """`std::stringstream >> int`: leading digits count, anything else reads as 0 (cv::CommandLineParser::get<int>)."""
    m = re.match(r"\s*([+-]?\d+)", text)
    return int(m.group(1)) if m else 0


def parse_args(argv):
    """cv::CommandLineParser over KEYS: `-k=v` or `--key=v`, a bare `-k` sets "true", the first token without a leading dash
    is the input and later ones are ignored, unknown keys are ignored.  Returns a dict keyed by the long names plus "input"."""
    raw = {names[1]: ("" if default is None else default) for names, default, _ in KEYS}
    positional = []
    for s in argv:
        if len(s) > 1 and s[0] == "-":
            key, eq, value = s[2 if len(s) > 2 and s[1] == "-" else 1:].partition("=")
            for names, _, _ in KEYS:
                if key in names:
                    raw[names[1]] = value if eq else "true"
        else:
            positional.append(s)

    def has(name):
        v = raw[name].strip()
        return v != "" and v != "<none>"

    return {"input": positional[0].strip() if positional else "", "help": has("help"), "outputDir": raw["outputDir"].strip(),
            "algorithm": raw["algorithm"].strip(), "step": _cpp_int(raw["step"]), "bound": _cpp_int(raw["bound"]),
            "newWidth": _cpp_int(raw["newWidth"]), "newHeight": _cpp_int(raw["newHeight"]), "newShort": _cpp_int(raw["newShort"]),
            "classFolder": has("classFolder"), "inputFrames": has("inputFrames"), "saveType": raw["saveType"].strip(),
            "force": has("force"), "verbose": has("verbose")}


def help_text():
    lines = ["GPU optical flow extraction.", "Usage: python -m denseflow_b200 [params] input", ""]
    for names, default, text in sorted(KEYS, key=lambda k: k[0][0]):
        lines.append("\t-%s, --%s%s" % (names[0], names[1], "" if default is None else " (value:%s)" % default))
        lines.append("\t\t" + text)
    lines += ["", "\tinput", "\t\t" + INPUT_HELP]
    return "\n".join(lines)


# ---- boost::filesystem::path (v3), as the reference names directories and prints paths ---------------------------------

def path_join(*parts):
    """operator/: empty parts add nothing; no separator is added next to one that is there."""
    out = ""
    for p in parts:
        if not p:
            continue
        out = p if not out else out + p if out.endswith("/") or p.startswith("/") else out + "/" + p
    return out


def path_filename(p):
    """filename(): the last element; "." for a path that ends in a separator (boost v3)."""
    if not p:
        return ""
    if p.endswith("/"):
        return "/" if p.strip("/") == "" else "."
    return p.rsplit("/", 1)[-1]


def path_parent(p):
    """parent_path(): everything before the last element."""
    if "/" not in p:
        return ""
    head = p.rsplit("/", 1)[0]
    return head.rstrip("/") or "/"


def path_stem(p):
    """stem() of the filename: "." and ".." stay, otherwise everything before the last dot (".bashrc" has an empty stem)."""
    name = path_filename(p)
    if name in (".", ".."):
        return name
    return name[:name.rfind(".")] if "." in name else name


def path_extension(p):
    name = path_filename(p)
    if name in (".", "..") or "." not in name:
        return ""
    return name[name.rfind("."):]


def quoted(p):
    """operator<<(ostream, path): boost::io::quoted with '&' as the escape character."""
    return '"' + p.replace("&", "&&").replace('"', '&"') + '"'


# ---- the list ------------------------------------------------------------------------------------------------------------

def read_list(path):
    """std::getline over list.txt: one path per line, a last empty line is no entry; a file that cannot be read is empty."""
    try:
        with open(path, "rb") as f:
            data = f.read()
    except OSError:
        return []
    lines = data.split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()
    return [os.fsdecode(x) for x in lines]


def frame_files(folder):
    """An `-if` folder's frames: regular files whose extension is exactly ".jpg", sorted by path."""
    out = []
    for e in os.scandir(folder):
        p = path_join(folder, e.name)
        if e.is_file() and path_extension(p) == ".jpg":
            out.append(p)
    return sorted(out)


def plan(opt, out=_print):
    """tools/denseflow.cpp:51-87: the videos to process and their output directories, which are created.  A list entry whose
    .done marker exists is skipped unless -f is given.  Returns (videos, output_dirs, is_record)."""
    src, odir = opt["input"], opt["outputDir"]
    videos, outdirs = [], []
    if path_extension(src) == ".txt":
        for vid in read_list(src):
            cls, stem = path_filename(path_parent(vid)), path_stem(vid)
            if opt["classFolder"]:
                outdir, donedir = path_join(odir, cls, stem), path_join(odir, ".done", cls)
            else:
                outdir, donedir = path_join(odir, stem), path_join(odir, ".done")
            if not opt["force"] and os.path.isfile(path_join(donedir, stem)):
                if opt["verbose"]:
                    out("skip " + quoted(path_join(cls, stem)))
                continue
            os.makedirs(outdir, exist_ok=True)
            os.makedirs(donedir, exist_ok=True)
            videos.append(vid)
            outdirs.append(outdir)
        return videos, outdirs, True
    outdir = path_join(odir, path_stem(src))
    os.makedirs(outdir, exist_ok=True)
    return [src], [outdir], False


def check_param(opt, videos, outdirs):
    """DenseFlow::check_param (src/denseflow_gpu.cpp:9-42): the first failure's text, or None."""
    for v, d in zip(videos, outdirs):
        if not os.path.exists(v):
            return quoted(v) + " does not exist!"
        if not os.path.isdir(d):
            return quoted(d) + " is not a valid dir!"
    if opt["algorithm"] not in ("nv", "tvl1", "farn", "brox"):
        return opt["algorithm"] + " not supported!"
    if opt["bound"] <= 0:
        return "bound should > 0!"
    if opt["newHeight"] < 0 or opt["newWidth"] < 0 or opt["newShort"] < 0:
        return "height and width cannot < 0!"
    if opt["newShort"] > 0 and opt["newHeight"] + opt["newWidth"] != 0:
        return "do not set height and width when set short!"
    if opt["saveType"] not in ("jpg", "png", "h5"):
        return "only jpg/png/h5 are supported (no %s) for output" % opt["saveType"]
    return None


def marker(outdir, has_class):
    """The .done file and the title encode_save gives a finished video (src/denseflow_gpu.cpp:456-470), both taken from its
    output directory: the marker is named by that directory's stem."""
    parent = path_parent(outdir)
    if has_class:
        donedir = path_join(path_parent(parent), ".done", path_filename(parent))
        title = path_join(path_filename(parent), path_filename(outdir))
    else:
        donedir, title = path_join(parent, ".done"), path_filename(outdir)
    return path_join(donedir, path_stem(outdir)), title


def cpp_number(x):
    """A double through std::ostream's default format."""
    return "%g" % x


def _per_second(count, seconds):
    """count / seconds as a double division: inf, or nan for 0 / 0, when no time has passed."""
    return count / seconds if seconds else float("nan") if count == 0 else float("inf")


# ---- frame sources -------------------------------------------------------------------------------------------------------

class VideoReader:
    """A video read in order with cv2.VideoCapture; a window reuses the frames of the previous one it overlaps."""

    def __init__(self, path):
        import cv2
        self.cap = cv2.VideoCapture(path)
        if not self.cap.isOpened():
            raise CliError("cannot open video_path stream:" + path)
        self.base, self.held = 0, []

    def window(self, first, max_n):
        self.held = self.held[first - self.base:]
        self.base = first
        while self.cap is not None and len(self.held) < max_n:
            ok, frame = self.cap.read()
            if not ok or frame is None:
                self.close()
                break
            self.held.append(frame)
        return list(self.held)

    def close(self):
        if self.cap is not None:
            self.cap.release()
            self.cap = None


class FolderReader:
    """An `-if` folder: each window is its files' bytes, decoded on the GPU."""

    def __init__(self, files):
        self.files = files

    def window(self, first, max_n):
        out = []
        for p in self.files[first:first + max_n]:
            with open(p, "rb") as f:
                out.append(f.read())
        return out

    def close(self):
        pass


# ---- the command ---------------------------------------------------------------------------------------------------------

def _unsupported_algorithm(L, algorithm):
    """The library's refusal of an algorithm it does not build (nv, brox), or None."""
    import ctypes as C
    from . import _lib
    if algorithm in ("tvl1", "farn"):
        return None
    h = C.c_void_p()
    rc = L.dfb_create(algorithm.encode(), 0, 64, 64, C.byref(h))
    if rc == _lib.DFB_OK:
        L.dfb_destroy(h)
        return None
    return L.dfb_last_error(None).decode()


def _unsupported_h5(L):
    """The library's refusal of -st=h5 when it is built without HDF5 support, or None.  A null path is refused before any
    file is touched by a library that has the writer."""
    import ctypes as C
    from . import _lib
    f = C.c_void_p()
    if L.dfb_h5_create(None, C.byref(f)) == _lib.DFB_ERR_UNSUPPORTED:
        return L.dfb_last_error(None).decode()
    return None


def run(opt, out=_print, variant="default"):
    """calcDenseFlowVideoGPU (src/denseflow_gpu.cpp:479-497) for the planned videos on every visible GPU, with the library
    `variant` (the command uses $DFB_LIBRARY, default "default")."""
    from . import _lib, listrun
    videos, outdirs, is_record = plan(opt, out)
    if not videos:
        return
    msg = check_param(opt, videos, outdirs)
    if msg is not None:
        out(msg)
        raise CliError("check init param error.")
    step, save_type, verbose = opt["step"], opt["saveType"], opt["verbose"]
    L = _lib.load(variant)
    h5_out = step != 0 and save_type == "h5"
    if h5_out:
        refusal = _unsupported_h5(L)
        if refusal:
            raise CliError(refusal)
    if step != 0:
        refusal = _unsupported_algorithm(L, opt["algorithm"])
        if refusal:
            raise CliError(refusal)
    n_dev = L.dfb_device_count()
    if n_dev <= 0:
        raise CliError("no CUDA device available (the engine has no CPU path)")
    # -s=0 computes no flow, so its workers may hold any engine the library builds (extract_frames_only creates none)
    algorithm = opt["algorithm"] if opt["algorithm"] in ("tvl1", "farn") else "tvl1"
    lock = threading.Lock()

    def say(text):
        with lock:
            out(text)

    # `-if` folders are listed up front: an empty one is skipped without a marker
    jobs = []
    for vid, outdir in zip(videos, outdirs):
        if opt["inputFrames"]:
            files = frame_files(vid)
            if not files:
                if verbose:
                    say(quoted(vid) + " is empty!")
                if h5_out:  # the reference creates the file before it finds no frame, and closes it empty (no marker)
                    from . import h5
                    h5.File(listrun.h5_path(outdir, step), variant=variant).close()
                continue
            jobs.append((vid, outdir, files))
        else:
            jobs.append((vid, outdir, None))
    return _run_jobs(opt, algorithm, n_dev, jobs, len(videos), is_record, say, variant)


def _source_message(error, failures):
    """The command's message for a failed run: the source exception the runner reported ("video k: <message>") as its own
    text, as the reference prints it; any other error as it is.  A source call that failed after an earlier window of its
    video had failed is not the reported error."""
    for video, ex in failures:
        prefix = "video %d: " % video
        text = str(ex) or type(ex).__name__
        if error.startswith(prefix) and text.startswith(error[len(prefix):]):
            return str(ex)
    return error


def _run_jobs(opt, algorithm, n_dev, jobs, n_listed, is_record, say, variant):
    """The non-empty inputs through ListRunner.run_windows: files into each output directory, then the summary line.

    Once the list is handed out, idle workers join the unfinished videos, so `source` may be called for one video from several
    threads, but one call at a time and in frame order, and each window's on_chunk comes after its source call and after the
    video's earlier chunks.  So a video's reader is only touched by one call at a time, its size is recorded by its first
    window before any chunk needs it, and its h5 file is created by its first window and written in dataset order."""
    from . import _lib, listrun
    import numpy as np
    from . import api, h5
    step, save_type = opt["step"], opt["saveType"]
    h5_out = step != 0 and save_type == "h5"
    readers = {}
    h5_files = {}  # video -> its open h5 file, from the video's start to its last chunk
    sizes = {}     # video -> (dh, dw), the size of its flows
    failures = []  # (video, exception) of the source

    def source(video, first, max_n):
        try:
            if first == 0:
                vid, outdir, files = jobs[video]
                if h5_out:  # created (or truncated) before the first frame is decoded
                    h5_files[video] = h5.File(listrun.h5_path(outdir, step), variant=variant)
                readers[video] = FolderReader(files) if files is not None else VideoReader(vid)
            frames = readers[video].window(first, max_n)
            if h5_out and video not in sizes and frames:
                f0 = frames[0]
                sw, sh = (f0.shape[1], f0.shape[0]) if hasattr(f0, "shape") else api.jpeg_info(f0, variant)
                dw, dh = api.new_size(sw, sh, opt["newWidth"], opt["newHeight"], opt["newShort"], variant)
                sizes[video] = (dh, dw)
            if len(frames) < max_n:
                readers.pop(video).close()
            return frames
        except Exception as ex:
            failures.append((video, ex))
            raise

    def on_chunk(video, dev, first, last, files):
        outdir = jobs[video][1]
        if h5_out:
            # writeHDF5's order: every x of the chunk, then every y (files 2 i / 2 i + 1 are flow i's x / y plane)
            n = len(files) // 2
            f = h5_files[video]
            for name, k in zip(listrun.h5_names(step, first, n), [2 * i for i in range(n)] + [2 * i + 1 for i in range(n)]):
                f.write_float(name, np.frombuffer(files[k], np.float32).reshape(sizes[video]))
            if last:
                h5_files.pop(video).close()  # before the marker
                if is_record:
                    done_file, title = marker(outdir, opt["classFolder"])
                    open(done_file, "wb").close()
                    say("done video " + quoted(title))
            return
        for name, data in zip(listrun.output_names(step, first, len(files) // (2 if step != 0 and save_type == "jpg" else 1), save_type),
                              files):
            with open(path_join(outdir, name), "wb") as f:
                f.write(data)
        if last and is_record and step != 0:
            done_file, title = marker(outdir, opt["classFolder"])
            open(done_file, "wb").close()
            say("done video " + quoted(title))

    t0 = time.time()  # CurrentSeconds() is read once the parameters are checked
    st = {"frames": 0, "flows": 0}
    if jobs:
        devices = [d for d in range(n_dev) for _ in range(WORKERS_PER_DEVICE)][:_lib.LIST_MAX_WORKERS]
        r = listrun.ListRunner(algorithm, devices, 64, 64, variant=variant)
        try:
            st = r.run_windows(len(jobs), source, on_chunk, step=step, bound=opt["bound"], save_type=save_type if step != 0 else "jpg",
                               quality=95, jpeg_exact=1, new_width=opt["newWidth"], new_height=opt["newHeight"],
                               new_short=opt["newShort"], chunk_flows=CHUNK_FLOWS)
        except RuntimeError as ex:
            raise CliError(_source_message(str(ex), failures)) from None
        finally:
            r.close()
            for rd in readers.values():
                rd.close()
            for f in h5_files.values():  # a failed video's file keeps what was written before the failure; it gets no marker
                f.close()
    t = time.time() - t0
    n, f = st["frames"], st["flows"]
    say("%d videos (%d frames, %d %s flows) processed, using %ss, decoding speed %sfps, flow speed %sfps"
        % (n_listed, n, f, opt["algorithm"], cpp_number(t), cpp_number(_per_second(n, t)), cpp_number(_per_second(f, t))))
    return st


def main(argv=None, out=_print):
    """The command: exit code 0, or 1 after printing the failure (tools/denseflow.cpp:93-96)."""
    opt = parse_args(sys.argv[1:] if argv is None else argv)
    if opt["input"] == "" or opt["help"]:
        out(help_text())
        return 0
    try:
        variant = os.environ.get("DFB_LIBRARY", "default")
        from . import _lib
        if variant not in _lib.LIB_PATHS:
            raise CliError("unknown DFB_LIBRARY %s (%s)" % (variant, " | ".join(sorted(_lib.LIB_PATHS))))
        run(opt, out, variant=variant)
    except (CliError, OSError, RuntimeError) as ex:
        out(str(ex))
        return 1
    return 0
