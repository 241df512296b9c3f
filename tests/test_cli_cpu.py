"""`python -m denseflow_b200` without a GPU: the reference's flag syntax and defaults, the output tree it plans (directories,
.done markers, skips), list and `-if` folder reading, the texts and exit codes of its failures, and what it does when no
device is visible."""
import os
import subprocess
import sys

import pytest

from denseflow_b200 import cli

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_cli(args, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, "-m", "denseflow_b200"] + args, cwd=cwd, env=env, capture_output=True, text=True)


def main(args):
    lines = []
    rc = cli.main(args, out=lines.append)
    return rc, lines


# ---- parser -----------------------------------------------------------------------------------------------------------

def test_defaults():
    o = cli.parse_args(["v.avi"])
    assert o == {"input": "v.avi", "help": False, "outputDir": ".", "algorithm": "tvl1", "step": 0, "bound": 32, "newWidth": 0,
                 "newHeight": 0, "newShort": 0, "classFolder": False, "inputFrames": False, "saveType": "jpg", "force": False,
                 "verbose": False}


def test_equals_forms_switches_and_positionals():
    o = cli.parse_args(["-o=out", "--algorithm=farn", "-s=-2", "--bound=20", "-nw=340", "--newHeight=256", "-cf", "--inputFrames",
                        "-st=png", "-f", "-v", "list.txt", "ignored.avi", "-unknown=3"])
    assert o["input"] == "list.txt" and o["outputDir"] == "out" and o["algorithm"] == "farn"
    assert (o["step"], o["bound"], o["newWidth"], o["newHeight"], o["newShort"]) == (-2, 20, 340, 256, 0)
    assert o["classFolder"] and o["inputFrames"] and o["force"] and o["verbose"] and o["saveType"] == "png"
    # long names with one dash, short names with two, as cv::CommandLineParser takes them
    o = cli.parse_args(["-outputDir=x", "--s=3", "-ns=128", "v"])
    assert (o["outputDir"], o["step"], o["newShort"]) == ("x", 3, 128)
    # integers read as a stream does: leading digits, else 0
    assert cli.parse_args(["-s=abc", "-b=7px", "v"])["step"] == 0 and cli.parse_args(["-b=7px", "v"])["bound"] == 7
    # a switch given an empty value is not set
    assert not cli.parse_args(["-cf=", "v"])["classFolder"]


@pytest.mark.parametrize("args", [[], ["-h"], ["--help", "v.avi"], ["-s=1"]])
def test_help_exits_zero(args):
    rc, lines = main(args)
    assert rc == 0 and lines[0].startswith("GPU optical flow extraction.")
    assert "--outputDir (value:.)" in lines[0] and "--saveType (value:jpg)" in lines[0]


def test_module_entry_point(tmp_path):
    r = run_cli(["-h"], tmp_path)
    assert r.returncode == 0 and "GPU optical flow extraction." in r.stdout
    r = run_cli([str(tmp_path / "missing.avi"), "-o=" + str(tmp_path / "o")], tmp_path)
    assert r.returncode == 1 and r.stdout.splitlines()[-2:] == ['"%s" does not exist!' % (tmp_path / "missing.avi"),
                                                                 "check init param error."]


# ---- paths as boost::filesystem names and prints them -------------------------------------------------------------------

def test_boost_path_helpers():
    assert cli.path_join("out", "", "v") == "out/v" and cli.path_join("out/", "v") == "out/v" and cli.path_join(".", "v") == "./v"
    assert cli.path_filename("a/b/c.avi") == "c.avi" and cli.path_filename("a/b/") == "." and cli.path_filename("c") == "c"
    assert cli.path_parent("a/b/c.avi") == "a/b" and cli.path_parent("c.avi") == "" and cli.path_parent("/c.avi") == "/"
    assert cli.path_stem("a/v.x.avi") == "v.x" and cli.path_stem("a/v") == "v" and cli.path_stem("a/.hidden") == ""
    assert cli.path_extension("l.txt") == ".txt" and cli.path_extension("f.JPG") == ".JPG" and cli.path_extension("f") == ""
    assert cli.quoted('a&b"c') == '"a&&b&"c"'


def test_summary_number_format():
    assert [cli.cpp_number(x) for x in (2.5, 1234567.0, 0.000123456789, 100.0)] == ["2.5", "1.23457e+06", "0.000123457", "100"]


# ---- the tree it plans ----------------------------------------------------------------------------------------------------

def _list(tmp_path, entries):
    lst = tmp_path / "list.txt"
    lst.write_text("".join(e + "\n" for e in entries))
    return str(lst)


def test_list_layout_markers_skip_and_force(tmp_path):
    out = str(tmp_path / "o")
    lst = _list(tmp_path, ["data/jump/v_1.avi", "data/run/v_2.mp4", "plain.avi"])
    opt = cli.parse_args([lst, "-o=" + out, "-cf", "-v"])
    videos, dirs, record = cli.plan(opt)
    assert record and videos == ["data/jump/v_1.avi", "data/run/v_2.mp4", "plain.avi"]
    assert dirs == [out + "/jump/v_1", out + "/run/v_2", out + "/plain"]
    for d in dirs + [out + "/.done/jump", out + "/.done/run", out + "/.done"]:
        assert os.path.isdir(d), d
    # the marker a finished video gets, and its title
    assert cli.marker(dirs[0], True) == (out + "/.done/jump/v_1", "jump/v_1")
    assert cli.marker(out + "/v_1", False) == (out + "/.done/v_1", "v_1")
    open(out + "/.done/jump/v_1", "w").close()
    said = []
    videos, dirs, _ = cli.plan(opt, said.append)
    assert videos == ["data/run/v_2.mp4", "plain.avi"] and said == ['skip "jump/v_1"']
    videos, _, _ = cli.plan(cli.parse_args([lst, "-o=" + out, "-cf", "-f"]))
    assert len(videos) == 3
    # without -cf: <o>/<stem>, markers in <o>/.done; the skip line still names the class
    out2 = str(tmp_path / "o2")
    opt = cli.parse_args([lst, "-o=" + out2, "-v"])
    _, dirs, _ = cli.plan(opt)
    assert dirs == [out2 + "/v_1", out2 + "/v_2", out2 + "/plain"] and os.path.isdir(out2 + "/.done")
    open(out2 + "/.done/v_2", "w").close()
    said = []
    assert cli.plan(opt, said.append)[0] == ["data/jump/v_1.avi", "plain.avi"] and said == ['skip "run/v_2"']


def test_single_input_layout(tmp_path):
    out = str(tmp_path / "o")
    videos, dirs, record = cli.plan(cli.parse_args(["/x/y/clip.avi", "-o=" + out, "-cf"]))
    assert (videos, dirs, record) == (["/x/y/clip.avi"], [out + "/clip"], False)
    assert os.path.isdir(out + "/clip") and not os.path.exists(out + "/.done")


def test_list_reading(tmp_path):
    p = tmp_path / "l.txt"
    p.write_bytes(b"a.avi\nb c.avi\n\nd.avi")
    assert cli.read_list(str(p)) == ["a.avi", "b c.avi", "", "d.avi"]
    assert cli.read_list(str(tmp_path / "missing.txt")) == []


def test_frame_folder_listing(tmp_path):
    d = tmp_path / "frames"
    d.mkdir()
    for name in ["img_10.jpg", "img_02.jpg", "a.jpeg", "b.JPG", "c.png", "img_01.jpg.bak"]:
        (d / name).write_bytes(b"x")
    (d / "sub.jpg").mkdir()
    (d / "sub.jpg" / "img_00.jpg").write_bytes(b"x")
    assert cli.frame_files(str(d)) == [str(d / "img_02.jpg"), str(d / "img_10.jpg")]


# ---- failures ------------------------------------------------------------------------------------------------------------

@pytest.fixture
def video(tmp_path):
    p = tmp_path / "v.avi"
    p.write_bytes(b"not decoded before the checks")
    return str(p)


@pytest.mark.parametrize("args,text", [
    (["-b=0"], "bound should > 0!"),
    (["-a=lk"], "lk not supported!"),
    (["-nw=-1"], "height and width cannot < 0!"),
    (["-ns=128", "-nw=64"], "do not set height and width when set short!"),
    (["-st=bmp"], "only jpg/png/h5 are supported (no bmp) for output"),
])
def test_check_param_failures(tmp_path, video, args, text):
    rc, lines = main([video, "-o=" + str(tmp_path / "o"), "-s=1"] + args)
    assert rc == 1 and lines == [text, "check init param error."]


def test_missing_inputs(tmp_path):
    out = str(tmp_path / "o")
    rc, lines = main([str(tmp_path / "gone.avi"), "-o=" + out])
    assert rc == 1 and lines == ['"%s" does not exist!' % (tmp_path / "gone.avi"), "check init param error."]
    lst = _list(tmp_path, [str(tmp_path / "gone.avi")])
    rc, lines = main([lst, "-o=" + out, "-s=1"])
    assert rc == 1 and lines[0] == '"%s" does not exist!' % (tmp_path / "gone.avi")
    # a list that cannot be read is an empty list: nothing to do, no summary
    assert main([str(tmp_path / "missing.txt"), "-o=" + out]) == (0, [])


@pytest.mark.parametrize("args,text", [
    (["-s=1", "-st=h5"], "HDF5 support is not enabled, pls recompile"),
    (["-s=1", "-a=nv"], "NV hardware flow not enabled, pls recompile"),
    (["-s=1", "-a=brox"], "brox is not supported in this build (tvl1 | farn)"),
])
def test_unsupported_modes(tmp_path, video, args, text):
    rc, lines = main([video, "-o=" + str(tmp_path / "o")] + args)
    assert rc == 1 and lines == [text]


def test_every_video_already_done_needs_no_device(tmp_path, video):
    out = str(tmp_path / "o")
    os.makedirs(out + "/.done")
    open(out + "/.done/v", "w").close()
    assert main([_list(tmp_path, [video]), "-o=" + out, "-s=1", "-v"]) == (0, ['skip "%s"' % cli.path_join(tmp_path.name, "v")])


def test_without_a_device(tmp_path, video):
    from denseflow_b200 import _lib
    if _lib.load().dfb_device_count() > 0:
        pytest.skip("a CUDA device is visible")
    for args in (["-s=1"], ["-s=0"], ["-s=1", "-if"]):
        src = video if "-if" not in args else str(tmp_path)
        rc, lines = main([src, "-o=" + str(tmp_path / "o")] + args)
        assert rc == 1 and lines == ["no CUDA device available (the engine has no CPU path)"]
