"""The -st=h5 file writer (dfb_h5_*, denseflow_b200.h5) without a GPU: its files read back through tests/h5_read.py, a reader
written from the HDF5 format and checked here against a file libhdf5 wrote; the default library refuses as the reference's
build without HDF5 does."""
import ctypes as C
import os

import numpy as np
import pytest

import h5_read

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
NODE_BYTES, SNOD_BYTES = 24 + 33 * 8 + 32 * 8, 8 + 8 * 40


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from denseflow_b200 import _lib
    return _lib


def _write(path, items):
    from denseflow_b200 import h5
    with h5.File(path, variant="hdf5") as f:
        for name, a in items:
            f.write_float(name, a)
    return h5_read.H5File(path)


def _reference_names(n, step=1, first=0):
    """the datasets of one video in the order writeHDF5 makes them: every x of a chunk, then every y"""
    return [("/flow_x_%05d" % (first + i), "x") for i in range(n)] + [("/flow_y_%05d" % (first + i), "y") for i in range(n)]


def _check_structure(r, size):
    assert r.eof == size
    assert all(a < size for a in r.addresses())
    assert r.heap_free == 1  # no free block: the list ends at once
    # keys: sorted, key i = the last name below child i - 1, and the leaf entries in strcmp order
    enc = [n.encode() for n in r.names]
    assert enc == sorted(enc)
    for n in r.nodes:
        assert len(n.keys) == n.entries + 1
        ks = [k.encode() for k in n.keys]
        assert ks == sorted(ks)
    # every node and SNOD owns its full 2K allocation: no block starts inside another
    blocks = sorted([(n.addr, NODE_BYTES) for n in r.nodes] + [(a, SNOD_BYTES) for a, _ in r.snods])
    for (a, n), (b, _) in zip(blocks, blocks[1:]):
        assert a + n <= b
    assert blocks[-1][0] + blocks[-1][1] <= size
    assert all(s <= 8 for _, s in r.snods)
    # libhdf5 finds a name by descending through the keys: every name resolves, names between and beyond them do not
    for nm in r.names:
        assert r.lookup(nm) is not None, nm
    for nm in r.names[::max(1, len(r.names) // 50)]:
        assert r.lookup(nm + "!") is None and r.lookup(nm[:-1]) is None
    assert r.lookup("") is None and r.lookup("\x7f") is None


def test_reader_against_a_libhdf5_file():
    """scipy's testhdf5_7.4_GLNX86.mat: written by libhdf5 behind a 512-byte user block"""
    import scipy.io
    r = h5_read.H5File(os.path.join(GOLDEN, "testhdf5_7.4_GLNX86.mat"))
    assert r.base == 0x200 and r.eof == os.path.getsize(os.path.join(GOLDEN, "testhdf5_7.4_GLNX86.mat"))
    assert r.names == ["testdouble"]
    want = scipy.io.loadmat(os.path.join(GOLDEN, "testdouble_7.4_GLNX86.mat"))["testdouble"]
    got = r.read("testdouble")
    assert got.dtype == np.float64 and got.shape == (9, 1)
    np.testing.assert_array_equal(got.T, want)
    np.testing.assert_allclose(got.ravel(), np.linspace(0, 2 * np.pi, 9), rtol=0, atol=1e-15)
    # the two facts the writer takes from libhdf5: a free list ends with the value 1, and key i is the last name of child i - 1
    seg = r._at(r.heap_data, r.heap_size)
    assert int.from_bytes(seg[r.heap_free:r.heap_free + 8], "little") == 1
    (root,) = r.nodes
    assert root.keys == ["", "testdouble"]
    assert r.lookup("testdouble") is not None
    assert r.lookup("testdoublf") is None


@pytest.mark.parametrize("n", [0, 1, 8, 9, 256, 257])
def test_dataset_counts(lib, tmp_path, n):
    rng = np.random.default_rng(n)
    items = []
    for name, c in _reference_names((n + 1) // 2)[:n]:
        items.append((name, rng.standard_normal((3, 5)).astype(np.float32)))
    path = str(tmp_path / "f.h5")
    r = _write(path, items)
    assert sorted(r.names) == sorted(nm.lstrip("/") for nm, _ in items)
    for name, a in items:
        got = r.read(name.lstrip("/"))
        assert got.dtype == np.float32 and got.shape == a.shape
        assert got.tobytes() == a.tobytes()
    _check_structure(r, os.path.getsize(path))
    levels = {nd.level for nd in r.nodes}
    assert max(levels) == (0 if n <= 256 else 1)


def test_twenty_thousand_datasets_make_a_deeper_tree(lib, tmp_path):
    items = [(name, np.full((1, 2), i, np.float32)) for i, (name, _) in enumerate(_reference_names(10000))]
    path = str(tmp_path / "f.h5")
    r = _write(path, items)
    assert len(r.names) == 20000
    assert max(nd.level for nd in r.nodes) >= 2
    for i, (name, _) in enumerate(items[::997]):
        assert r.read(name.lstrip("/")).tobytes() == items[i * 997][1].tobytes()
    _check_structure(r, os.path.getsize(path))


@pytest.mark.parametrize("shape", [(1, 1), (1, 37), (41, 1), (1080, 1920)])
def test_shapes_and_special_values(lib, tmp_path, shape):
    rng = np.random.default_rng(0)
    a = rng.standard_normal(shape).astype(np.float32)
    flat = a.reshape(-1)
    for i, v in enumerate([np.nan, np.inf, -np.inf, -0.0, np.float32(1e-45)]):
        if i < flat.size:
            flat[(i * 7919) % flat.size] = v
    b = (a * 3).astype(np.float32)
    path = str(tmp_path / "f.h5")
    r = _write(path, [("/flow_x_00000", a), ("/flow_y_00000", b)])
    assert r.read("flow_x_00000").shape == shape
    assert r.read("flow_x_00000").tobytes() == a.tobytes()
    assert r.read("flow_y_00000").tobytes() == b.tobytes()
    _check_structure(r, os.path.getsize(path))


def test_duplicate_and_bad_names_are_refused(lib, tmp_path):
    from denseflow_b200 import h5
    a = np.zeros((2, 2), np.float32)
    path = str(tmp_path / "f.h5")
    with h5.File(path, variant="hdf5") as f:
        f.write_float("/flow_x_00000", a)
        with pytest.raises(RuntimeError, match="already exists"):
            f.write_float("flow_x_00000", a)
        for bad in ("", "/", "a/b"):
            with pytest.raises(RuntimeError, match="not a name in the root group"):
                f.write_float(bad, a)
        f.write_float("/flow_y_00000", a)
    r = h5_read.H5File(path)
    assert r.names == ["flow_x_00000", "flow_y_00000"]


def test_same_calls_same_bytes(lib, tmp_path):
    rng = np.random.default_rng(1)
    items = [(name, rng.standard_normal((4, 6)).astype(np.float32)) for name, _ in _reference_names(12, first=30)]
    p1, p2 = str(tmp_path / "a.h5"), str(tmp_path / "b.h5")
    _write(p1, items)
    _write(p2, items)
    assert open(p1, "rb").read() == open(p2, "rb").read()


def test_create_truncates(lib, tmp_path):
    path = tmp_path / "f.h5"
    path.write_bytes(b"x" * 100000)
    r = _write(str(path), [("/flow_x_00000", np.ones((2, 3), np.float32))])
    assert os.path.getsize(path) == r.eof < 100000


def test_default_library_refuses(lib, tmp_path):
    L = lib.load("default")
    f = C.c_void_p(1)
    path = tmp_path / "f.h5"
    assert L.dfb_h5_create(str(path).encode(), C.byref(f)) == lib.DFB_ERR_UNSUPPORTED
    assert L.dfb_last_error(None) == b"HDF5 support is not enabled, pls recompile"
    assert not f.value and not path.exists()
    from denseflow_b200 import h5
    with pytest.raises(RuntimeError, match="HDF5 support is not enabled, pls recompile"):
        h5.File(str(path))


def test_hdf5_library_exports_what_the_default_one_does(lib):
    a = C.CDLL(lib.LIB_PATHS["hdf5"])
    for name in lib.SIGNATURES:
        assert hasattr(a, name), name
    assert lib.load("hdf5").dfb_version() == lib.load("default").dfb_version()


def test_files_open_with_h5py(lib, tmp_path):
    h5py = pytest.importorskip("h5py")
    for n in (0, 9, 257):
        rng = np.random.default_rng(n)
        items = [(name, rng.standard_normal((3, 4)).astype(np.float32)) for name, _ in _reference_names((n + 1) // 2)[:n]]
        path = str(tmp_path / ("f%d.h5" % n))
        _write(path, items)
        with h5py.File(path, "r") as f:
            assert sorted(f.keys()) == sorted(nm.lstrip("/") for nm, _ in items)
            for name, a in items:
                assert f[name][()].tobytes() == a.tobytes()


@pytest.mark.parametrize("step", [1, 2, -1, -3])
@pytest.mark.parametrize("first", [0, 64, 500])
def test_h5_names_and_path_restate_write_hdf5(step, first):
    """writeHDF5 (src/common.cpp:120-150): sprintf("/flow_x%s_%05d") over the chunk's flows, then the same for y, with the
    index offset by |step| for negative steps; the file <outdir>.h5 with _p<s> / _m<|s|> before .h5"""
    from denseflow_b200 import listrun
    tag = {1: "", 2: "_p2", -1: "_m1", -3: "_m3"}[step]
    off = -step if step < 0 else 0
    n = 5
    assert listrun.h5_names(step, first, n) == (["/flow_x%s_%05d" % (tag, first + i + off) for i in range(n)] +
                                                 ["/flow_y%s_%05d" % (tag, first + i + off) for i in range(n)])
    assert listrun.h5_path("out/cls/video", step) == "out/cls/video%s.h5" % tag
    assert listrun.h5_path("out/video/", step) == "out/video%s.h5" % tag
    assert listrun.h5_names(step, first, 0) == []
