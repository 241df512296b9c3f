"""No-GPU checks of the C-ABI library: it loads, exports every symbol include/*.h declares, and refuses to
run without a device (there is no CPU fallback in the product path)."""
import ctypes as C
import glob
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    names = set()
    for hdr in glob.glob(os.path.join(ROOT, "include", "*.h")):
        src = open(hdr).read()
        src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
        names |= set(re.findall(r"\b(dfb_[a-z0-9_]+)\s*\(", src))
    return names


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    from denseflow_b200 import _lib
    return _lib


@pytest.mark.parametrize("variant", ["default", "strict"])
def test_library_exports_every_declared_symbol(built, variant):
    L = C.CDLL(built.LIB_PATHS[variant])
    declared = _declared_symbols()
    assert len(declared) >= 15
    for name in declared:
        assert hasattr(L, name), "missing export: " + name
    assert declared == set(built.SIGNATURES), "ctypes table and header disagree"


def test_version_and_error_behaviour_without_running_compute(built):
    L = built.load()
    assert b"sm_90a" in L.dfb_version()
    h = C.c_void_p()
    # reference error texts (src/denseflow_gpu.cpp:296, :336) come back through dfb_last_error
    assert L.dfb_create(b"lk", 0, 64, 64, C.byref(h)) == built.DFB_ERR_UNKNOWN_ALGORITHM
    assert b"unknown optical algorithm lk" in L.dfb_last_error(None)
    assert L.dfb_create(b"nv", 0, 64, 64, C.byref(h)) == built.DFB_ERR_UNSUPPORTED
    assert b"NV hardware flow not enabled" in L.dfb_last_error(None)
    assert L.dfb_create(b"tvl1", 0, 0, 64, C.byref(h)) == built.DFB_ERR_INVALID_ARG
    if L.dfb_device_count() == 0:
        # the product path fails loudly when there is no GPU — no CPU fallback
        assert L.dfb_create(b"tvl1", 0, 64, 64, C.byref(h)) == built.DFB_ERR_NO_DEVICE
        assert b"no CPU path" in L.dfb_last_error(None)
        import denseflow_b200 as d
        with pytest.raises(RuntimeError, match="no CUDA device"):
            d.create("tvl1")


def test_product_never_imports_the_oracle():
    for path in glob.glob(os.path.join(ROOT, "denseflow_b200", "**", "*"), recursive=True):
        if path.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
            src = open(path).read()
            assert "pyoracle" not in src and "liboracle" not in src and "oracle/" not in src.replace("oracle/ ", ""), path


def test_cpp_host_links_against_the_header_only(built, tmp_path):
    """examples/c_abi_host.cpp uses nothing but include/denseflow_b200.h; error behaviour = message + exit 1
    (tools/denseflow.cpp:93-96)."""
    import subprocess
    import __graft_entry__ as g
    exe = g.build_example()
    raw = tmp_path / "f.raw"
    raw.write_bytes(bytes(64 * 64 * 2))
    r = subprocess.run([exe, str(raw), "64", "64", "2", "lk", "1", "20", str(tmp_path)], capture_output=True, text=True)
    assert r.returncode == 1 and "unknown optical algorithm lk" in r.stderr
    r = subprocess.run([exe, str(raw), "64", "64", "2", "tvl1", "1", "0", str(tmp_path)], capture_output=True, text=True)
    assert r.returncode == 1 and "bound should > 0!" in r.stderr
    assert subprocess.run([exe], capture_output=True).returncode == 0  # no arguments: usage, exit 0 (tools/denseflow.cpp:26-29)
