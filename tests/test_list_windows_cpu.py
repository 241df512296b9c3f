"""No-GPU checks of dfb_list_run_windows: a call without a runner, without a source or with a save type it does not write is
refused before any work, with DFB_ERR_INVALID_ARG and a message that names the entry point."""
import ctypes as C

import pytest


@pytest.fixture(scope="module")
def L():
    import __graft_entry__ as g
    g.build()
    from denseflow_b200 import _lib
    return _lib.load()


def _call(L, runner, source, save_type=0, n_videos=1):
    from denseflow_b200 import _lib
    st = _lib.ListStats()
    err = C.create_string_buffer(512)
    rc = L.dfb_list_run_windows(runner, n_videos, source, 1, 20, save_type, 95, 0, 0, 0, 0, 4, None, None, None, C.byref(st), err, 512)
    return rc, err.value.decode()


def test_refusals_name_the_entry_point(L):
    from denseflow_b200 import _lib
    calls = []

    def source(user, video, first, max_n, out, msg, msg_len):
        calls.append(video)
        return 1

    src = _lib.FRAMES_FN(source)
    ptr = C.cast(src, C.c_void_p)
    cases = {
        "no runner": (None, ptr, 0, 1),
        "no source": (None, None, 0, 1),
        "bad save_type": (None, ptr, 7, 1),
        "negative n_videos": (None, ptr, 0, -1),
    }
    messages = set()
    for name, (runner, source_ptr, save_type, n) in cases.items():
        rc, msg = _call(L, runner, source_ptr, save_type, n)
        assert rc == _lib.DFB_ERR_INVALID_ARG, name
        assert msg.startswith("dfb_list_run_windows"), (name, msg)
        messages.add(msg)
    assert len(messages) == 3  # a missing runner, a missing source or n_videos, and the save type are told apart
    assert "save_type" in _call(L, None, ptr, 7)[1]
    assert "runner" in _call(L, None, ptr, 0)[1]
    assert calls == []  # nothing was read
