"""HDF5 flow files (`-st=h5`) over the C ABI's writer: dfb_h5_create / dfb_h5_write_float / dfb_h5_close.

    with h5.File("video.h5", variant="hdf5") as f:
        f.write_float("/flow_x_00000", flow_x)      # H5LTmake_dataset_float, rank 2, (rows, cols)

Only the "hdf5" library (the counterpart of the reference's -DUSE_HDF5=yes build) has the writer; the default library
refuses with "HDF5 support is not enabled, pls recompile".  Errors raise RuntimeError with the library's message.
"""
import ctypes as C
import threading

import numpy as np

from . import _lib

# The writer's messages go to dfb_last_error(NULL), which every handle-less call shares: a call and the read of its message
# happen under this lock, so files written from several threads each report their own error.
_calls = threading.Lock()


class File:
    """One HDF5 file, created (or truncated) on construction; its metadata is written by close()."""

    def __init__(self, path, variant="default"):
        self._L = _lib.load(variant)
        self._f = C.c_void_p()
        with _calls:
            if self._L.dfb_h5_create(str(path).encode(), C.byref(self._f)) != _lib.DFB_OK:
                self._f = None
                raise RuntimeError(self._L.dfb_last_error(None).decode())

    def _call(self, fn, *args):
        with _calls:
            if fn(*args) != _lib.DFB_OK:
                raise RuntimeError(self._L.dfb_last_error(None).decode())

    def write_float(self, name, data):
        """data: a 2-D float32 array, written as dataset `name` of shape data.shape.  A name already written raises."""
        if self._f is None:
            raise RuntimeError("the file is closed")
        a = np.ascontiguousarray(data)
        if a.dtype != np.float32 or a.ndim != 2:
            raise RuntimeError("write_float: expected a 2-D float32 array")
        self._call(self._L.dfb_h5_write_float, self._f, name.encode(), a.shape[0], a.shape[1], a.ctypes.data)

    def close(self):
        if self._f is not None:
            f, self._f = self._f, None
            self._call(self._L.dfb_h5_close, f)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
