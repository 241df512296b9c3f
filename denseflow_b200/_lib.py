"""ctypes binding of the C ABI in include/denseflow_b200.h.

There is NO fallback: if the CUDA library is missing this module raises at first use, and
dfb_create fails when no GPU is present (the engine has no CPU path).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATHS = {
    "default": os.path.join(_HERE, "lib", "libdenseflow_b200.so"),
    "strict": os.path.join(_HERE, "lib", "libdenseflow_b200_strict.so"),
    # the default library with the -st=h5 file writer (the reference's -DUSE_HDF5=yes build)
    "hdf5": os.path.join(_HERE, "lib", "libdenseflow_b200_hdf5.so"),
    "strict_hdf5": os.path.join(_HERE, "lib", "libdenseflow_b200_strict_hdf5.so"),
}

DFB_OK = 0
DFB_ERR_INVALID_ARG = -1
DFB_ERR_UNKNOWN_ALGORITHM = -2
DFB_ERR_CUDA = -3
DFB_ERR_SIZE = -4
DFB_ERR_UNSUPPORTED = -5
DFB_ERR_NO_DEVICE = -6


class Tvl1Stats(C.Structure):
    _fields_ = [("nscales", C.c_int), ("warps", C.c_int), ("level_w", C.c_int * 16), ("level_h", C.c_int * 16),
                ("iters", C.c_int * 256)]


class Counters(C.Structure):
    _fields_ = [("pairs", C.c_uint64), ("kernel_launches", C.c_uint64), ("pixel_iters", C.c_uint64),
                ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("timed_kernel_launches", C.c_uint64),
                ("timed_kernel_ns", C.c_uint64), ("timed_kernel_pairs", C.c_uint64), ("pixel_chunks", C.c_uint64)]


LIST_MAX_WORKERS = 32


class Clip(C.Structure):
    _fields_ = [("frames", C.POINTER(C.c_void_p)), ("n_frames", C.c_int), ("width", C.c_int), ("height", C.c_int)]


class ListStats(C.Structure):
    _fields_ = [("clips", C.c_uint64), ("flows", C.c_uint64), ("frames", C.c_uint64), ("seconds", C.c_double), ("workers", C.c_int),
                ("clips_per_worker", C.c_uint64 * LIST_MAX_WORKERS), ("flows_per_worker", C.c_uint64 * LIST_MAX_WORKERS),
                ("busy_seconds_per_worker", C.c_double * LIST_MAX_WORKERS), ("finish_seconds_per_worker", C.c_double * LIST_MAX_WORKERS),
                ("kernel_launches", C.c_uint64), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64)]


VIDEO_BGR = 0
VIDEO_JPEG = 1
SAVE_JPG = 0
SAVE_PNG = 1
SAVE_H5 = 2


class Video(C.Structure):
    _fields_ = [("kind", C.c_int), ("n_frames", C.c_int), ("bgr", C.POINTER(C.c_void_p)), ("width", C.c_int), ("height", C.c_int),
                ("jpeg", C.POINTER(C.c_void_p)), ("jpeg_len", C.POINTER(C.c_size_t))]


FILES_DONE_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t))

FRAMES_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(Video), C.c_void_p, C.c_size_t)

CHUNK_DONE_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                            C.POINTER(C.c_void_p))

# every symbol include/denseflow_b200.h declares, with its signature
SIGNATURES = {
    "dfb_version": (C.c_char_p, []),
    "dfb_device_count": (C.c_int, []),
    "dfb_create": (C.c_int, [C.c_char_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "dfb_destroy": (None, [C.c_void_p]),
    "dfb_last_error": (C.c_char_p, [C.c_void_p]),
    "dfb_set_param": (C.c_int, [C.c_void_p, C.c_char_p, C.c_double]),
    "dfb_get_param": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_double)]),
    "dfb_calc_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, C.c_int,
                                  C.c_void_p, C.c_size_t, C.c_void_p]),
    "dfb_calc_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "dfb_calc_batch_host": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.POINTER(C.c_void_p)]),
    "dfb_calc_batch_host_u8": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]),
    "dfb_calc_batch_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                        C.c_void_p]),
    "dfb_calc_batch_host_planes": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]),
    "dfb_calc_batch_device_planes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                               C.c_void_p]),
    "dfb_quantise_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                      C.c_void_p, C.c_size_t, C.c_void_p]),
    "dfb_flow_to_png_image_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                               C.POINTER(C.c_double), C.c_void_p]),
    "dfb_bgr_to_gray_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dfb_resize_gray_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_int,
                                         C.c_int, C.c_void_p]),
    "dfb_jpeg_max_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "dfb_encode_jpeg_gray_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                              C.POINTER(C.c_size_t), C.c_void_p]),
    "dfb_encode_jpeg_gray_batch_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int,
                                                    C.POINTER(C.c_void_p), C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p]),
    "dfb_decode_jpeg_gray_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.POINTER(C.c_int),
                                              C.POINTER(C.c_int), C.c_void_p]),
    "dfb_process_bgr_batch_host": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_size_t,
                                             C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "dfb_bgr_to_ycc420_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                           C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dfb_jpeg_max_bytes_bgr": (C.c_size_t, [C.c_int, C.c_int]),
    "dfb_encode_jpeg_bgr_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                             C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p]),
    "dfb_extract_frames_host": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                          C.POINTER(C.c_void_p), C.c_size_t, C.POINTER(C.c_size_t)]),
    "dfb_png_max_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "dfb_encode_png_bgr_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                            C.POINTER(C.c_size_t), C.c_void_p]),
    "dfb_calc_batch_host_png": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p),
                                          C.c_size_t, C.POINTER(C.c_size_t)]),
    "dfb_process_bgr_batch_host_png": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                                 C.POINTER(C.c_void_p), C.c_size_t, C.POINTER(C.c_size_t)]),
    "dfb_process_jpeg_batch_host_png": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_int, C.c_int,
                                                  C.c_int, C.POINTER(C.c_void_p), C.c_size_t, C.POINTER(C.c_size_t)]),
    "dfb_process_bgr_batch_host_planes": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                                    C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]),
    "dfb_process_jpeg_batch_host_planes": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_int,
                                                     C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]),
    "dfb_h5_create": (C.c_int, [C.c_char_p, C.POINTER(C.c_void_p)]),
    "dfb_h5_write_float": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_void_p]),
    "dfb_h5_close": (C.c_int, [C.c_void_p]),
    "dfb_extract_frames_jpeg_host": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_int, C.c_int, C.c_int,
                                               C.POINTER(C.c_void_p), C.c_size_t, C.POINTER(C.c_size_t)]),
    "dfb_new_size": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "dfb_jpeg_info": (C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "dfb_decode_jpeg_batch_device": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_int, C.c_void_p,
                                               C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                               C.c_void_p]),
    "dfb_process_jpeg_batch_host": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_int, C.c_int, C.c_int,
                                              C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_size_t,
                                              C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "dfb_debug_jpeg_coefficients": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_int),
                                              C.POINTER(C.c_int)]),
    "dfb_debug_run_kernel":(C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_void_p), C.c_int, C.c_int,
                                       C.c_int, C.POINTER(C.c_double), C.c_int, C.POINTER(C.c_double)]),
    "dfb_debug_time_kernel": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double)]),
    "dfb_get_tvl1_stats": (C.c_int, [C.c_void_p, C.POINTER(Tvl1Stats)]),
    "dfb_get_tvl1_pair_stats": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(Tvl1Stats)]),
    "dfb_get_counters": (C.c_int, [C.c_void_p, C.POINTER(Counters)]),
    "dfb_get_tvl1_phase_ns": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64)]),
    "dfb_reset_counters": (C.c_int, [C.c_void_p]),
    "dfb_queue_open": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]),
    "dfb_queue_next": (C.c_long, [C.c_void_p]),
    "dfb_queue_reset": (None, [C.c_void_p]),
    "dfb_queue_close": (None, [C.c_void_p, C.c_int]),
    "dfb_list_open": (C.c_int, [C.c_char_p, C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.c_char_p, C.c_size_t]),
    "dfb_list_run": (C.c_int, [C.c_void_p, C.POINTER(Clip), C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.POINTER(ListStats), C.c_char_p, C.c_size_t]),
    "dfb_list_close": (None, [C.c_void_p]),
    "dfb_list_run_videos": (C.c_int, [C.c_void_p, C.POINTER(Video), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(ListStats), C.c_char_p, C.c_size_t]),
    "dfb_list_run_stream": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(ListStats), C.c_char_p, C.c_size_t]),
    "dfb_list_run_windows": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(ListStats), C.c_char_p, C.c_size_t]),
    "dfb_run_list": (C.c_int, [C.c_char_p, C.POINTER(C.c_int), C.c_int, C.POINTER(Clip), C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                               C.c_void_p, C.c_void_p, C.POINTER(ListStats), C.c_char_p, C.c_size_t]),
}

_libs = {}


def load(variant="default"):
    """Load the CUDA library; raises (never falls back) if it has not been built."""
    if variant not in _libs:
        path = LIB_PATHS[variant]
        if not os.path.exists(path):
            raise ImportError("denseflow_b200: %s is missing — run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(there is no CPU fallback)" % path)
        L = C.CDLL(path)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _libs[variant] = L
    return _libs[variant]
