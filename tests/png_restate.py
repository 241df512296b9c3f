"""`cv2.imencode(".png", img)` restated on the standard library's zlib: OpenCV's default PNG parameters (filter SUB on every
row, compression level 1 = Z_BEST_SPEED, strategy Z_RLE) as libpng drives zlib.  The GPU encoder (png_encode.cu) is pinned
to this, and this to cv2 and to the golden bytes in tests/golden/png_imencode_cases.npz (tests/test_png_encode_cpu.py).

Only the two zlib header bytes differ from plain `compressobj` output: libpng declares the smallest window that covers the
data.  The deflate body does not depend on the window size for these inputs.  The pin is "equal to the cv2 that can be run",
like every other pin of this repository; the reference's OpenCV 4.5.2 uses the same defaults.
"""
import struct
import zlib

import numpy as np

IDAT_BYTES = 8192  # libpng's default compression buffer: one IDAT chunk per full buffer


def chunk(t, d):
    return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d))


def scanlines(img):
    """The filtered scanlines libpng hands to zlib: per row the filter byte, then RGB under SUB (NONE when the width is 1)."""
    h, w = img.shape[:2]
    rgb = img[:, :, ::-1].reshape(h, 3 * w).astype(np.int16)  # libpng is told BGR; the file stores RGB
    sub = rgb.copy()
    sub[:, 3:] = (rgb[:, 3:] - rgb[:, :-3]) % 256  # filter 1 (SUB), 3 bytes per pixel
    f = 0 if w == 1 else 1  # width 1: libpng writes filter 0 (NONE)
    return np.concatenate([np.full((h, 1), f, np.uint8), (sub if f else rgb).astype(np.uint8)], 1).tobytes()


def zlib_stream(raw):
    c = zlib.compressobj(1, zlib.DEFLATED, 15, 8, zlib.Z_RLE)
    z = bytearray(c.compress(raw) + c.flush())
    cinfo = 7  # libpng shrinks the declared window to fit the data
    while cinfo > 0 and (1 << (cinfo + 7)) >= len(raw):
        cinfo -= 1
    z[0] = (cinfo << 4) | 8
    z[1] = 31 - (z[0] * 256) % 31  # FLEVEL 0, FCHECK
    return bytes(z)


def encode(img):
    """img: uint8 [h, w, 3] BGR, as passed to imencode.  Returns the PNG file's bytes."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    z = zlib_stream(scanlines(img))
    out = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0))
    for p in range(0, len(z), IDAT_BYTES):
        out += chunk(b"IDAT", z[p:p + IDAT_BYTES])
    return out + chunk(b"IEND", b"")


def idat_stream(png):
    """The zlib stream of a PNG file: its IDAT payloads joined."""
    out, p = b"", 8
    while p < len(png):
        n = struct.unpack(">I", png[p:p + 4])[0]
        if png[p + 4:p + 8] == b"IDAT":
            out += png[p + 8:p + 8 + n]
        p += 12 + n
    return out
