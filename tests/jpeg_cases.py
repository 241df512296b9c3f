"""JPEG files for the decoder tests: contents, the samplings and encoder options cv2 and Pillow write, and the files the
decoder refuses."""
import io

import cv2
import numpy as np

SAMPLINGS = ("gray", "444", "422", "440", "420")
_CV_SAMPLING = {"444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
                "440": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440, "420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420,
                "411": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411}


def image(kind, h, w, seed=0):
    """uint8 [h, w, 3]: i.i.d. noise (long codes, many symbols) or smooth colour gradients (short codes, chroma that matters)"""
    rng = np.random.default_rng(seed + 31 * h + w)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), np.uint8)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.stack([128 + 90 * np.sin(xx / 5 + yy / 7), 128 + 80 * np.cos(yy / 4 - xx / 9), 60 + 3 * xx + 5 * yy], -1)
    return np.clip(img, 0, 255).astype(np.uint8)


def encode(img, sampling="420", quality=95, restart=0, optimize=False, luma=None, chroma=None, progressive=False):
    """cv2.imencode(".jpg") bytes; sampling "gray" encodes the green channel as a one-component file"""
    params = [cv2.IMWRITE_JPEG_QUALITY, quality]
    if restart:
        params += [cv2.IMWRITE_JPEG_RST_INTERVAL, restart]
    if optimize:
        params += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    if luma is not None:
        params += [cv2.IMWRITE_JPEG_LUMA_QUALITY, luma, cv2.IMWRITE_JPEG_CHROMA_QUALITY, chroma]
    if progressive:
        params += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    if sampling == "gray":
        ok, buf = cv2.imencode(".jpg", np.ascontiguousarray(img[:, :, 1]), params)
    else:
        ok, buf = cv2.imencode(".jpg", img, params + [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, _CV_SAMPLING[sampling]])
    assert ok
    return buf.tobytes()


def pillow_files(h=37, w=53):
    """Files Pillow writes: 16-bit quantisation tables, a COM segment, an EXIF segment with orientation 1; name -> bytes"""
    from PIL import Image
    img = Image.fromarray(image("smooth", h, w)[:, :, ::-1].copy())
    out = {}
    b = io.BytesIO()
    img.save(b, "JPEG", qtables=[[300 + k for k in range(64)], [700] * 64], subsampling=2)  # values > 255: 16-bit DQT
    out["qt16"] = b.getvalue()
    ex = Image.Exif()
    ex[0x0112] = 1
    b = io.BytesIO()
    img.save(b, "JPEG", quality=80, exif=ex.tobytes(), comment=b"frame folder", subsampling=1)
    out["exif1_com"] = b.getvalue()
    b = io.BytesIO()
    img.convert("L").save(b, "JPEG", quality=60)
    out["gray"] = b.getvalue()
    return out


def exif6(h=24, w=40):
    from PIL import Image
    ex = Image.Exif()
    ex[0x0112] = 6
    b = io.BytesIO()
    Image.fromarray(image("smooth", h, w)).save(b, "JPEG", quality=90, exif=ex.tobytes())
    return b.getvalue()


def bad_rst(h=64, w=64):
    """A file with restart interval 1 whose second RST marker carries the wrong number"""
    b = bytearray(encode(image("smooth", h, w), "420", 90, restart=1))
    seen = 0
    for i in range(len(b) - 1):
        if b[i] == 0xFF and 0xD0 <= b[i + 1] <= 0xD7:
            seen += 1
            if seen == 2:
                b[i + 1] = 0xD5
                return bytes(b)
    raise AssertionError("no RST markers")


def truncated(h=64, w=64):
    """The first 60 % of a file's bytes, then EOI"""
    b = encode(image("noise", h, w), "420", 90)
    return b[:int(len(b) * 0.6)] + b"\xff\xd9"


def refusals():
    """name -> (bytes, 'unsupported' | 'corrupt', fragment of the message)"""
    img = image("smooth", 40, 48)
    return {
        "progressive": (encode(img, "420", 90, progressive=True), "unsupported", "progressive"),
        "411": (encode(img, "411", 90), "unsupported", "subsampling"),
        "orientation6": (exif6(), "unsupported", "orientation 6"),
        "truncated": (truncated(), "corrupt", "ends before the last MCU"),
        "bad_rst": (bad_rst(), "corrupt", "RST"),
    }
