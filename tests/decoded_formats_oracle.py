"""Oracle for pigo_gray_images on *image.Gray16, RGBA64, NRGBA64, CMYK and Paletted sources (test infrastructure only): the
reference's detector input RgbToGrayscale(ImgToNRGBA(img)) (core/grayscale.go:8-23, core/image.go:35-90) of such an image,
composed from the existing CPU oracle (oracle_lib) and restatements of Go's color.NRGBAModel for these types, each written
twice, independently: in C (decoded_formats_oracle.c, built into a temporary directory on first use) and vectorised in
numpy here.  decoded_gray extends decoded_oracle.decoded_gray, which it calls for the other formats."""
from __future__ import annotations

import ctypes as C

import numpy as np

import decoded_oracle
import oracle_lib as O

GRAY16, RGBA64, NRGBA64, CMYK, PALETTED = 5, 6, 7, 8, 9

_LIB = None


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        L = decoded_oracle.compile_c("decoded_formats_oracle")
        for name in ("oracle_gray16_to_nrgba", "oracle_cmyk_to_nrgba"):
            getattr(L, name).argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
            getattr(L, name).restype = None
        L.oracle_rgba64_to_nrgba.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_void_p]
        L.oracle_rgba64_to_nrgba.restype = None
        _LIB = L
    return _LIB


def _c_model(fn, px: np.ndarray, bpp: int, *extra) -> np.ndarray:
    px = np.ascontiguousarray(px, dtype=np.uint8)
    out = np.zeros(px.shape[:-1] + (4,), dtype=np.uint8)
    fn(px.ctypes.data, px.size // bpp, *extra, out.ctypes.data)
    return out


def gray16_to_nrgba(px: np.ndarray) -> np.ndarray:
    """color.NRGBAModel of *image.Gray16 pixels [..., 2] (big-endian bytes as in Pix; the C restatement)."""
    return _c_model(lib().oracle_gray16_to_nrgba, px, 2)


def rgba64_to_nrgba(px: np.ndarray, premultiplied: bool) -> np.ndarray:
    """color.NRGBAModel of *image.RGBA64 (premultiplied) or *image.NRGBA64 pixels [..., 8] (the C restatement)."""
    return _c_model(lib().oracle_rgba64_to_nrgba, px, 8, int(premultiplied))


def cmyk_to_nrgba(px: np.ndarray) -> np.ndarray:
    """color.NRGBAModel of *image.CMYK pixels [..., 4] (the C restatement)."""
    return _c_model(lib().oracle_cmyk_to_nrgba, px, 4)


def _nrgba_model_np(r, g, b, a) -> np.ndarray:
    """color.nrgbaModel on int64 arrays of 16-bit channels: opaque keeps the high bytes, transparent is all zero, else the
    un-premultiplied (c*0xffff)//a keeps its high byte with Go's uint8 truncation."""
    safe = np.where(a == 0, 1, a)
    ch = [np.where(a == 0xFFFF, c >> 8, np.where(a == 0, 0, ((c * 0xFFFF) // safe >> 8) & 0xFF)) for c in (r, g, b)]
    return np.stack(ch + [a >> 8], axis=-1).astype(np.uint8)


def _be16_np(px: np.ndarray) -> np.ndarray:
    p = np.asarray(px, dtype=np.int64)
    return p[..., 0::2] * 256 + p[..., 1::2]


def gray16_to_nrgba_np(px: np.ndarray) -> np.ndarray:
    y = _be16_np(px)[..., 0]
    return _nrgba_model_np(y, y, y, np.full_like(y, 0xFFFF))


def rgba64_to_nrgba_np(px: np.ndarray, premultiplied: bool) -> np.ndarray:
    v = _be16_np(px)
    a = v[..., 3]
    rgb = [v[..., k] if premultiplied else v[..., k] * a // 0xFFFF for k in range(3)]
    return _nrgba_model_np(*rgb, a)


def cmyk_to_nrgba_np(px: np.ndarray) -> np.ndarray:
    p = np.asarray(px, dtype=np.int64)
    w = 0xFFFF - p[..., 3] * 0x101
    rgb = [(0xFFFF - p[..., k] * 0x101) * w // 0xFFFF for k in range(3)]
    return _nrgba_model_np(*rgb, np.full_like(w, 0xFFFF))


def palette_lookup(idx: np.ndarray, palette: np.ndarray, length: int) -> np.ndarray:
    """The NRGBA pixels of palette indices; an index at or past the palette's length gives the zero pixel (gray 0)."""
    pal = np.zeros((256, 4), dtype=np.uint8)
    pal[:length] = np.asarray(palette, dtype=np.uint8).reshape(-1, 4)[:length]
    return pal[np.asarray(idx, dtype=np.uint8)]


def _rows(plane, stride: int, height: int, row_bytes: int) -> np.ndarray:
    """[height][row_bytes] rows of a plane given as a uint8 array that starts at the rectangle's origin (flattened row-major)."""
    flat = np.asarray(plane, dtype=np.uint8).reshape(-1)
    return np.stack([flat[r * stride:r * stride + row_bytes] for r in range(height)])


def decoded_gray(fmt: int, planes, strides, width: int, height: int, subsample: int = 0, min_x: int = 0, min_y: int = 0) -> np.ndarray:
    """RgbToGrayscale(ImgToNRGBA(img)) of one decoded image given as pigo_decoded fields: fmt 5..9 = Gray16, RGBA64, NRGBA64,
    CMYK, Paletted (the palette as planes[1], its length as strides[1]); fmt 0..3 as decoded_oracle.decoded_gray.  Host planes
    at the rectangle's origin with the given strides.  Returns [height][width] uint8."""
    if fmt < GRAY16:
        return decoded_oracle.decoded_gray(fmt, planes, strides, width, height, subsample, min_x, min_y)
    if fmt == GRAY16:
        nrgba = gray16_to_nrgba(_rows(planes[0], strides[0], height, 2 * width).reshape(height, width, 2))
    elif fmt in (RGBA64, NRGBA64):
        nrgba = rgba64_to_nrgba(_rows(planes[0], strides[0], height, 8 * width).reshape(height, width, 8), fmt == RGBA64)
    elif fmt == CMYK:
        nrgba = cmyk_to_nrgba(_rows(planes[0], strides[0], height, 4 * width).reshape(height, width, 4))
    elif fmt == PALETTED:
        nrgba = palette_lookup(_rows(planes[0], strides[0], height, width), planes[1], strides[1])
    else:
        raise ValueError("unknown format %d" % fmt)
    return O.rgba_to_gray(nrgba)
