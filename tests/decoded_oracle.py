"""Oracle for pigo_gray_images (test infrastructure only): the reference's detector input RgbToGrayscale(ImgToNRGBA(img))
(core/grayscale.go:8-23, core/image.go:35-90) of a decoded image, composed from the existing CPU oracle (oracle_lib) and
a restatement of Go's color.NRGBAModel for *image.RGBA pixels written twice, independently: in C (decoded_oracle.c, built
into a temporary directory on first use) and vectorised in numpy here."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import oracle_lib as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def compile_c(name: str) -> C.CDLL:
    """Compiles tests/<name>.c like oracle/Makefile compiles the main oracle (-ffp-contract=off), into the temporary directory,
    once per version of the source, and loads it."""
    src = os.path.join(_HERE, name + ".c")
    with open(src, "rb") as f:
        tag = hashlib.sha256(f.read()).hexdigest()[:16]
    so = os.path.join(tempfile.gettempdir(), f"pigo_{name}_{os.getuid()}_{tag}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}"
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-std=c11", "-Wall", "-Wextra", "-ffp-contract=off", "-shared",
                               "-o", tmp, src])
        os.replace(tmp, so)
    return C.CDLL(so)


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        L = compile_c("decoded_oracle")
        L.oracle_rgba_to_nrgba.argtypes = [C.c_void_p, C.c_int64, C.c_void_p]
        L.oracle_rgba_to_nrgba.restype = None
        _LIB = L
    return _LIB


def rgba_to_nrgba(rgba: np.ndarray) -> np.ndarray:
    """color.NRGBAModel of alpha-premultiplied color.RGBA pixels [..., 4] (the C restatement)."""
    rgba = np.ascontiguousarray(rgba, dtype=np.uint8)
    out = np.zeros_like(rgba)
    lib().oracle_rgba_to_nrgba(rgba.ctypes.data, rgba.size // 4, out.ctypes.data)
    return out


def rgba_to_nrgba_np(rgba: np.ndarray) -> np.ndarray:
    """The same, vectorised in int64: un-premultiply the 16-bit channels c*257 by alpha a*257 as (c*0xffff)//a and keep the
    high byte; opaque pixels keep their bytes, transparent ones become all zero; a channel above alpha keeps Go's uint8
    truncation (& 0xff)."""
    px = np.asarray(rgba, dtype=np.int64)
    a16 = px[..., 3:4] * 257
    c16 = px[..., :3] * 257
    safe = np.where(a16 == 0, 1, a16)
    straight = ((c16 * 65535) // safe >> 8) & 0xFF
    rgb = np.where(a16 == 65535, px[..., :3], np.where(a16 == 0, 0, straight))
    return np.concatenate([rgb, px[..., 3:4]], axis=-1).astype(np.uint8)


def nrgba_luma_np(nrgba: np.ndarray) -> np.ndarray:
    """core/grayscale.go:8-23 on NRGBA pixels [..., 4] with any alpha, in numpy: color.NRGBA.RGBA() channels c*257*a//255,
    then the float64 luma truncated to uint8."""
    px = np.asarray(nrgba, dtype=np.int64)
    v = (px[..., :3] * 257 * px[..., 3:4] // 255).astype(np.float64)
    return ((0.299 * v[..., 0] + 0.587 * v[..., 1] + 0.114 * v[..., 2]) / 256).astype(np.uint8)


def _rows(plane, stride: int, height: int, row_bytes: int) -> np.ndarray:
    """[height][row_bytes] rows of a plane given as a uint8 array that starts at the rectangle's origin (flattened row-major)."""
    flat = np.asarray(plane, dtype=np.uint8).reshape(-1)
    return np.stack([flat[r * stride:r * stride + row_bytes] for r in range(height)])


def decoded_gray(fmt: int, planes, strides, width: int, height: int, subsample: int = 0, min_x: int = 0, min_y: int = 0) -> np.ndarray:
    """RgbToGrayscale(ImgToNRGBA(img)) of one decoded image given as pigo_decoded fields (fmt 0..3 = YCbCr, NRGBA, RGBA, Gray;
    host planes at the rectangle's origin with the given strides).  Returns [height][width] uint8."""
    if fmt == 0:
        xd, yd = (1, 2, 2, 1, 4, 4)[subsample], (1, 1, 2, 2, 1, 2)[subsample]
        ch = (min_y + height - 1) // yd - min_y // yd + 1
        cw = (min_x + width - 1) // xd - min_x // xd + 1
        y = _rows(planes[0], strides[0], height, width)
        cb, cr = (_rows(p, strides[1], ch, cw) for p in planes[1:3])
        nrgba = O.ycbcr_to_nrgba(y, cb, cr, subsample, width, height, min_x, min_y)
    elif fmt in (1, 2):
        nrgba = _rows(planes[0], strides[0], height, 4 * width).reshape(height, width, 4)
        if fmt == 2:
            nrgba = rgba_to_nrgba(nrgba)
    elif fmt == 3:
        g = _rows(planes[0], strides[0], height, width)
        nrgba = np.stack([g, g, g, np.full_like(g, 0xff)], axis=-1)
    else:
        raise ValueError("unknown format %d" % fmt)
    return O.rgba_to_gray(nrgba)
