"""Decoded-image sources shared by the GPU suites of pigo_gray_images and the decoded calls: host planes in each format with
the gray image the oracles (decoded_oracle, decoded_formats_oracle) make of them, and the source lists those suites use."""
import numpy as np
import pytest

import decoded_formats_oracle as F
import decoded_oracle as D
import oracle_lib as O
from pigo_b200 import DecodedImage, ImageParams, synth

GRAY16, RGBA64, NRGBA64, CMYK, PALETTED = 5, 6, 7, 8, 9


def face_gray(h, w, seed):
    return synth.frame_faces(synth.sample_gray(), h, w, shift=(seed % 7 * 5, seed % 5 * 9), noise_seed=seed)


class Src:
    """One decoded source: host planes (flat buffers from the rectangle's origin), the pigo_decoded fields and the oracle's gray."""

    def __init__(self, fmt, w, h, planes, strides, sub=0, min_x=0, min_y=0):
        self.fmt, self.w, self.h, self.planes, self.strides, self.sub, self.min_x, self.min_y = fmt, w, h, planes, strides, sub, min_x, min_y
        self.want = D.decoded_gray(fmt, planes, strides, w, h, sub, min_x, min_y)

    def decoded(self, planes=None):
        return DecodedImage(self.fmt, self.w, self.h, tuple(planes or self.planes), self.strides, self.sub, self.min_x, self.min_y)


class WideSrc(Src):
    """A source of a format above 8 bits per sample, CMYK or Paletted: the fields Src.decoded reads, and the gray
    decoded_formats_oracle makes of it."""

    def __init__(self, fmt, w, h, planes, strides):
        self.fmt, self.w, self.h, self.planes, self.strides, self.sub, self.min_x, self.min_y = fmt, w, h, planes, strides, 0, 0, 0
        self.want = F.decoded_gray(fmt, planes, strides, w, h)


def ycbcr_src(sub, w, h, min_x, min_y, seed, luma=None):
    y, cb, cr = O.make_ycbcr_planes(seed, sub, w, h, min_x, min_y)
    if luma is not None:   # face content in Y, chroma near neutral
        y[:, :w] = luma
        cb[:] = 128 + cb % 9 - 4
        cr[:] = 128 + cr % 7 - 3
    return Src(0, w, h, (y.reshape(-1), cb.reshape(-1), cr.reshape(-1)), (y.shape[1], cb.shape[1]), sub, min_x, min_y)


def rgba_src(fmt, w, h, pad, seed, luma=None, alpha=None):
    rng = np.random.default_rng(seed)
    px = rng.integers(0, 256, size=(h, w, 4), dtype=np.uint8)
    if luma is not None:
        px[..., 0] = px[..., 1] = px[..., 2] = luma
        px[..., 3] = 255
    if alpha is not None:
        px[..., 3] = alpha
    buf = np.full((h, 4 * w + pad), 0x5A, dtype=np.uint8)
    buf[:, :4 * w] = px.reshape(h, 4 * w)
    return Src(fmt, w, h, (buf.reshape(-1),), (4 * w + pad, 0))


def gray_src(w, h, pad, seed, luma=None):
    buf = np.full((h, w + pad), 0x33, dtype=np.uint8)
    buf[:, :w] = luma if luma is not None else np.random.default_rng(seed).integers(0, 256, size=(h, w), dtype=np.uint8)
    return Src(3, w, h, (buf.reshape(-1),), (w + pad, 0))


def premultiplied_alpha(h, w, seed):
    """Alpha 0, 255, intermediate values; channels above alpha stay in (invalid premultiplied input)."""
    a = np.random.default_rng(seed).integers(0, 256, size=(h, w), dtype=np.uint8)
    a[::3, ::2] = 0
    a[1::3, ::2] = 255
    return a


def be16(v: np.ndarray) -> np.ndarray:
    """uint16 values [h][w][k] as the big-endian bytes [h][w*2k] Go stores in Pix."""
    v = np.asarray(v, dtype=np.uint32)
    return np.stack([v >> 8, v & 0xFF], axis=-1).reshape(v.shape[0], -1).astype(np.uint8)


def flat(rows: np.ndarray, pad: int, off: int, fill: int):
    """rows [h][row bytes] laid out with `pad` bytes of row padding, `off` bytes into a buffer (so the plane's address is
    off mod 16 when off < 16).  Returns (plane from the first pixel, stride)."""
    h, rb = rows.shape
    stride = rb + pad
    buf = np.full(off + h * stride, fill, dtype=np.uint8)
    plane = buf[off:]
    plane.reshape(h, stride)[:, :rb] = rows
    return plane, stride


def alpha16(h, w, rng):
    """Alpha 0, 0xffff and intermediate values (the channels drawn next to it are often above it)."""
    a = rng.integers(0, 65536, size=(h, w))
    a[::3, ::2] = 0
    a[1::3, ::2] = 0xFFFF
    a[2::3, 1::4] = rng.integers(0, 256, size=a[2::3, 1::4].shape)
    return a


def wide_src(fmt, w, h, pad=0, off=0, seed=0, luma=None, palette_len=256):
    """A seeded source of a format of WideSrc; with `luma` its gray is exactly luma (the encodings of tools/ragged_bench.py)."""
    rng = np.random.default_rng(seed)
    noise = rng.integers(0, 256, size=(h, w))
    if fmt == GRAY16:
        y = (luma.astype(np.int64) << 8 | noise) if luma is not None else rng.integers(0, 65536, size=(h, w))
        rows = be16(y[..., None])
    elif fmt in (RGBA64, NRGBA64):
        if luma is not None:
            c = luma.astype(np.int64) << 8 | noise
            v = np.stack([c, c, c, np.full_like(c, 0xFFFF)], axis=-1)
        else:
            v = rng.integers(0, 65536, size=(h, w, 4))
            v[..., 3] = alpha16(h, w, rng)
        rows = be16(v)
    elif fmt == CMYK:
        px = rng.integers(0, 256, size=(h, w, 4))
        if luma is not None:
            px[..., :3] = 0
            px[..., 3] = 255 - luma.astype(np.int64)
        rows = px.astype(np.uint8).reshape(h, 4 * w)
    else:
        if luma is not None:   # a permuted gray palette
            perm = rng.permutation(256)
            pal = np.stack([perm, perm, perm, np.full(256, 255)], axis=-1).astype(np.uint8)
            rows = np.argsort(perm)[luma].astype(np.uint8)
        else:
            pal = rng.integers(0, 256, size=(palette_len, 4)).astype(np.uint8)
            pal[::5, 3] = 255
            rows = rng.integers(0, 256, size=(h, w)).astype(np.uint8)
        plane, stride = flat(rows, pad, off, 0x77)
        pal = pal[:palette_len]
        return WideSrc(fmt, w, h, (plane, np.ascontiguousarray(pal).reshape(-1)), (stride, len(pal)))
    plane, stride = flat(rows, pad, off, 0x5A)
    return WideSrc(fmt, w, h, (plane,), (stride, 0))


def narrow_sources():
    """One small source of each 8-bit format (YCbCr, NRGBA, RGBA with premultiplied alpha, Gray)."""
    return [ycbcr_src(2, 45, 31, 3, 1, 11), rgba_src(1, 33, 20, 12, 30), rgba_src(2, 29, 31, 8, 40, alpha=premultiplied_alpha(31, 29, 40)),
            gray_src(45, 19, 3, 51)]


def slot(arena, im):
    off = im.Pixels - arena.data_ptr()
    return arena[off:off + im.Rows * im.Cols].cpu().numpy().reshape(im.Rows, im.Cols)


def host_images(srcs):
    return [ImageParams(s.want.reshape(-1), s.h, s.w, s.w) for s in srcs]


@pytest.fixture(scope="module")
def eight_bit_sources():
    """The 8-bit formats: every YCbCr subsample ratio, odd sizes, rectangle origins, padded strides, face content."""
    s = [ycbcr_src(sub, w, h, mx, my, 10 + sub) for sub, (w, h, mx, my) in
         enumerate([(37, 23, 0, 0), (64, 48, 1, 0), (101, 77, 5, 3), (17, 9, 3, 1), (45, 31, 3, 2), (29, 13, 1, 1)])]
    s += [ycbcr_src(2, 1, 1, 1, 1, 20), ycbcr_src(2, 1, 50, 3, 0, 21), ycbcr_src(5, 50, 1, 0, 3, 22), ycbcr_src(4, 3, 5, 1, 1, 23),
          ycbcr_src(2, 320, 400, 1, 1, 24, luma=synth.sample_gray()), ycbcr_src(1, 961, 541, 0, 1, 25, luma=face_gray(541, 961, 25))]
    s += [rgba_src(1, 33, 20, 12, 30), rgba_src(1, 1, 1, 0, 31), rgba_src(1, 16, 16, 0, 32), rgba_src(1, 640, 480, 16, 33, luma=face_gray(480, 640, 33))]
    s += [rgba_src(2, 29, 31, 8, 40, alpha=premultiplied_alpha(31, 29, 40)), rgba_src(2, 1, 3, 4, 41, alpha=np.array([[0], [255], [77]], np.uint8)),
          rgba_src(2, 300, 200, 0, 42, luma=face_gray(200, 300, 42), alpha=np.full((200, 300), 255, np.uint8))]
    s += [gray_src(1, 7, 0, 50), gray_src(45, 19, 3, 51), gray_src(320, 400, 0, 52, luma=synth.sample_gray()), gray_src(17, 1, 5, 53),
          gray_src(900, 300, 7, 54, luma=face_gray(300, 900, 54))]
    return s


SHAPES = [(1, 1, 0, 1), (1, 37, 3, 5), (37, 1, 0, 0), (16, 16, 0, 0), (33, 20, 5, 15), (64, 9, 0, 7), (961, 541, 16, 0), (961, 541, 9, 3)]


@pytest.fixture(scope="module")
def wide_sources():
    """Gray16, RGBA64, NRGBA64, CMYK and Paletted in each of SHAPES (width, height, row padding, plane offset)."""
    out = []
    for fmt in (GRAY16, RGBA64, NRGBA64, CMYK, PALETTED):
        for k, (w, h, pad, off) in enumerate(SHAPES):
            out.append(wide_src(fmt, w, h, pad, off, seed=100 * fmt + k, palette_len=256 if k % 2 else 1 + 37 * k))
    return out


@pytest.fixture(scope="module")
def face_sources():
    """Face content in each format of WideSrc, its gray exactly the face image."""
    shapes = [(640, 480, 16, 0), (320, 400, 0, 3), (961, 541, 7, 1), (500, 300, 0, 0), (700, 450, 5, 9)]
    out = []
    for k, (fmt, (w, h, pad, off)) in enumerate(zip((GRAY16, RGBA64, NRGBA64, CMYK, PALETTED), shapes)):
        g = synth.sample_gray() if (h, w) == (400, 320) else face_gray(h, w, 60 + k)
        s = wide_src(fmt, w, h, pad, off, seed=60 + k, luma=g)
        assert np.array_equal(s.want, g), fmt
        out.append(s)
    return out
