"""Oracles for pigo_blur_faces (test infrastructure only), the semantics of include/pigo_b200.h restated twice: in C
(blur_oracle.c, plain loops) and vectorised in numpy here, and the seeded sources and faces the blur suites draw.

A source is a BlurSrc: pigo_decoded fields with host planes that are whole buffers (every row `stride` bytes long, the
padding included), so that a test can check every byte of every plane."""
from __future__ import annotations

import ctypes as C

import numpy as np

import decoded_oracle as D
from pigo_b200 import DET_DTYPE, DecodedImage

FORMATS = (0, 1, 2, 3, 8)   # YCbCr, NRGBA, RGBA, Gray, CMYK
XSHIFT, YSHIFT = (0, 1, 1, 0, 2, 2), (0, 0, 1, 1, 0, 1)
_LIB = None


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        L = D.compile_c("blur_oracle")
        vp, i, d = C.c_void_p, C.c_int, C.c_double
        L.oracle_blur.argtypes = [i, i, i, i, i, i, vp, vp, vp, i, i, vp, i, d, d, d, i]
        L.oracle_blur.restype = None
        _LIB = L
    return _LIB


class BlurSrc:
    """One decoded source: format, size, YCbCr ratio and origin, strides, and its planes as whole flat uint8 buffers."""

    def __init__(self, fmt, w, h, planes, strides, sub=0, min_x=0, min_y=0):
        self.fmt, self.w, self.h, self.planes, self.strides, self.sub, self.min_x, self.min_y = fmt, w, h, planes, strides, sub, min_x, min_y

    def copy(self) -> "BlurSrc":
        return BlurSrc(self.fmt, self.w, self.h, [p.copy() for p in self.planes], self.strides, self.sub, self.min_x, self.min_y)

    def decoded(self, planes=None) -> DecodedImage:
        return DecodedImage(self.fmt, self.w, self.h, tuple(planes if planes is not None else self.planes), self.strides, self.sub, self.min_x,
                            self.min_y)

    def chroma(self):
        """(rows, cols) of the chroma planes: the extent decoded_oracle.decoded_gray computes."""
        xd, yd = 1 << XSHIFT[self.sub], 1 << YSHIFT[self.sub]
        return (self.min_y + self.h - 1) // yd - self.min_y // yd + 1, (self.min_x + self.w - 1) // xd - self.min_x // xd + 1

    def layout(self):
        """Per plane (rows, samples per row, bytes per sample, stride, x shift, y shift)."""
        if self.fmt == 0:
            ch, cw = self.chroma()
            xs, ys = XSHIFT[self.sub], YSHIFT[self.sub]
            return [(self.h, self.w, 1, self.strides[0], 0, 0), (ch, cw, 1, self.strides[1], xs, ys), (ch, cw, 1, self.strides[1], xs, ys)]
        return [(self.h, self.w, 1 if self.fmt == 3 else 4, self.strides[0], 0, 0)]


def blur_c(src: BlurSrc, faces, min_q, disc_ratio, radius_ratio, radius) -> BlurSrc:
    """The C restatement on a copy of src."""
    out = src.copy()
    f = np.ascontiguousarray(faces, dtype=DET_DTYPE)
    p = [pl.ctypes.data for pl in out.planes] + [None] * (3 - len(out.planes))
    lib().oracle_blur(src.fmt, src.sub, src.min_x, src.min_y, src.w, src.h, p[0], p[1], p[2], src.strides[0], src.strides[1],
                      f.ctypes.data if len(f) else None, len(f), min_q, disc_ratio, radius_ratio, radius)
    return out


def rmax_np(w, h, faces, min_q, disc_ratio, radius_ratio, radius) -> np.ndarray:
    """[h][w] Rmax of every luma pixel, -1 where no blurred face covers it."""
    m = np.full((h, w), -1, dtype=np.int64)
    lim = 1 << 24
    for f in np.asarray(faces, dtype=DET_DTYPE):
        row, col, scale, q = int(f["row"]), int(f["col"]), int(f["scale"]), float(f["q"])
        if not q >= min_q or scale < 0 or scale > lim or abs(row) > lim or abs(col) > lim:
            continue
        d = int(np.float64(scale) * np.float64(disc_ratio))
        R = min(1023, max(radius, int(np.float64(scale) * np.float64(radius_ratio))))
        ys = np.arange(max(0, row - d), min(h, row + d + 1))
        xs = np.arange(max(0, col - d), min(w, col + d + 1))
        if ys.size == 0 or xs.size == 0:
            continue
        inside = (ys[:, None] - row) ** 2 + (xs[None, :] - col) ** 2 <= d * d
        block = m[ys[0]:ys[-1] + 1, xs[0]:xs[-1] + 1]
        block[inside] = np.maximum(block[inside], R)
    return m


def blur_np(src: BlurSrc, faces, min_q, disc_ratio, radius_ratio, radius) -> BlurSrc:
    """The numpy restatement on a copy of src: per plane, Rmax at each sample's anchor, then box sums from the cumulative sums
    of the edge-padded plane, gathered for all covered samples at once."""
    out = src.copy()
    m = rmax_np(src.w, src.h, faces, min_q, disc_ratio, radius_ratio, radius)
    mx, my = (src.min_x, src.min_y) if src.fmt == 0 else (0, 0)
    for plane, (rows, cols, chans, stride, xs, ys) in zip(out.planes, src.layout()):
        ay = np.clip(((my >> ys) + np.arange(rows)) << ys, my, my + src.h - 1) - my
        ax = np.clip(((mx >> xs) + np.arange(cols)) << xs, mx, mx + src.w - 1) - mx
        R = m[ay][:, ax]
        jj, ii = np.nonzero(R >= 0)
        if jj.size == 0:
            continue
        ry, rx = R[jj, ii] >> ys, R[jj, ii] >> xs
        py, px = int(ry.max()), int(rx.max())
        view = plane[:rows * stride].reshape(rows, stride)
        samples = view[:, :cols * chans].reshape(rows, cols, chans).astype(np.int64)
        padded = np.pad(samples, ((py, py), (px, px), (0, 0)), mode="edge")
        S = np.zeros((padded.shape[0] + 1, padded.shape[1] + 1, chans), dtype=np.int64)
        S[1:, 1:] = padded.cumsum(0).cumsum(1)
        y0, y1, x0, x1 = jj - ry + py, jj + ry + py + 1, ii - rx + px, ii + rx + px + 1
        total = S[y1, x1] - S[y0, x1] - S[y1, x0] + S[y0, x0]
        n = ((2 * ry + 1) * (2 * rx + 1))[:, None]
        vals = ((total + n // 2) // n).astype(np.uint8)
        for c in range(chans):
            view[jj, ii * chans + c] = vals[:, c]
    return out


# ---- seeded sources and faces ------------------------------------------------------------------------------------------------
def make_src(fmt, w, h, rng, sub=0, min_x=0, min_y=0, pad=0, luma=None) -> BlurSrc:
    """A source with random samples (or, given `luma`, that gray content in Y / every colour channel) and `pad` bytes of
    padding per row, padding filled with its own random bytes."""
    def plane(rows, row_bytes):
        stride = row_bytes + pad
        return rng.integers(0, 256, size=rows * stride, dtype=np.uint8), stride
    if fmt == 0:
        src = BlurSrc(0, w, h, [], (0, 0), sub, min_x, min_y)
        ch, cw = src.chroma()
        y, ys = plane(h, w)
        cb, cs = plane(ch, cw)
        cr, _ = plane(ch, cw)
        if luma is not None:
            y.reshape(h, ys)[:, :w] = luma
        src.planes, src.strides = [y, cb, cr], (ys, cs)
        return src
    chans = 1 if fmt == 3 else 4
    p, s = plane(h, w * chans)
    if luma is not None:
        v = p.reshape(h, s)[:, :w * chans].reshape(h, w, chans)
        v[..., :min(chans, 3)] = luma[..., None]
        if chans == 4:
            v[..., 3] = 255 if fmt != 8 else 0
            if fmt == 8:
                v[..., :3] = 0
                v[..., 3] = 255 - luma
    return BlurSrc(fmt, w, h, [p], (s, 0))


def random_faces(w, h, rng, n, min_q=5.0):
    """n faces inside, straddling and outside the image, with Q around min_q (some equal to it, some NaN)."""
    f = np.zeros(n, dtype=DET_DTYPE)
    big = max(w, h)
    f["row"] = rng.integers(-big // 4, h + big // 4 + 1, size=n)
    f["col"] = rng.integers(-big // 4, w + big // 4 + 1, size=n)
    f["scale"] = rng.integers(0, max(2, big // 2), size=n)
    q = rng.uniform(min_q - 3, min_q + 6, size=n).astype(np.float32)
    q[rng.random(n) < 0.15] = np.float32(min_q)
    q[rng.random(n) < 0.05] = np.nan
    f["q"] = q
    return f


def random_case(seed: int):
    """(source, faces, (min_q, disc_ratio, radius_ratio, radius)) of a small seeded case: any format, YCbCr at any ratio and
    origin, padded strides, any size down to 1x1, box radii from 0 past the plane's size."""
    rng = np.random.default_rng(seed)
    fmt = FORMATS[seed % len(FORMATS)]
    w, h = (int(v) for v in rng.integers(1, 48, size=2))
    if seed % 7 == 0:
        w = 1
    elif seed % 7 == 1:
        h = 1
    src = make_src(fmt, w, h, rng, sub=int(rng.integers(0, 6)), min_x=int(rng.integers(0, 5)), min_y=int(rng.integers(0, 5)),
                   pad=int(rng.integers(0, 4)))
    faces = random_faces(w, h, rng, int(rng.integers(0, 6)))
    params = (5.0, float(rng.choice([0.0, 0.3, 0.5, 1.0])), float(rng.choice([0.0, 0.1, 0.5, 2.0])), int(rng.choice([0, 1, 3, 15, 60])))
    return src, faces, params
