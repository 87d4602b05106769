"""pigo_gray_images for *image.Gray16, RGBA64, NRGBA64, CMYK and Paletted on the H100: every slot is the oracle's
RgbToGrayscale(ImgToNRGBA(img)) byte for byte over odd sizes, padded strides and unaligned planes; a call mixing all nine
formats shares slots and writes nothing else; host and device planes give the same arena; and detection on the converted
images equals detection on the oracle-made host gray images."""
import ctypes as C

import numpy as np
import pytest
import torch

import decoded_formats_oracle as F
import pigo_b200
from pigo_b200 import CascadeParams, ImageParams, pipeline, synth
from option_guard import options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)
from test_decoded_gpu import Src, face_gray, gray_src, host_images, premultiplied_alpha, rgba_src, slot, ycbcr_src

pytestmark = pytest.mark.gpu

GRAY16, RGBA64, NRGBA64, CMYK, PALETTED = 5, 6, 7, 8, 9
TEST_PARAMS = (20, 1000, 0.2, 1.1)   # core/pigo_test.go:44-50
NCALLS = 15


class WideSrc(Src):
    """A source of a new format: the fields Src.decoded reads, and the gray decoded_formats_oracle makes of it."""

    def __init__(self, fmt, w, h, planes, strides):
        self.fmt, self.w, self.h, self.planes, self.strides, self.sub, self.min_x, self.min_y = fmt, w, h, planes, strides, 0, 0, 0
        self.want = F.decoded_gray(fmt, planes, strides, w, h)


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
    """A seeded source of a new format; with `luma` its gray is exactly luma (the encodings of tools/ragged_bench.py)."""
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


SHAPES = [(1, 1, 0, 1), (1, 37, 3, 5), (37, 1, 0, 0), (16, 16, 0, 0), (33, 20, 5, 15), (64, 9, 0, 7), (961, 541, 16, 0), (961, 541, 9, 3)]


@pytest.fixture(scope="module")
def sources():
    out = []
    for fmt in (GRAY16, RGBA64, NRGBA64, CMYK, PALETTED):
        for k, (w, h, pad, off) in enumerate(SHAPES):
            out.append(wide_src(fmt, w, h, pad, off, seed=100 * fmt + k, palette_len=256 if k % 2 else 1 + 37 * k))
    return out


def to_device(p: np.ndarray) -> torch.Tensor:
    """A device copy of a host plane at the same address modulo 16 (so unaligned planes stay unaligned)."""
    off = p.ctypes.data % 16
    t = torch.zeros(p.size + 16, dtype=torch.uint8, device="cuda")
    t[off:off + p.size].copy_(torch.from_numpy(np.ascontiguousarray(p)))
    return t[off:off + p.size]


def convert(srcs, device=False, stream=None):
    keep = [s.decoded([to_device(p) for p in s.planes]) if device else s.decoded() for s in srcs]
    if device:
        torch.cuda.synchronize()
    arena, images = pigo_b200.gray_images(keep, stream=stream, device_sources=device)
    return arena, images, keep


def test_every_new_format_is_the_reference_gray_image(sources):
    assert {s.planes[0].ctypes.data % 16 for s in sources} >= {0, 1, 3, 5, 7, 15}
    arena, images, _ = convert(sources)
    for s, im in zip(sources, images):
        assert (im.Rows, im.Cols, im.Dim) == (s.h, s.w, s.w)
        assert np.array_equal(slot(arena, im), s.want), (s.fmt, s.w, s.h, s.strides)


def test_palette_indices_past_a_short_palette_give_zero():
    idx = np.arange(256, dtype=np.uint8).reshape(8, 32)
    pal = np.array([[255, 255, 255, 255], [200, 100, 50, 255], [10, 20, 30, 128]], dtype=np.uint8)
    s = WideSrc(PALETTED, 32, 8, (idx.reshape(-1), pal.reshape(-1)), (32, 3))
    arena, images, _ = convert([s])
    got = slot(arena, images[0])
    assert np.array_equal(got, s.want)
    assert got.reshape(-1)[0] == 255 and not got.reshape(-1)[3:].any()


def narrow_sources():
    return [ycbcr_src(2, 45, 31, 3, 1, 11), rgba_src(1, 33, 20, 12, 30), rgba_src(2, 29, 31, 8, 40, alpha=premultiplied_alpha(31, 29, 40)),
            gray_src(45, 19, 3, 51)]


def test_all_nine_formats_in_one_call_share_slots_and_write_nothing_else(sources):
    nine = narrow_sources() + [sources[k] for k in (4, 12, 20, 28, 36)]
    assert sorted({s.fmt for s in nine}) == [0, 1, 2, 3, 5, 6, 7, 8, 9]
    picks = [nine[k] for k in (8, 0, 4, 5, 8, 1, 6, 2, 7, 3, 4, 0)]
    decoded = [p.decoded() for p in picks]
    need = pigo_b200.gray_images_bytes(decoded)
    assert need == sum((s.w * s.h + 255) // 256 * 256 for s in nine)
    buf = torch.full((need + 4096,), 0xEE, dtype=torch.uint8, device="cuda")
    imgs = (pigo_b200.PigoImage * len(decoded))()
    size = C.c_size_t(need)
    before = pigo_b200.launch_count()
    assert pigo_b200.lib().pigo_gray_images(pigo_b200.decoded_descs(decoded), len(decoded), buf.data_ptr(), C.byref(size), imgs, 0, None) == 0
    assert pigo_b200.launch_count() - before == 2   # one launch for each kernel
    host = buf.cpu().numpy()
    written = np.zeros(host.size, dtype=bool)
    for p, im in zip(picks, imgs):
        off = im.pixels - buf.data_ptr()
        assert np.array_equal(host[off:off + p.w * p.h].reshape(p.h, p.w), p.want), p.fmt
        written[off:off + p.w * p.h] = True
    assert imgs[0].pixels == imgs[4].pixels and imgs[1].pixels == imgs[11].pixels and imgs[2].pixels == imgs[10].pixels
    assert len({im.pixels for im in imgs}) == 9
    assert (host[~written] == 0xEE).all()


def test_host_and_device_planes_give_the_same_arena(sources):
    a_host, i_host, _ = convert(sources)
    a_sync, i_sync, _ = convert(sources, device=True)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        a_dev, i_dev, keep = convert(sources, device=True, stream=s)
    s.synchronize()
    for ih, isy, idv in zip(i_host, i_sync, i_dev):
        assert np.array_equal(slot(a_host, ih), slot(a_sync, isy))
        assert np.array_equal(slot(a_host, ih), slot(a_dev, idv))
    assert [im.Pixels - a_host.data_ptr() for im in i_host] == [im.Pixels - a_dev.data_ptr() for im in i_dev]


# ---- detection on the converted images ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cascades():
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
    names = sorted(set(pipeline.EYE_CASCADES + pipeline.MOUTH_CASCADES))
    flp = {n: pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("lps/" + n)) for n in names}
    return plc, flp


@pytest.fixture(scope="module")
def face_sources():
    shapes = [(640, 480, 16, 0), (320, 400, 0, 3), (961, 541, 7, 1), (500, 300, 0, 0), (700, 450, 5, 9)]
    out = []
    for k, (fmt, (w, h, pad, off)) in enumerate(zip((GRAY16, RGBA64, NRGBA64, CMYK, PALETTED), shapes)):
        g = synth.sample_gray() if (h, w) == (400, 320) else face_gray(h, w, 60 + k)
        s = wide_src(fmt, w, h, pad, off, seed=60 + k, luma=g)
        assert np.array_equal(s.want, g), fmt
        out.append(s)
    return out


def test_run_cascade_on_each_new_format_equals_host_gray(gpu_face, face_sources):
    cp = CascadeParams(ImageParams(), *TEST_PARAMS)
    angles = [0.0, 0.05, 0.0, 0.3, 0.0]
    arena, images, _ = convert(face_sources)
    got, n = gpu_face.RunCascadeImagesAngles(images, cp, angles, 512)
    want, m = gpu_face.RunCascadeImagesAngles(host_images(face_sources), cp, angles, 512)
    assert np.array_equal(n, m) and got.tobytes() == want.tobytes()
    assert n.sum() > 0


def test_detect_on_each_new_format_equals_host_gray(gpu_face, cascades, face_sources):
    plc, flp = cascades
    cp = CascadeParams(ImageParams(), *TEST_PARAMS)
    arena, images, _ = convert(face_sources)
    angles = [0.0] * len(face_sources)
    rnd = np.random.default_rng(71).random((len(face_sources), 16, 2 + NCALLS, 63, 3), dtype=np.float32)
    got = pipeline.detect_images_angles_device(gpu_face, plc, flp, images, cp, angles, face_cap=16, randoms=rnd, raw=True)
    want = pipeline.detect_images_angles_device(gpu_face, plc, flp, host_images(face_sources), cp, angles, face_cap=16, randoms=rnd, raw=True)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want))
    assert got[1].sum() > 0


def test_detect_decoded_on_a_mixed_list(gpu_face, cascades, face_sources):
    plc, flp = cascades
    srcs = face_sources + [ycbcr_src(2, 320, 400, 1, 1, 24, luma=synth.sample_gray()), face_sources[1]]
    cp = CascadeParams(ImageParams(), *TEST_PARAMS)
    rnd = np.random.default_rng(91).random((len(srcs), 8, 2 + NCALLS, 63, 3), dtype=np.float32)
    got = pipeline.detect_decoded(gpu_face, plc, flp, [s.decoded() for s in srcs], cp, face_cap=8, randoms=rnd, raw=True)
    want = pipeline.detect_images_angles_device(gpu_face, plc, flp, host_images(srcs), cp, [0.0] * len(srcs), face_cap=8, randoms=rnd, raw=True)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want))
    assert got[1].sum() > 0
