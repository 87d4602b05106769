"""pigo_gray_images for *image.Gray16, RGBA64, NRGBA64, CMYK and Paletted on the H100: every slot is the oracle's
RgbToGrayscale(ImgToNRGBA(img)) byte for byte over odd sizes, padded strides and unaligned planes; a call mixing all nine
formats shares slots and writes nothing else; host and device planes give the same arena; and detection on the converted
images equals detection on the oracle-made host gray images."""
import ctypes as C

import numpy as np
import pytest
import torch

import pigo_b200
from decoded_sources import PALETTED, WideSrc, face_sources, host_images, narrow_sources, slot, wide_sources, ycbcr_src  # noqa: F401
from mixed_images import NCALLS, TEST_PARAMS, cascades   # noqa: F401 (fixture)
from pigo_b200 import CascadeParams, ImageParams, pipeline, synth
from option_guard import options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)

pytestmark = pytest.mark.gpu


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


def test_every_new_format_is_the_reference_gray_image(wide_sources):
    assert {s.planes[0].ctypes.data % 16 for s in wide_sources} >= {0, 1, 3, 5, 7, 15}
    arena, images, _ = convert(wide_sources)
    for s, im in zip(wide_sources, images):
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


def test_all_nine_formats_in_one_call_share_slots_and_write_nothing_else(wide_sources):
    nine = narrow_sources() + [wide_sources[k] for k in (4, 12, 20, 28, 36)]
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


def test_host_and_device_planes_give_the_same_arena(wide_sources):
    a_host, i_host, _ = convert(wide_sources)
    a_sync, i_sync, _ = convert(wide_sources, device=True)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        a_dev, i_dev, keep = convert(wide_sources, device=True, stream=s)
    s.synchronize()
    for ih, isy, idv in zip(i_host, i_sync, i_dev):
        assert np.array_equal(slot(a_host, ih), slot(a_sync, isy))
        assert np.array_equal(slot(a_host, ih), slot(a_dev, idv))
    assert [im.Pixels - a_host.data_ptr() for im in i_host] == [im.Pixels - a_dev.data_ptr() for im in i_dev]


# ---- detection on the converted images ---------------------------------------------------------------------------------
def test_run_cascade_on_each_new_format_equals_host_gray(gpu_face, face_sources):
    cp = CascadeParams(ImageParams(), *TEST_PARAMS)
    angles = [0.0, 0.05, 0.0, 0.3, 0.0]
    arena, images, _ = convert(face_sources)
    got, n = gpu_face.RunCascadeImagesAngles(images, cp, angles, 512)
    want, m = gpu_face.RunCascadeImagesAngles(host_images(face_sources), cp, angles, 512)
    assert np.array_equal(n, m) and got.tobytes() == want.tobytes()
    assert n.sum() > 0


def test_detect_on_each_new_format_equals_host_gray(gpu_face, cascades, face_sources):
    plc, flp, _, _ = cascades
    cp = CascadeParams(ImageParams(), *TEST_PARAMS)
    arena, images, _ = convert(face_sources)
    angles = [0.0] * len(face_sources)
    rnd = np.random.default_rng(71).random((len(face_sources), 16, 2 + NCALLS, 63, 3), dtype=np.float32)
    got = pipeline.detect_images_angles_device(gpu_face, plc, flp, images, cp, angles, face_cap=16, randoms=rnd, raw=True)
    want = pipeline.detect_images_angles_device(gpu_face, plc, flp, host_images(face_sources), cp, angles, face_cap=16, randoms=rnd, raw=True)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want))
    assert got[1].sum() > 0


def test_detect_decoded_on_a_mixed_list(gpu_face, cascades, face_sources):
    plc, flp, _, _ = cascades
    srcs = face_sources + [ycbcr_src(2, 320, 400, 1, 1, 24, luma=synth.sample_gray()), face_sources[1]]
    cp = CascadeParams(ImageParams(), *TEST_PARAMS)
    rnd = np.random.default_rng(91).random((len(srcs), 8, 2 + NCALLS, 63, 3), dtype=np.float32)
    got = pipeline.detect_decoded(gpu_face, plc, flp, [s.decoded() for s in srcs], cp, face_cap=8, randoms=rnd, raw=True)
    want = pipeline.detect_images_angles_device(gpu_face, plc, flp, host_images(srcs), cp, [0.0] * len(srcs), face_cap=8, randoms=rnd, raw=True)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want))
    assert got[1].sum() > 0
