"""pigo_gray_images on the H100: every slot is RgbToGrayscale(ImgToNRGBA(img)) byte for byte (oracle composition and the
single-image conversions), host and device sources give the same arena, repeated sources share a slot, nothing outside the
slots is written, and detection on the converted device images equals detection on the oracle-made host gray images."""
import ctypes as C

import numpy as np
import pytest
import torch

import pigo_b200
from decoded_sources import eight_bit_sources, host_images, slot   # noqa: F401 (fixture)
from mixed_images import NCALLS, TEST_PARAMS, cascades   # noqa: F401 (fixture)
from pigo_b200 import CascadeParams, ImageParams, pipeline
from option_guard import options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)

pytestmark = pytest.mark.gpu


def convert(srcs, device=False, stream=None):
    keep = []
    if device:   # every plane uploaded as it is laid out on the host
        for s in srcs:
            keep.append(s.decoded([torch.from_numpy(p).cuda() for p in s.planes]))
        torch.cuda.synchronize()
    else:
        keep = [s.decoded() for s in srcs]
    arena, images = pigo_b200.gray_images(keep, stream=stream, device_sources=device)
    return arena, images, keep


def test_every_slot_is_the_reference_gray_image(eight_bit_sources):
    sources = eight_bit_sources
    assert len(sources) >= 24 and {s.fmt for s in sources} == {0, 1, 2, 3} and {s.sub for s in sources if s.fmt == 0} == set(range(6))
    arena, images, _ = convert(eight_bit_sources)
    assert arena.numel() == sum((s.w * s.h + 255) // 256 * 256 for s in eight_bit_sources)
    for s, im in zip(eight_bit_sources, images):
        assert (im.Rows, im.Cols, im.Dim) == (s.h, s.w, s.w)
        assert (im.Pixels - arena.data_ptr()) % 256 == 0 and im.Pixels % 256 == 0
        assert np.array_equal(slot(arena, im), s.want), (s.fmt, s.w, s.h, s.sub)


def test_single_image_conversions_agree(eight_bit_sources):
    arena, images, _ = convert(eight_bit_sources)
    for s, im in zip(eight_bit_sources, images):
        if s.fmt == 0:
            y = s.planes[0].reshape(s.h, s.strides[0])
            c = s.planes[1].reshape(-1, s.strides[1])
            _, g = pigo_b200.YCbCrToNRGBA(y, c, s.planes[2].reshape(-1, s.strides[1]), s.sub, s.w, s.h, s.min_x, s.min_y, want_gray=True)
        elif s.fmt == 1:
            g = pigo_b200.RgbToGrayscale(s.planes[0].reshape(s.h, s.strides[0])[:, :4 * s.w].reshape(s.h, s.w, 4))
        else:
            continue
        assert np.array_equal(slot(arena, im), g)


def test_host_and_device_sources_give_the_same_arena(eight_bit_sources):
    a_host, i_host, _ = convert(eight_bit_sources)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        a_dev, i_dev, keep = convert(eight_bit_sources, device=True, stream=s)
    s.synchronize()
    for ih, idv in zip(i_host, i_dev):
        assert np.array_equal(slot(a_host, ih), slot(a_dev, idv))
    assert [im.Pixels - a_host.data_ptr() for im in i_host] == [im.Pixels - a_dev.data_ptr() for im in i_dev]


def test_repeats_share_a_slot_and_nothing_else_is_written(eight_bit_sources):
    picks = [eight_bit_sources[k] for k in (0, 10, 3, 10, 0, 17, 14, 14, 22)]
    decoded = [p.decoded() for p in picks]
    need = pigo_b200.gray_images_bytes(decoded)
    assert need == sum((s.w * s.h + 255) // 256 * 256 for s in {id(p): p for p in picks}.values())
    buf = torch.full((need + 4096,), 0xEE, dtype=torch.uint8, device="cuda")
    imgs = (pigo_b200.PigoImage * len(decoded))()
    size = C.c_size_t(need - 1)
    L = pigo_b200.lib()
    assert L.pigo_gray_images(pigo_b200.decoded_descs(decoded), len(decoded), buf.data_ptr(), C.byref(size), imgs, 0, None) == pigo_b200.PIGO_E_CAP
    assert size.value == need
    assert L.pigo_gray_images(pigo_b200.decoded_descs(decoded), len(decoded), buf.data_ptr(), C.byref(size), imgs, 0, None) == pigo_b200.PIGO_OK
    host = buf.cpu().numpy()
    written = np.zeros(host.size, dtype=bool)
    for p, im in zip(picks, imgs):
        off = im.pixels - buf.data_ptr()
        assert np.array_equal(host[off:off + p.w * p.h].reshape(p.h, p.w), p.want)
        written[off:off + p.w * p.h] = True
    assert [im.pixels for im in imgs][1] == imgs[3].pixels and imgs[0].pixels == imgs[4].pixels and imgs[6].pixels == imgs[7].pixels
    assert len({im.pixels for im in imgs}) == 6
    assert (host[~written] == 0xEE).all()


def test_a_capturing_stream_is_refused(eight_bit_sources):
    decoded = [s.decoded() for s in eight_bit_sources[:3]]
    buf = torch.empty(pigo_b200.gray_images_bytes(decoded), dtype=torch.uint8, device="cuda")
    imgs = (pigo_b200.PigoImage * 3)()
    size = C.c_size_t(buf.numel())
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="relaxed"):
        rc = pigo_b200.lib().pigo_gray_images(pigo_b200.decoded_descs(decoded), 3, buf.data_ptr(), C.byref(size), imgs, 0, s.cuda_stream)
    assert rc == pigo_b200.PIGO_E_INVALID


# ---- detection on the converted images ---------------------------------------------------------------------------------
def detection_cases(sources):
    faces = [s for s in sources if s.w * s.h >= 200 * 200]
    wide = [s for s in faces if s.w > s.h]
    assert len(wide) >= 3
    sweep = [wide[0]] * 5 + [faces[0]]
    return [(faces, [0.0] * len(faces)), (sweep, [0.0, 0.02, 0.05, 0.25, 0.7, 0.0]), (wide, [0.3, 0.05, 1.0][:len(wide)] + [0.2] * (len(wide) - 3))]


def test_run_cascade_on_converted_images_equals_host_gray(gpu_face, eight_bit_sources):
    cp = CascadeParams(ImageParams(), *TEST_PARAMS)
    for srcs, angles in detection_cases(eight_bit_sources):
        arena, images, _ = convert(srcs)
        assert len({im.Pixels for im in images}) == len({id(s) for s in srcs})
        got, n = gpu_face.RunCascadeImagesAngles(images, cp, angles, 512)
        want, m = gpu_face.RunCascadeImagesAngles(host_images(srcs), cp, angles, 512)
        assert np.array_equal(n, m) and got.tobytes() == want.tobytes()
        assert n.sum() > 0


def test_detect_on_converted_images_equals_host_gray(gpu_face, cascades, eight_bit_sources):
    plc, flp, _, _ = cascades
    cp = CascadeParams(ImageParams(), *TEST_PARAMS)
    for k, (srcs, angles) in enumerate(detection_cases(eight_bit_sources)):
        arena, images, _ = convert(srcs)
        rnd = np.random.default_rng(70 + k).random((len(srcs), 16, 2 + NCALLS, 63, 3), dtype=np.float32)
        got = pipeline.detect_images_angles_device(gpu_face, plc, flp, images, cp, angles, face_cap=16, randoms=rnd, raw=True)
        want = pipeline.detect_images_angles_device(gpu_face, plc, flp, host_images(srcs), cp, angles, face_cap=16, randoms=rnd, raw=True)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want))
        assert got[1].sum() > 0


def test_device_sources_on_a_caller_stream_feed_an_asynchronous_detect(gpu_face, cascades, eight_bit_sources):
    """pigo_gray_images from device planes returns without synchronising; pigo_detect_images(PIGO_OUT_DEVICE) on the same
    stream, with no sync in between, sees the finished arena."""
    plc, flp, _, _ = cascades
    srcs = [s for s in eight_bit_sources if s.w * s.h >= 200 * 200]
    face_cap = 16
    rnd = np.random.default_rng(80).random((len(srcs), face_cap, 2 + NCALLS, 63, 3), dtype=np.float32)
    want = pipeline.detect_images_device(gpu_face, plc, flp, host_images(srcs), CascadeParams(ImageParams(), *TEST_PARAMS), face_cap=face_cap,
                                         randoms=rnd, raw=True)
    hs, fl = pipeline.landmark_call_arrays(flp)
    prm = pigo_b200.PipelineParams(*TEST_PARAMS[:4], 0.0, 0.1, 50, 50, 63, 0)
    n = len(srcs)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        planes = [s_.decoded([torch.from_numpy(p).cuda() for p in s_.planes]) for s_ in srcs]
        d_rnd = torch.from_numpy(rnd).cuda()
        faces = torch.zeros((n, face_cap, 4), dtype=torch.int32, device="cuda")
        nfaces = torch.zeros(n, dtype=torch.int32, device="cuda")
        points = torch.zeros((n, face_cap, 2 + NCALLS, 4), dtype=torch.int32, device="cuda")
        arena, images = pigo_b200.gray_images(planes, stream=s, device_sources=True)
        desc = pigo_b200.image_descs(images)
        pigo_b200._check(pigo_b200.lib().pigo_detect_images(gpu_face._h, plc._h, hs, fl.ctypes.data, NCALLS, desc, n, C.byref(prm), d_rnd.data_ptr(), 0,
                                                            faces.data_ptr(), face_cap, nfaces.data_ptr(), points.data_ptr(),
                                                            pigo_b200.FRAMES_DEVICE | pigo_b200.OUT_DEVICE, s.cuda_stream))
    s.synchronize()
    assert faces.cpu().numpy().tobytes() == want[0].tobytes()
    assert nfaces.cpu().numpy().tobytes() == want[1].tobytes()
    assert points.cpu().numpy().tobytes() == want[2].tobytes()


def test_detect_decoded_mirror(gpu_face, cascades, eight_bit_sources):
    plc, flp, _, _ = cascades
    srcs = [s for s in eight_bit_sources if s.w * s.h >= 200 * 200][:3]
    cp = CascadeParams(ImageParams(), *TEST_PARAMS)
    rnd = np.random.default_rng(90).random((len(srcs), 8, 2 + NCALLS, 63, 3), dtype=np.float32)
    got = pipeline.detect_decoded(gpu_face, plc, flp, [s.decoded() for s in srcs], cp, face_cap=8, randoms=rnd, raw=True)
    want = pipeline.detect_images_angles_device(gpu_face, plc, flp, host_images(srcs), cp, [0.0] * len(srcs), face_cap=8, randoms=rnd, raw=True)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want))
