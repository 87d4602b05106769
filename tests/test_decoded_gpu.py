"""pigo_gray_images on the H100: every slot is RgbToGrayscale(ImgToNRGBA(img)) byte for byte (oracle composition and the
single-image conversions), host and device sources give the same arena, repeated sources share a slot, nothing outside the
slots is written, and detection on the converted device images equals detection on the oracle-made host gray images."""
import ctypes as C

import numpy as np
import pytest
import torch

import decoded_oracle as D
import oracle_lib as O
import pigo_b200
from pigo_b200 import CascadeParams, DecodedImage, ImageParams, pipeline, synth
from option_guard import options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)

pytestmark = pytest.mark.gpu

TEST_PARAMS = (20, 1000, 0.2, 1.1)   # core/pigo_test.go:44-50
NCALLS = 15


def face_gray(h, w, seed):
    return synth.frame_faces(synth.sample_gray(), h, w, shift=(seed % 7 * 5, seed % 5 * 9), noise_seed=seed)


class Src:
    """One decoded source: host planes (flat buffers from the rectangle's origin), the pigo_decoded fields and the oracle's gray."""

    def __init__(self, fmt, w, h, planes, strides, sub=0, min_x=0, min_y=0):
        self.fmt, self.w, self.h, self.planes, self.strides, self.sub, self.min_x, self.min_y = fmt, w, h, planes, strides, sub, min_x, min_y
        self.want = D.decoded_gray(fmt, planes, strides, w, h, sub, min_x, min_y)

    def decoded(self, planes=None):
        return DecodedImage(self.fmt, self.w, self.h, tuple(planes or self.planes), self.strides, self.sub, self.min_x, self.min_y)


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


@pytest.fixture(scope="module")
def sources():
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


def convert(sources, device=False, stream=None):
    keep = []
    if device:   # every plane uploaded as it is laid out on the host
        for s in sources:
            keep.append(s.decoded([torch.from_numpy(p).cuda() for p in s.planes]))
        torch.cuda.synchronize()
    else:
        keep = [s.decoded() for s in sources]
    arena, images = pigo_b200.gray_images(keep, stream=stream, device_sources=device)
    return arena, images, keep


def slot(arena, im):
    off = im.Pixels - arena.data_ptr()
    return arena[off:off + im.Rows * im.Cols].cpu().numpy().reshape(im.Rows, im.Cols)


def test_every_slot_is_the_reference_gray_image(sources):
    assert len(sources) >= 24 and {s.fmt for s in sources} == {0, 1, 2, 3} and {s.sub for s in sources if s.fmt == 0} == set(range(6))
    arena, images, _ = convert(sources)
    assert arena.numel() == sum((s.w * s.h + 255) // 256 * 256 for s in sources)
    for s, im in zip(sources, images):
        assert (im.Rows, im.Cols, im.Dim) == (s.h, s.w, s.w)
        assert (im.Pixels - arena.data_ptr()) % 256 == 0 and im.Pixels % 256 == 0
        assert np.array_equal(slot(arena, im), s.want), (s.fmt, s.w, s.h, s.sub)


def test_single_image_conversions_agree(sources):
    arena, images, _ = convert(sources)
    for s, im in zip(sources, images):
        if s.fmt == 0:
            y = s.planes[0].reshape(s.h, s.strides[0])
            c = s.planes[1].reshape(-1, s.strides[1])
            _, g = pigo_b200.YCbCrToNRGBA(y, c, s.planes[2].reshape(-1, s.strides[1]), s.sub, s.w, s.h, s.min_x, s.min_y, want_gray=True)
        elif s.fmt == 1:
            g = pigo_b200.RgbToGrayscale(s.planes[0].reshape(s.h, s.strides[0])[:, :4 * s.w].reshape(s.h, s.w, 4))
        else:
            continue
        assert np.array_equal(slot(arena, im), g)


def test_host_and_device_sources_give_the_same_arena(sources):
    a_host, i_host, _ = convert(sources)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        a_dev, i_dev, keep = convert(sources, device=True, stream=s)
    s.synchronize()
    for ih, idv in zip(i_host, i_dev):
        assert np.array_equal(slot(a_host, ih), slot(a_dev, idv))
    assert [im.Pixels - a_host.data_ptr() for im in i_host] == [im.Pixels - a_dev.data_ptr() for im in i_dev]


def test_repeats_share_a_slot_and_nothing_else_is_written(sources):
    picks = [sources[k] for k in (0, 10, 3, 10, 0, 17, 14, 14, 22)]
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


def test_a_capturing_stream_is_refused(sources):
    decoded = [s.decoded() for s in sources[:3]]
    buf = torch.empty(pigo_b200.gray_images_bytes(decoded), dtype=torch.uint8, device="cuda")
    imgs = (pigo_b200.PigoImage * 3)()
    size = C.c_size_t(buf.numel())
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="relaxed"):
        rc = pigo_b200.lib().pigo_gray_images(pigo_b200.decoded_descs(decoded), 3, buf.data_ptr(), C.byref(size), imgs, 0, s.cuda_stream)
    assert rc == pigo_b200.PIGO_E_INVALID


# ---- detection on the converted images ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cascades():
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
    names = sorted(set(pipeline.EYE_CASCADES + pipeline.MOUTH_CASCADES))
    flp = {n: pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("lps/" + n)) for n in names}
    return plc, flp


def host_images(srcs):
    return [ImageParams(s.want.reshape(-1), s.h, s.w, s.w) for s in srcs]


def detection_cases(sources):
    faces = [s for s in sources if s.w * s.h >= 200 * 200]
    wide = [s for s in faces if s.w > s.h]
    assert len(wide) >= 3
    sweep = [wide[0]] * 5 + [faces[0]]
    return [(faces, [0.0] * len(faces)), (sweep, [0.0, 0.02, 0.05, 0.25, 0.7, 0.0]), (wide, [0.3, 0.05, 1.0][:len(wide)] + [0.2] * (len(wide) - 3))]


def test_run_cascade_on_converted_images_equals_host_gray(gpu_face, sources):
    cp = CascadeParams(ImageParams(), *TEST_PARAMS)
    for srcs, angles in detection_cases(sources):
        arena, images, _ = convert(srcs)
        assert len({im.Pixels for im in images}) == len({id(s) for s in srcs})
        got, n = gpu_face.RunCascadeImagesAngles(images, cp, angles, 512)
        want, m = gpu_face.RunCascadeImagesAngles(host_images(srcs), cp, angles, 512)
        assert np.array_equal(n, m) and got.tobytes() == want.tobytes()
        assert n.sum() > 0


def test_detect_on_converted_images_equals_host_gray(gpu_face, cascades, sources):
    plc, flp = cascades
    cp = CascadeParams(ImageParams(), *TEST_PARAMS)
    for k, (srcs, angles) in enumerate(detection_cases(sources)):
        arena, images, _ = convert(srcs)
        rnd = np.random.default_rng(70 + k).random((len(srcs), 16, 2 + NCALLS, 63, 3), dtype=np.float32)
        got = pipeline.detect_images_angles_device(gpu_face, plc, flp, images, cp, angles, face_cap=16, randoms=rnd, raw=True)
        want = pipeline.detect_images_angles_device(gpu_face, plc, flp, host_images(srcs), cp, angles, face_cap=16, randoms=rnd, raw=True)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want))
        assert got[1].sum() > 0


def test_device_sources_on_a_caller_stream_feed_an_asynchronous_detect(gpu_face, cascades, sources):
    """pigo_gray_images from device planes returns without synchronising; pigo_detect_images(PIGO_OUT_DEVICE) on the same
    stream, with no sync in between, sees the finished arena."""
    plc, flp = cascades
    srcs = [s for s in sources if s.w * s.h >= 200 * 200]
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


def test_detect_decoded_mirror(gpu_face, cascades, sources):
    plc, flp = cascades
    srcs = [s for s in sources if s.w * s.h >= 200 * 200][:3]
    cp = CascadeParams(ImageParams(), *TEST_PARAMS)
    rnd = np.random.default_rng(90).random((len(srcs), 8, 2 + NCALLS, 63, 3), dtype=np.float32)
    got = pipeline.detect_decoded(gpu_face, plc, flp, [s.decoded() for s in srcs], cp, face_cap=8, randoms=rnd, raw=True)
    want = pipeline.detect_images_angles_device(gpu_face, plc, flp, host_images(srcs), cp, [0.0] * len(srcs), face_cap=8, randoms=rnd, raw=True)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want))
