"""The deep kernel's queue in image order: a call of more than 4 M windows sorts the deep queue by frame and region and
consumes it in per-CTA runs; a single 1080p frame (0.9 M windows) keeps the one-atomic-per-item order.  Both must give the
same detections, bit for bit, with the default queue and with one so small that every producer overflows it."""
import pytest

import pigo_b200
from pigo_b200 import CascadeParams, ImageParams, synth
from option_guard import options, options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)

pytestmark = pytest.mark.gpu

PARAMS = (20, 1000, 0.2, 1.1)
R, C = 1080, 1920


def _one(gpu_face, img: ImageParams, angle: float):
    return gpu_face.run_cascade_array(CascadeParams(img, *PARAMS), angle)


def _check(dets, cnt, singles):
    for f, one in enumerate(singles):
        assert cnt[f] == len(one) and dets[f, :cnt[f]].tobytes() == one.tobytes(), f"image {f}"


@pytest.mark.parametrize("queue_cap", [0, 50])
def test_ordered_deep_queue_equals_per_frame_calls(gpu_face, oracle_face, queue_cap):
    with options(queue_cap=queue_cap):
        _ordered_deep_queue_equals_per_frame_calls(gpu_face, oracle_face)


def _ordered_deep_queue_equals_per_frame_calls(gpu_face, oracle_face):
    nf = 8   # 7.2 M windows
    frames = synth.make_batch(nf, R, C, "USF", seed0=7)
    cp = CascadeParams(ImageParams(None, R, C, C), *PARAMS)
    for angle in (0.0, 0.25):   # uniform batch: unrotated and rotated deep kernel
        dets, cnt = gpu_face.RunCascadeBatch(frames, cp, angle)
        singles = [_one(gpu_face, ImageParams(frames[f], R, C, C), angle) for f in range(nf)]
        _check(dets, cnt, singles)
        assert sum(len(s) for s in singles) > 0
        for f in (0, 4):
            o = oracle_face.run_cascade(frames[f], R, C, C, *PARAMS, angle)
            assert singles[f].tobytes() == o.tobytes()
    # mixed sizes (5.5 M windows): one angle for the call, then one per image (all rotated: one pass over every image)
    imgs = [ImageParams(frames[i], R - 40 * i, C - 64 * i, C) for i in range(nf)]
    dets, cnt = gpu_face.RunCascadeImages(imgs, cp, 0.0)
    _check(dets, cnt, [_one(gpu_face, im, 0.0) for im in imgs])
    angles = [0.25 + 0.25 * (i % 2) for i in range(nf)]
    dets, cnt = gpu_face.RunCascadeImagesAngles(imgs, cp, angles)
    _check(dets, cnt, [_one(gpu_face, im, a) for im, a in zip(imgs, angles)])
