"""Inputs and byte-equality checks shared by the GPU suites of the mixed-size entry points (images, angles, sweep, sharded,
detect images, decoded images): parameter sets, image tables, one image maker, lone reference calls, and the cascades
fixture."""
import os
import subprocess

import numpy as np
import pytest

import pigo_b200
from pigo_b200 import CascadeParams, ImageParams, pipeline, synth
from pipeline_oracle import oracle_cascades

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TEST_PARAMS = (20, 1000, 0.2, 1.1)   # core/pigo_test.go:44-50 (eye Perturbs 50, core/flploc_test.go:107)
DOC_PARAMS = (20, 1000, 0.1, 1.1)    # README
CLI_PARAMS = (20, 1000, 0.15, 1.15)  # cmd/pigo/main.go:110-111 (eye Perturbs 63)
EYE = {TEST_PARAMS: 50, CLI_PARAMS: 63}
NCALLS = 15

# (rows, cols, dim, content class): no windows (1x1, 10x10, 21 rows), exactly one window (22x22), the sample, common sizes
# up to 4K, odd sizes and strides (dim > cols), wide and tall shapes
MIXED = [(1, 1, 1, "U"), (10, 10, 10, "U"), (22, 22, 22, "U"), (400, 320, 320, "sample"), (480, 640, 640, "F"),
         (720, 1280, 1280, "S"), (1080, 1920, 1920, "F"), (2160, 3840, 3840, "F"), (97, 131, 160, "U"), (333, 517, 531, "F"),
         (240, 320, 320, "S"), (600, 800, 800, "F"), (123, 777, 800, "U"), (50, 60, 64, "S"), (768, 1024, 1024, "U"),
         (301, 299, 301, "F"), (1080, 1920, 1920, "S"), (45, 1200, 1216, "F"), (900, 41, 48, "U"), (360, 640, 640, "F"),
         (511, 383, 400, "S"), (200, 200, 200, "F"), (64, 64, 80, "U"), (1000, 700, 701, "F"), (150, 1500, 1500, "S"),
         (480, 640, 700, "U"), (21, 300, 300, "F"), (272, 480, 496, "F"), (540, 960, 960, "U"), (333, 250, 256, "S")]

# the pipeline's images: no windows (10x10, 21 rows), the sample, face frames of several sizes with dim > cols, 1080p, one 4K
# frame, tall and wide shapes, noise and smooth content
GEOMS = [(10, 10, 10, "U"), (21, 300, 300, "U"), (400, 320, 320, "sample"), (540, 960, 960, "F"), (480, 640, 656, "F"),
         (333, 517, 531, "F"), (1080, 1920, 1920, "F"), (2160, 3840, 3840, "F"), (700, 260, 272, "F"), (300, 900, 912, "F"),
         (600, 800, 800, "F"), (45, 1200, 1216, "U"), (360, 640, 640, "S"), (272, 480, 496, "F"), (1000, 700, 701, "F"),
         (200, 200, 200, "F"), (900, 41, 48, "U"), (50, 60, 64, "S"), (768, 1024, 1024, "U"), (301, 299, 301, "F")]


# scan options under which a mixed-size call must give the same outputs
KNOBS = [{"queue_cap": 1}, {"queue_cap": 16, "gather_ks": 2}, {"gather_ks": 8}, {"gather_block": 8}, {"gather_block": 16},
         {"deep_group": 8}, {"deep_group": 32}, {"gather_ctas_per_sm": 1}, {"gather_ni": 2}, {"gather_ni": 3}, {"gather_limit": 3},
         {"sub_batch": 4},                     # several groups of images per call
         {"scan_mode": 1}, {"rot_mode": 1}]    # universal kernel: the single-image path, image by image


def make_image(rows, cols, dim, cls, seed) -> ImageParams:
    if cls == "sample":
        return ImageParams(synth.sample_gray(), rows, cols, dim)
    buf = np.full((rows, dim), 0xA5, dtype=np.uint8)   # the bytes past Cols are never read
    if cls == "U":
        buf[:, :cols] = synth.frame_noise(rows, cols, seed)
    elif cls == "S":
        buf[:, :cols] = synth.frame_smooth(rows, cols, seed)
    else:
        buf[:, :cols] = synth.frame_faces(None, rows, cols, shift=((37 * seed) % 400, (53 * seed) % 320), noise_seed=seed)
    return ImageParams(buf, rows, cols, dim)


def cp_of(params=TEST_PARAMS):
    return CascadeParams(ImageParams(), *params)


def canonical(a):
    """The angle the reference scans at (core/pigo.go:232-238): <= 0 and NaN unrotated, > 1 clamped to 1."""
    return 0.0 if not a > 0 else min(a, 1.0)


def randoms_for(n, face_cap, seed):
    return np.random.default_rng(seed).random((n, face_cap, 2 + NCALLS, 63, 3), dtype=np.float32)


def lone_scan(face, im, params, angle=0.0):
    """pigo_run_cascade on one image."""
    return face.run_cascade_array(CascadeParams(im, *params), angle)


def lone_detect_batch(gpu_face, cascades, im, params, face_cap, randoms, angle, eye):
    """pigo_detect_batch on one image (nframes = 1), raw outputs."""
    plc, flp, _, _ = cascades
    frame = np.ascontiguousarray(im.Pixels).reshape(1, im.Rows, im.Dim)
    cp = CascadeParams(ImageParams(None, im.Rows, im.Cols, im.Dim), *params)
    return pipeline.detect_batch_device(gpu_face, plc, flp, frame, cp, face_cap=face_cap, randoms=randoms, angle=angle, eye_perturbs=eye, raw=True)


def assert_slices(dets, cnt, expect):
    assert len(cnt) == len(expect)
    for i, e in enumerate(expect):
        assert int(cnt[i]) == len(e), f"image {i}: {int(cnt[i])} detections vs {len(e)}"
        assert dets[i, :len(e)].tobytes() == e.tobytes(), f"image {i} differs"


def assert_same_outputs(a, b, idx_a=None, idx_b=None):
    fa, na, pa = a
    fb, nb, pb = b
    ia = range(len(na)) if idx_a is None else idx_a
    ib = range(len(nb)) if idx_b is None else idx_b
    for i, j in zip(ia, ib):
        assert int(na[i]) == int(nb[j]), (i, j)
        assert fa[i].tobytes() == fb[j].tobytes(), f"faces of image {i} differ"
        assert pa[i].tobytes() == pb[j].tobytes(), f"points of image {i} differ"


def same(a, b):
    return all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def run_cpp_mirror(name, *args, timeout=300):
    """Runs the C++ mirror test tests/cpp/<name> (built by __graft_entry__.build(), run here if it is missing) with the
    repository root and args; returns its stdout."""
    exe = os.path.join(ROOT, "tests", "cpp", name)
    if not os.path.exists(exe):
        import __graft_entry__
        __graft_entry__.build()
    r = subprocess.run([exe, ROOT, *map(str, args)], capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


def image_of(im: ImageParams):
    """(pixels, rows, cols, dim), the oracle's form of an image."""
    return im.Pixels, im.Rows, im.Cols, im.Dim


@pytest.fixture(scope="module")
def images():
    return [make_image(r, c, d, k, 21 + i) for i, (r, c, d, k) in enumerate(GEOMS)]


@pytest.fixture(scope="module")
def cascades():
    """(puploc, {name: landmark cascade}) on the GPU, then the same on the C oracle."""
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
    names = sorted(set(pipeline.EYE_CASCADES + pipeline.MOUTH_CASCADES))
    flp = {n: pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("lps/" + n)) for n in names}
    return (plc, flp) + oracle_cascades()
