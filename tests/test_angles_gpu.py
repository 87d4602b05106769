"""pigo_run_cascade_images_angles / pigo_detect_images_angles: every image of a mixed-size call at its own angle.  Bar:
every image's slice equals a lone pigo_run_cascade (scan) or a lone pigo_detect_images (pipeline) at that image's angle,
byte for byte, and the C oracle up to 1080p.  Rotated angles go only on images with Cols >= Rows: on tall images the
rotated column clamp (Rows-1, core/pigo.go:168,:171) indexes past the image, where the reference itself would too."""
import ctypes as C
import math
import threading

import numpy as np
import pytest

import pigo_b200
import pipeline_oracle as P
from mixed_images import (CLI_PARAMS, DOC_PARAMS, KNOBS, MIXED, NCALLS, TEST_PARAMS, assert_slices, canonical, cascades, cp_of, image_of,  # noqa: F401 (fixtures)
                          images, lone_scan, make_image, randoms_for, run_cpp_mirror, same)
from pigo_b200 import ImageParams, pipeline, synth
from option_guard import options, options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)
from synthetic import synthetic_cascade

pytestmark = pytest.mark.gpu

ANGLES = [0.0, -0.1, math.nan, 1 / 64, 1 / 32, 7 / 32, 0.25, 0.5, 31 / 32, 1.0, 1.3, math.inf]
UNROTATED = [0.0, -0.1, math.nan]
SWEEP = [0.0] + [k / 32 for k in range(1, 33)]


def draw_angles(images, seed):
    rng = np.random.default_rng(seed)
    return [float(rng.choice(ANGLES if im.Cols >= im.Rows else UNROTATED)) for im in images]


@pytest.fixture(scope="module")
def mixed():
    return [make_image(r, c, d, k, 11 + i) for i, (r, c, d, k) in enumerate(MIXED)]


@pytest.fixture(scope="module")
def mixed_angles(mixed):
    a = draw_angles(mixed, 5)
    assert sum(x > 0 for x in a) >= 5 and sum(not x > 0 for x in a) >= 5
    return a


@pytest.fixture(scope="module")
def sweep():
    """One 1080p frame and three wide images, each listed at angle 0 and k/32 (k = 1..32), image-major."""
    base = [make_image(1080, 1920, 1920, "F", 3), make_image(300, 900, 900, "F", 5), make_image(480, 640, 700, "F", 8),
            make_image(200, 1200, 1216, "S", 6)]
    return base, [im for im in base for _ in SWEEP], [a for _ in base for a in SWEEP]


def run(face, images, angles, params=TEST_PARAMS, cap=1024):
    return face.RunCascadeImagesAngles(images, cp_of(params), angles, cap)


@pytest.mark.parametrize("params", [TEST_PARAMS, CLI_PARAMS, DOC_PARAMS])
def test_each_image_equals_a_lone_call_at_its_angle(gpu_face, oracle_face, mixed, mixed_angles, params):
    dets, cnt = run(gpu_face, mixed, mixed_angles, params)
    expect = [lone_scan(gpu_face, im, params, a) for im, a in zip(mixed, mixed_angles)]
    assert_slices(dets, cnt, expect)
    assert sum(len(e) for e, a in zip(expect, mixed_angles) if a > 0) > 0
    for i, (im, a) in enumerate(zip(mixed, mixed_angles)):
        if im.Rows * im.Cols <= 1080 * 1920:
            o = oracle_face.run_cascade(im.Pixels, im.Rows, im.Cols, im.Dim, *params, canonical(a))
            assert expect[i].tobytes() == o.tobytes(), f"image {i} at angle {a} differs from the oracle"


def test_sweep_equals_lone_calls_in_either_listing(gpu_face, sweep):
    base, ims, angles = sweep
    d0, c0 = run(gpu_face, ims, angles)
    assert_slices(d0, c0, [lone_scan(gpu_face, im, TEST_PARAMS, a) for im, a in zip(ims, angles)])
    # angle-major: position p lists image p % 4 at angle p // 4, i.e. the image-major entry (p % 4) * 33 + p // 4
    nb, na = len(base), len(SWEEP)
    perm = [(p % nb) * na + p // nb for p in range(nb * na)]
    d1, c1 = run(gpu_face, [ims[j] for j in perm], [angles[j] for j in perm])
    for k, j in enumerate(perm):
        assert c1[k] == c0[j] and d1[k, :c1[k]].tobytes() == d0[j, :c0[j]].tobytes(), (k, j)
    assert (c0[1:na] > 0).sum() > 0


@pytest.mark.parametrize("angle", [0.0, 0.25])
def test_equal_angles_equal_the_images_call(gpu_face, mixed, angle):
    ims = mixed if angle == 0.0 else [im for im in mixed if im.Cols >= im.Rows]
    ed, ec = gpu_face.RunCascadeImages(ims, cp_of(TEST_PARAMS), angle)
    d, c = run(gpu_face, ims, [angle] * len(ims))
    assert np.array_equal(c, ec) and c.sum() > 0
    assert d.tobytes() == ed.tobytes()


def test_repeated_host_descriptors_device_and_stream_forms_agree(gpu_face, sweep):
    import torch
    base, _, _ = sweep
    angles = [0.0, 0.1, 0.5]
    ims = [im for im in base for _ in angles]
    ang = [a for _ in base for a in angles]
    hd, hc = run(gpu_face, ims, ang)
    assert_slices(hd, hc, [lone_scan(gpu_face, im, TEST_PARAMS, a) for im, a in zip(ims, ang)])
    bufs = [torch.from_numpy(np.ascontiguousarray(im.Pixels).reshape(-1)[:im.Rows * im.Dim].copy()).cuda() for im in base]
    dev = [(b.data_ptr(), im.Rows, im.Cols, im.Dim) for b, im in zip(bufs, base) for _ in angles]
    dd, dc = run(gpu_face, [ImageParams(p, r, c, d) for p, r, c, d in dev], ang)
    assert np.array_equal(dc, hc) and dd.tobytes() == hd.tobytes()
    n, cap = len(ims), max(int(hc.max()), 1)
    out = torch.zeros((n, cap, 4), dtype=torch.int32, device="cuda")
    cnt = torch.zeros(n, dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for _ in range(2):   # back-to-back asynchronous calls reuse the same workspace
            gpu_face.run_cascade_images_angles_device(dev, ang, *TEST_PARAMS, out.data_ptr(), cap, cnt.data_ptr(), st.cuda_stream)
    st.synchronize()
    o = out.cpu().numpy().view(np.uint8).reshape(n, cap, 16)
    assert np.array_equal(cnt.cpu().numpy(), hc)
    for i in range(n):
        assert o[i, :hc[i]].tobytes() == hd[i, :hc[i]].tobytes()


@pytest.mark.parametrize("knobs", KNOBS)
def test_options_leave_the_outputs_unchanged(gpu_face, mixed, mixed_angles, knobs):
    ed, ec = run(gpu_face, mixed, mixed_angles)
    with options(**knobs):
        d, c = run(gpu_face, mixed, mixed_angles)
    assert np.array_equal(c, ec)
    for i in range(len(mixed)):
        assert d[i, :c[i]].tobytes() == ed[i, :ec[i]].tobytes(), i


def test_cascade_of_another_depth_takes_the_single_image_path(mixed, mixed_angles):
    face = pigo_b200.NewPigo().Unpack(synthetic_cascade(4, 9, seed=409))
    some, angles = mixed[:12], mixed_angles[:12]
    dets, cnt = run(face, some, angles)
    assert_slices(dets, cnt, [lone_scan(face, im, TEST_PARAMS, a) for im, a in zip(some, angles)])
    assert cnt.sum() > 0


def test_tables_past_the_bound_run_in_passes(gpu_face):
    """A long ladder (scale factor 1.01) makes each node table ~57 MB: 33 slots exceed the 1 GiB bound of one pass, so the
    rotated images run in two passes (two table builds per call), and the results still equal lone calls."""
    params = (20, 1000, 0.2, 1.01)
    ims = [make_image(720, 1280, 1280, "F", 9), make_image(300, 900, 900, "F", 10)]
    angles = [0.0, 1 / 64] + [k / 32 for k in range(1, 33)]
    lst = [im for im in ims for _ in angles]
    ang = [a for _ in ims for a in angles]
    with options(timing=1):
        d, c = run(gpu_face, lst, ang, params)
        builds = pigo_b200.get_option("t_rottab_n")
    assert builds == 2, builds
    assert_slices(d, c, [lone_scan(gpu_face, im, params, a) for im, a in zip(lst, ang)])
    assert c.sum() > 0


def test_capacity_error_reports_the_required_counts(gpu_face, mixed, mixed_angles):
    _, c = run(gpu_face, mixed, mixed_angles)
    assert c.max() > 2
    desc = pigo_b200.image_descs([(im.Pixels.ctypes.data, im.Rows, im.Cols, im.Dim) for im in mixed])
    ang = np.array(mixed_angles, dtype=np.float64)
    out = np.zeros((len(mixed), 2), dtype=pigo_b200.DET_DTYPE)
    cnt = np.zeros(len(mixed), dtype=np.int32)
    rc = pigo_b200.lib().pigo_run_cascade_images_angles(gpu_face._h, desc, len(mixed), ang.ctypes.data, *TEST_PARAMS, out.ctypes.data, 2,
                                                        cnt.ctypes.data, pigo_b200.MEM_HOST, None)
    assert rc == pigo_b200.PIGO_E_CAP
    assert np.array_equal(cnt, c)


def test_concurrent_calls_on_one_classifier(gpu_face, mixed, mixed_angles):
    subsets = [(mixed[i::4], mixed_angles[i::4]) for i in range(4)]
    expect = [run(gpu_face, s, a) for s, a in subsets]
    errors = []

    def work(k):
        try:
            for _ in range(3):
                d, c = run(gpu_face, *subsets[k])
                ed, ec = expect[k]
                if not np.array_equal(c, ec) or d.tobytes() != ed.tobytes():
                    errors.append(k)
        except Exception as e:   # noqa: BLE001
            errors.append(repr(e))

    ts = [threading.Thread(target=work, args=(k,)) for k in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert errors == []


def test_a_sweep_leaves_the_single_image_cache_alone(gpu_face, oracle_face, sweep):
    """One thread, so that the calls reuse one workspace: a lone rotated call, a sweep, the lone call again."""
    base, ims, angles = sweep
    found = 0
    for im, a in ((base[1], 0.6), (base[2], 0.05), (base[0], 1 / 32), (base[0], 2 / 32)):
        before = lone_scan(gpu_face, im, TEST_PARAMS, a)
        run(gpu_face, ims, angles)
        after = lone_scan(gpu_face, im, TEST_PARAMS, a)
        o = oracle_face.run_cascade(im.Pixels, im.Rows, im.Cols, im.Dim, *TEST_PARAMS, a)
        assert before.tobytes() == after.tobytes() == o.tobytes()
        found += len(o)
    assert found > 0


# ---- pipeline ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def image_angles(images):
    """Small tilts as well as large ones, so that rotated eye refinement runs on faces the rotated scan still finds."""
    rng = np.random.default_rng(12)
    return [float(rng.choice([0.0, 0.02, 0.03, 0.05, 0.25, math.nan, -0.2] if im.Cols >= im.Rows else [0.0, -0.2])) for im in images]


@pytest.fixture(scope="module")
def face_cap(gpu_face, cascades, images, image_angles):
    plc, flp, _, _ = cascades
    _, n, _ = pipeline.detect_images_angles_device(gpu_face, plc, flp, images, cp_of(TEST_PARAMS), image_angles, face_cap=256, raw=True)
    return int(max(n.max(), 1))


@pytest.mark.parametrize("stage", [1, 2])
def test_pipeline_each_image_equals_a_lone_detect_images(gpu_face, cascades, images, image_angles, face_cap, stage):
    plc, flp, _, _ = cascades
    with options(puploc_stage=stage):
        rnd = randoms_for(len(images), face_cap, 41)
        got = pipeline.detect_images_angles_device(gpu_face, plc, flp, images, cp_of(TEST_PARAMS), image_angles, face_cap=face_cap,
                                                   randoms=rnd, raw=True)
        for i, (im, a) in enumerate(zip(images, image_angles)):
            one = pipeline.detect_images_device(gpu_face, plc, flp, [im], cp_of(TEST_PARAMS), face_cap=face_cap, randoms=rnd[i:i + 1],
                                                angle=a, raw=True)
            assert int(got[1][i]) == int(one[1][0]), i
            assert got[0][i].tobytes() == one[0][0].tobytes() and got[2][i].tobytes() == one[2][0].tobytes(), (i, a)
    faces, nfaces, _ = got
    rotated_refined = [i for i, a in enumerate(image_angles) if a > 0 and (faces[i, :nfaces[i]]["scale"] > 50).any()]
    assert len(rotated_refined) >= 2, rotated_refined


@pytest.mark.parametrize("angle", [0.0, 0.03])
def test_pipeline_equal_angles_equal_detect_images_with_the_library_generator(gpu_face, cascades, images, angle):
    plc, flp, _, _ = cascades
    ims = images if angle == 0.0 else [im for im in images if im.Cols >= im.Rows]
    a = pipeline.detect_images_device(gpu_face, plc, flp, ims, cp_of(TEST_PARAMS), face_cap=128, rng_seed=3, angle=angle, raw=True)
    b = pipeline.detect_images_angles_device(gpu_face, plc, flp, ims, cp_of(TEST_PARAMS), [angle] * len(ims), face_cap=128, rng_seed=3, raw=True)
    assert same(a, b) and (a[0]["scale"] > 50).sum() >= 2


def test_pipeline_replays_on_the_oracle(gpu_face, oracle_face, cascades):
    """Step by step on the C oracle, each image at its own angle: two rotated wide images and one unrotated image."""
    plc, flp, _, _ = cascades
    ims = [make_image(540, 960, 960, "F", 51), make_image(300, 900, 912, "F", 52), ImageParams(synth.sample_gray(), 400, 320, 320)]
    angles = [0.03, 0.05, 0.0]
    eye = 50
    rnd = randoms_for(len(ims), 8, 43)
    faces, nfaces, points = pipeline.detect_images_angles_device(gpu_face, plc, flp, ims, cp_of(TEST_PARAMS), angles, face_cap=8, randoms=rnd,
                                                                 eye_perturbs=eye, raw=True)
    cases = [(i, image_of(im), P.oracle_clusters(oracle_face, image_of(im), TEST_PARAMS, a), a) for i, (im, a) in enumerate(zip(ims, angles))]
    _, rotated = P.replay(cascades[2:], cases, lambda i, k, slot: rnd[i, k, slot], eye, (faces, nfaces, points))
    assert rotated >= 1


def test_pipeline_capacity_errors_report_the_required_counts(gpu_face, cascades, images, image_angles, face_cap):
    plc, flp, _, _ = cascades
    _, need, _ = pipeline.detect_images_angles_device(gpu_face, plc, flp, images, cp_of(TEST_PARAMS), image_angles, face_cap=face_cap, raw=True)
    assert need.max() > 1
    hs, fl = pipeline.landmark_call_arrays(flp)
    keep = [np.ascontiguousarray(im.Pixels) for im in images]
    desc = pigo_b200.image_descs([(k.ctypes.data, im.Rows, im.Cols, im.Dim) for k, im in zip(keep, images)])
    ang = np.array(image_angles, dtype=np.float64)
    n = len(images)
    for fcap, det_cap, msg in ((1, 0, "faces, face_cap is 1"), (face_cap, 2, "raw detections, det_cap is 2")):
        prm = pigo_b200.PipelineParams(*TEST_PARAMS[:2], *TEST_PARAMS[2:], 0.0, 0.1, 50, 50, 63, det_cap)
        faces = np.zeros((n, fcap), dtype=pigo_b200.DET_DTYPE)
        nfaces = np.zeros(n, dtype=np.int32)
        points = np.zeros((n, fcap, 2 + NCALLS), dtype=pigo_b200.POINT_DTYPE)
        rc = pigo_b200.lib().pigo_detect_images_angles(gpu_face._h, plc._h, hs, fl.ctypes.data, NCALLS, desc, n, ang.ctypes.data, C.byref(prm),
                                                       None, 0, faces.ctypes.data, fcap, nfaces.ctypes.data, points.ctypes.data,
                                                       pigo_b200.MEM_HOST, None)
        assert rc == pigo_b200.PIGO_E_CAP
        assert msg in pigo_b200.lib().pigo_last_error().decode()
        if det_cap == 0:
            assert np.array_equal(nfaces, need)


def test_cpp_mirror_sample_in_a_sweep():
    """tests/cpp/test_detect_images_angles.cpp (built by build()): the sample at angles 0, 0.1 and 0.5 through
    DetectImagesAngles; its angle-0 entry passes the reference's landmark assertions."""
    run_cpp_mirror("test_detect_images_angles")
