"""The sharded mixed-size and decoded calls on the H100.  Bar: for every shard count (option shard_split: 0 = one shard per
device, k > 0 = k shards that share the devices, here one card), every entry's slices equal the single-device call's byte
for byte: pigo_run_cascade_images_angles for the scan, pigo_detect_images_angles for the pipeline (with injected randoms
and with the library generator, whose keys must not depend on the split), pigo_gray_images + the matching call for the
decoded forms.  A too-small capacity reports every shard's counts; a sampled image is checked against the C oracle."""
import ctypes as C

import numpy as np
import pytest

import pigo_b200
from decoded_sources import face_sources, host_images, narrow_sources, wide_sources, ycbcr_src  # noqa: F401 (fixtures)
from mixed_images import MIXED, NCALLS, TEST_PARAMS, canonical, cascades, cp_of, make_image, run_cpp_mirror  # noqa: F401 (fixture)
from pigo_b200 import pipeline, synth
from option_guard import options, options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)

pytestmark = pytest.mark.gpu

SWEEP = [0.0] + [k / 32 for k in range(1, 33)]


def splits(n):
    return [0, 2, 3, 7, n + 2]


@pytest.fixture(autouse=True)
def shard_split():
    """Sets option shard_split within a test; every option is restored afterwards."""
    with options():
        yield lambda k: pigo_b200.set_option("shard_split", k)


@pytest.fixture(scope="module")
def mixed():
    """The MIXED geometries (odd sizes, dim > cols, no-window images, 1080p, one 4K frame), seeded."""
    return [make_image(r, c, d, k, 31 + i) for i, (r, c, d, k) in enumerate(MIXED)]


@pytest.fixture(scope="module")
def mixed_angles(mixed):
    rng = np.random.default_rng(17)
    # rotated angles only where Cols >= Rows (see test_angles_gpu)
    return [float(rng.choice([0.0, 0.1, 0.25, 0.5, 1.0, -0.2])) if im.Cols >= im.Rows else 0.0 for im in mixed]


def check_oracle(oracle_face, images, angles, dets, cnt, seed):
    """One image of the call (<= 1080p, chosen by seed) against the C oracle."""
    small = [i for i, im in enumerate(images) if im.Rows * im.Cols <= 1080 * 1920]
    i = small[np.random.default_rng(seed).integers(len(small))]
    im = images[i]
    o = oracle_face.run_cascade(im.Pixels, im.Rows, im.Cols, im.Dim, *TEST_PARAMS, canonical(angles[i]))
    assert int(cnt[i]) == len(o) and dets[i, :len(o)].tobytes() == o.tobytes(), f"image {i} differs from the oracle"


# ---- scan ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["zero", "mixed"])
def test_scan_equals_the_single_device_call_for_every_split(gpu_face, oracle_face, mixed, mixed_angles, which, shard_split):
    angles = [0.0] * len(mixed) if which == "zero" else mixed_angles
    want, wcnt = gpu_face.RunCascadeImagesAngles(mixed, cp_of(), angles, 512)
    assert wcnt.sum() > 0
    for k in splits(len(mixed)):
        shard_split(k)
        got, cnt = gpu_face.run_cascade_images_sharded(mixed, cp_of(), None if which == "zero" else angles, 512)
        assert np.array_equal(cnt, wcnt), k
        assert got.tobytes() == want.tobytes(), k
        check_oracle(oracle_face, mixed, angles, got, cnt, seed=k)


def test_an_angle_sweep_of_one_photo_equals_the_single_device_call(gpu_face, shard_split):
    photo = make_image(1080, 1920, 1920, "F", 3)
    ims = [photo] * len(SWEEP)
    want, wcnt = gpu_face.RunCascadeImagesAngles(ims, cp_of(), SWEEP, 512)
    assert (wcnt[1:] > 0).sum() > 0
    for k in splits(len(ims)):
        shard_split(k)
        got, cnt = gpu_face.run_cascade_images_sharded(ims, cp_of(), SWEEP, 512)
        assert np.array_equal(cnt, wcnt) and got.tobytes() == want.tobytes(), k


def test_scan_capacity_reports_every_shard_and_the_retry_matches(gpu_face, mixed, mixed_angles, shard_split):
    want, wcnt = gpu_face.RunCascadeImagesAngles(mixed, cp_of(), mixed_angles, 512)
    desc = pigo_b200.image_descs([(np.ascontiguousarray(im.Pixels).ctypes.data, im.Rows, im.Cols, im.Dim) for im in mixed])
    ang = np.ascontiguousarray(mixed_angles, dtype=np.float64)
    n = len(mixed)
    for k in (3, 7):
        shard_split(k)
        out = np.zeros((n, 1), dtype=pigo_b200.DET_DTYPE)
        cnt = np.zeros(n, dtype=np.int32)
        rc = pigo_b200.lib().pigo_run_cascade_images_sharded(gpu_face._h, desc, n, ang.ctypes.data, *TEST_PARAMS, out.ctypes.data, 1, cnt.ctypes.data)
        assert rc == pigo_b200.PIGO_E_CAP
        assert np.array_equal(cnt, wcnt), k   # every shard's required counts
        cap = int(cnt.max())
        out = np.zeros((n, 512), dtype=pigo_b200.DET_DTYPE)
        rc = pigo_b200.lib().pigo_run_cascade_images_sharded(gpu_face._h, desc, n, ang.ctypes.data, *TEST_PARAMS, out.ctypes.data, 512, cnt.ctypes.data)
        assert rc == 0 and cap <= 512 and np.array_equal(cnt, wcnt) and out.tobytes() == want.tobytes()


# ---- pipeline -----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pipe_images():
    """Face frames of several sizes (odd sizes, dim > cols), the sample among them twice, a 4K frame, no-window images."""
    geoms = [(10, 10, 10, "U"), (400, 320, 320, "sample"), (540, 960, 960, "F"), (333, 517, 531, "F"), (2160, 3840, 3840, "F"),
             (700, 260, 272, "F"), (21, 300, 300, "U"), (300, 900, 912, "F"), (400, 320, 320, "sample"), (1080, 1920, 1920, "F"),
             (97, 131, 160, "U"), (600, 800, 800, "F")]
    return [make_image(r, c, d, k, 51 + i) for i, (r, c, d, k) in enumerate(geoms)]


@pytest.fixture(scope="module")
def pipe_angles(pipe_images):
    # rotated angles only where Cols >= Rows (see test_angles_gpu)
    return [0.0, 0.0, 0.1, 0.0, 0.5, 0.0, 0.0, 0.25, 0.0, 0.0, 0.0, 0.05]


@pytest.fixture(scope="module")
def face_cap(gpu_face, cascades, pipe_images, pipe_angles):
    plc, flp, _, _ = cascades
    _, n, _ = pipeline.detect_images_angles_device(gpu_face, plc, flp, pipe_images, cp_of(), pipe_angles, face_cap=256, raw=True)
    return int(max(n.max(), 1))


@pytest.mark.parametrize("injected", [True, False])
def test_pipeline_equals_the_single_device_call_for_every_split(gpu_face, cascades, pipe_images, pipe_angles, face_cap, injected, shard_split):
    plc, flp, _, _ = cascades
    n = len(pipe_images)
    rnd = np.random.default_rng(5).random((n, face_cap, 2 + NCALLS, 63, 3), dtype=np.float32) if injected else None
    want = pipeline.detect_images_angles_device(gpu_face, plc, flp, pipe_images, cp_of(), pipe_angles, face_cap=face_cap, randoms=rnd,
                                                rng_seed=77, raw=True)
    assert want[1].sum() > 0 and (want[2]["scale"] != 0).any()
    for k in splits(n):
        shard_split(k)
        got = pipeline.detect_images_sharded(gpu_face, plc, flp, pipe_images, cp_of(), pipe_angles, face_cap=face_cap, randoms=rnd, rng_seed=77,
                                             raw=True)
        for a, b in zip(got, want):
            assert a.tobytes() == b.tobytes(), (k, injected)


def test_pipeline_angle_none_uses_the_params_angle(gpu_face, cascades, pipe_images, face_cap, shard_split):
    plc, flp, _, _ = cascades
    ims = [im for im in pipe_images if im.Cols >= im.Rows]
    want = pipeline.detect_images_device(gpu_face, plc, flp, ims, cp_of(), face_cap=face_cap, angle=0.1, rng_seed=3, raw=True)
    shard_split(3)
    got = pipeline.detect_images_sharded(gpu_face, plc, flp, ims, cp_of(), None, face_cap=face_cap, angle=0.1, rng_seed=3, raw=True)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want))


def test_pipeline_capacity_reports_every_shard_and_the_retry_matches(gpu_face, cascades, pipe_images, pipe_angles, face_cap, shard_split):
    plc, flp, _, _ = cascades
    want = pipeline.detect_images_angles_device(gpu_face, plc, flp, pipe_images, cp_of(), pipe_angles, face_cap=face_cap, rng_seed=9, raw=True)
    assert face_cap > 1
    hs, fl = pipeline.landmark_call_arrays(flp)
    n = len(pipe_images)
    desc = pigo_b200.image_descs([(np.ascontiguousarray(im.Pixels).ctypes.data, im.Rows, im.Cols, im.Dim) for im in pipe_images])
    ang = np.ascontiguousarray(pipe_angles, dtype=np.float64)
    prm = pigo_b200.PipelineParams(*TEST_PARAMS, 0.0, 0.1, 50, 50, 63, 0)
    for k in (2, 7):
        shard_split(k)
        faces = np.zeros((n, 1), dtype=pigo_b200.DET_DTYPE)
        nf = np.zeros(n, dtype=np.int32)
        pts = np.zeros((n, 1, 2 + NCALLS), dtype=pigo_b200.POINT_DTYPE)
        rc = pigo_b200.lib().pigo_detect_images_sharded(gpu_face._h, plc._h, hs, fl.ctypes.data, NCALLS, desc, n, ang.ctypes.data, C.byref(prm),
                                                       None, 9, faces.ctypes.data, 1, nf.ctypes.data, pts.ctypes.data)
        assert rc == pigo_b200.PIGO_E_CAP and np.array_equal(nf, want[1]), k
        got = pipeline.detect_images_sharded(gpu_face, plc, flp, pipe_images, cp_of(), pipe_angles, face_cap=int(nf.max()), rng_seed=9, raw=True)
        ref = pipeline.detect_images_angles_device(gpu_face, plc, flp, pipe_images, cp_of(), pipe_angles, face_cap=int(nf.max()), rng_seed=9,
                                                   raw=True)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(got, ref))


def test_the_reference_landmark_assertions_hold_on_the_sample_among_other_images(gpu_face, cascades, pipe_images, pipe_angles, face_cap,
                                                                                  shard_split):
    """core/flploc_test.go:75-154 on the sample (entries 1 and 8 of the call, both at angle 0): at least one face, and the
    refined face's 15 landmark points inside the image."""
    plc, flp, _, _ = cascades
    for k in (0, 3):
        shard_split(k)
        res = pipeline.detect_images_sharded(gpu_face, plc, flp, pipe_images, cp_of(), pipe_angles, face_cap=face_cap, rng_seed=1)
        for i in (1, 8):
            assert len(res[i]) >= 1
            refined = [f for f in res[i] if f.det[2] > 50]
            assert refined and all(len(f.landmarks) == 15 for f in refined)
            assert all(p.Row > 0 and p.Col > 0 for f in refined for p in f.landmarks)


# ---- decoded sources ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def decoded_mix(wide_sources, face_sources):
    """All nine formats, face content in five of them, with repeats, as host sources."""
    nine = narrow_sources() + [wide_sources[k] for k in (4, 12, 20, 28, 36)]
    faces = face_sources + [ycbcr_src(2, 320, 400, 1, 1, 24, luma=synth.sample_gray())]
    picks = [faces[5], nine[0], faces[0], nine[8], faces[1], nine[4], faces[2], faces[5], nine[1], faces[3], nine[5], nine[2], faces[4],
             nine[6], nine[7], nine[3], faces[0]]
    assert sorted({s.fmt for s in picks}) == [0, 1, 2, 3, 5, 6, 7, 8, 9]
    return picks


def test_decoded_scan_equals_gray_images_and_the_single_device_call(gpu_face, decoded_mix, shard_split):
    srcs = [s.decoded() for s in decoded_mix]
    angles = [0.0, 0.0, 0.1, 0.0, 0.0, 0.0, 0.3, 0.0, 0.0, 0.05, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.2]
    arena, images = pigo_b200.gray_images(srcs)
    want, wcnt = gpu_face.RunCascadeImagesAngles(images, cp_of(), angles, 512)
    del arena
    assert wcnt.sum() > 0
    for k in splits(len(srcs)):
        shard_split(k)
        got, cnt = gpu_face.run_cascade_decoded_sharded(srcs, cp_of(), angles, 512)
        assert np.array_equal(cnt, wcnt) and got.tobytes() == want.tobytes(), k
    # and the host gray images the oracle makes of the sources
    hw, hc = gpu_face.RunCascadeImagesAngles(host_images(decoded_mix), cp_of(), angles, 512)
    assert np.array_equal(hc, wcnt) and hw.tobytes() == want.tobytes()


@pytest.mark.parametrize("injected", [True, False])
def test_decoded_pipeline_equals_detect_decoded_for_every_split(gpu_face, cascades, decoded_mix, injected, shard_split):
    plc, flp, _, _ = cascades
    srcs = [s.decoded() for s in decoded_mix]
    n = len(srcs)
    rnd = np.random.default_rng(8).random((n, 8, 2 + NCALLS, 63, 3), dtype=np.float32) if injected else None
    want = pipeline.detect_decoded(gpu_face, plc, flp, srcs, cp_of(), face_cap=8, randoms=rnd, rng_seed=21, raw=True)
    assert want[1].sum() > 0
    for k in splits(n):
        shard_split(k)
        got = pipeline.detect_decoded(gpu_face, plc, flp, srcs, cp_of(), face_cap=8, randoms=rnd, rng_seed=21, raw=True, sharded=True)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want)), (k, injected)


def test_decoded_capacity_reports_every_shard(gpu_face, decoded_mix, shard_split):
    srcs = [s.decoded() for s in decoded_mix]
    _, wcnt = gpu_face.run_cascade_decoded_sharded(srcs, cp_of(), None, 512)
    n = len(srcs)
    shard_split(5)
    out = np.zeros((n, 1), dtype=pigo_b200.DET_DTYPE)
    cnt = np.zeros(n, dtype=np.int32)
    rc = pigo_b200.lib().pigo_run_cascade_decoded_sharded(gpu_face._h, pigo_b200.decoded_descs(srcs), n, None, *TEST_PARAMS, out.ctypes.data, 1,
                                                         cnt.ctypes.data)
    assert rc == pigo_b200.PIGO_E_CAP and np.array_equal(cnt, wcnt)


# ---- the C++ mirror -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("split", [0, 3, 9])
def test_cpp_mirror(split):
    run_cpp_mirror("test_images_sharded", split, timeout=600)
