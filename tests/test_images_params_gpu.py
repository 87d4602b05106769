"""pigo_run_cascade_images_params / pigo_detect_images_params: every image of a mixed-size call with its own CascadeParams, so
that a list of reference calls RunCascade(cp, angle) is one call.  Bar: every image's slice equals a lone pigo_run_cascade
(scan) or a lone pigo_detect_batch (pipeline) with that image's parameters and angle, byte for byte, and the C oracle on a
sample; with equal parameters both calls equal their shared-parameter forms.  Rotated angles go only on images with
Cols >= Rows, as in the angle suite (the reference's rotated column clamp indexes past tall images)."""
import ctypes as C
import math

import numpy as np
import pytest

import pigo_b200
from mixed_images import (CLI_PARAMS, KNOBS, MIXED, NCALLS, TEST_PARAMS, assert_slices, canonical, cascades, cp_of, images,  # noqa: F401 (fixtures)
                          lone_detect_batch, lone_scan, make_image, randoms_for, run_cpp_mirror, same)
from pigo_b200 import CascadeParams, ImageParams, pipeline
from option_guard import options, options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)
from synthetic import synthetic_cascade

pytestmark = pytest.mark.gpu

# MinSize, MaxSize, ShiftFactor, ScaleFactor of the reference's callers: cmd/pigo, the test suite, puploc / facial_landmark,
# facedet, talk_detector, masquerade, the wasm detector, blinkdet
REFERENCE_SETTINGS = [(20, 1000, 0.15, 1.15), (20, 1000, 0.2, 1.1), (60, 600, 0.1, 1.1), (100, 600, 0.15, 1.1), (100, 600, 0.1, 1.1),
                      (200, 600, 0.1, 1.1), (200, 480, 0.1, 1.1), (260, 640, 0.1, 1.1)]
ANGLES = [0.0, -0.1, math.nan, 1 / 64, 1 / 32, 7 / 32, 0.25, 0.5, 31 / 32, 1.0, 1.3]
UNROTATED = [0.0, -0.1, math.nan]


def random_params(im, rng):
    """MinSize 0..80, MaxSize below or above the image, ShiftFactor 0.05..0.3, ScaleFactor 1.05..1.5."""
    mn = int(rng.integers(0, 81))
    edge = max(im.Rows, im.Cols)
    mx = int(rng.integers(mn, mn + max(2, min(im.Rows, im.Cols)))) if rng.random() < 0.5 else int(rng.integers(edge, 2 * edge + 2))
    return mn, mx, float(rng.uniform(0.05, 0.3)), float(rng.uniform(1.05, 1.5))


def draw_params(ims, seed):
    """Even entries cycle through the reference's settings, odd entries draw seeded random ones."""
    rng = np.random.default_rng(seed)
    return [REFERENCE_SETTINGS[(i // 2) % 8] if i % 2 == 0 else random_params(im, rng) for i, im in enumerate(ims)]


def draw_angles(ims, seed):
    rng = np.random.default_rng(seed)
    return [float(rng.choice(ANGLES if im.Cols >= im.Rows else UNROTATED)) for im in ims]


def cps_of(ims, params):
    return [CascadeParams(im, *p) for im, p in zip(ims, params)]


def run(face, ims, params, angles=None, cap=1024):
    return face.RunCascadeImagesParams(cps_of(ims, params), angles, cap)


@pytest.fixture(scope="module")
def mixed():
    return [make_image(r, c, d, k, 31 + i) for i, (r, c, d, k) in enumerate(MIXED)]


@pytest.fixture(scope="module")
def mixed_params(mixed):
    return draw_params(mixed, 7)


@pytest.fixture(scope="module")
def mixed_angles(mixed):
    a = draw_angles(mixed, 9)
    assert sum(x > 0 for x in a) >= 5 and sum(not x > 0 for x in a) >= 5
    return a


def listing(mixed, kind, mixed_params, mixed_angles):
    """(images, params, angles) of one listing: unrotated, at mixed angles, or the same pixels several times under different
    parameters and angles."""
    if kind == "unrotated":
        return mixed, mixed_params, None
    if kind == "angles":
        return mixed, mixed_params, mixed_angles
    base = [mixed[3], mixed[4], mixed[6], mixed[9], mixed[17]]   # the sample, 480x640, 1080p, 333x517, 45x1200
    rng = np.random.default_rng(13)
    ims, prm, ang = [], [], []
    for im in base:
        for k in range(4):
            ims.append(im)
            prm.append(REFERENCE_SETTINGS[(2 * k + len(ims)) % 8] if k % 2 == 0 else random_params(im, rng))
            ang.append(float(rng.choice(ANGLES if im.Cols >= im.Rows else UNROTATED)))
    return ims, prm, ang


@pytest.mark.parametrize("kind", ["unrotated", "angles", "repeated"])
def test_each_image_equals_a_lone_call_with_its_parameters(gpu_face, oracle_face, mixed, mixed_params, mixed_angles, kind):
    ims, prm, ang = listing(mixed, kind, mixed_params, mixed_angles)
    a = ang if ang is not None else [0.0] * len(ims)
    dets, cnt = run(gpu_face, ims, prm, ang)
    expect = [lone_scan(gpu_face, im, p, x) for im, p, x in zip(ims, prm, a)]
    assert_slices(dets, cnt, expect)
    assert cnt.sum() > 0 and len({tuple(p) for p in prm}) >= 8
    if kind != "unrotated":
        assert sum(len(e) for e, x in zip(expect, a) if x > 0) > 0
    checked = 0
    for i, (im, p, x) in enumerate(zip(ims, prm, a)):
        if im.Rows * im.Cols <= 480 * 640:
            o = oracle_face.run_cascade(im.Pixels, im.Rows, im.Cols, im.Dim, *p, canonical(x))
            assert expect[i].tobytes() == o.tobytes(), f"image {i} with {p} at angle {x} differs from the oracle"
            checked += len(o)
    assert checked > 0


@pytest.mark.parametrize("params", [TEST_PARAMS, CLI_PARAMS])
def test_equal_parameters_equal_the_angles_call(gpu_face, mixed, mixed_angles, params):
    ed, ec = gpu_face.RunCascadeImagesAngles(mixed, cp_of(params), mixed_angles)
    d, c = run(gpu_face, mixed, [params] * len(mixed), mixed_angles)
    assert np.array_equal(c, ec) and c.sum() > 0
    assert d.tobytes() == ed.tobytes()
    ud, uc = gpu_face.RunCascadeImages(mixed, cp_of(params), 0.0)
    d, c = run(gpu_face, mixed, [params] * len(mixed))
    assert np.array_equal(c, uc) and d.tobytes() == ud.tobytes()


# ---- rotated node tables: one per (slot, MinSize, ScaleFactor) --------------------------------------------------------------
LONG = (20, 1000, 0.2, 1.01)   # scale factor 1.01: a long ladder, about 50 MB of node table per (slot, key) on 720x1280


def table_builds(face, ims, params, angles):
    """Runs the call under options(timing=1); (dets, counts, t_rottab_n): one table build per pass whose tables were not cached."""
    with options(timing=1):
        d, c = run(face, ims, params, angles)
        return d, c, pigo_b200.get_option("t_rottab_n")


def test_two_min_sizes_at_one_slot_build_two_tables(gpu_face):
    """Twelve slots with one key fit one pass (one build); the same images with two MinSize values need 24 tables, past the
    1 GiB bound of a pass, so they run in two passes: each MinSize has its own table.  Every entry equals a lone call."""
    im = make_image(720, 1280, 1280, "F", 9)
    angles = [k / 32 for k in range(1, 13)] * 2
    lst = [im] * len(angles)
    one_key = [LONG] * len(angles)
    two_keys = [LONG] * 12 + [(22,) + LONG[1:]] * 12
    d1, c1, b1 = table_builds(gpu_face, lst, one_key, angles)
    d2, c2, b2 = table_builds(gpu_face, lst, two_keys, angles)
    assert (b1, b2) == (1, 2), (b1, b2)
    assert_slices(d1, c1, [lone_scan(gpu_face, im, p, a) for p, a in zip(one_key, angles)])
    assert_slices(d2, c2, [lone_scan(gpu_face, im, p, a) for p, a in zip(two_keys, angles)])
    assert c2[12:].sum() > 0


def test_equal_min_size_and_scale_factor_share_one_table(gpu_face):
    """MaxSize, ShiftFactor and geometry only shorten a ladder: 24 entries over two images, every one of twelve slots listed
    under both (MaxSize, ShiftFactor) pairs, share twelve tables in one pass.  One table per full parameter set would be 24
    tables of about 50 MB, past the 1 GiB bound of a pass: two passes, two builds."""
    ims = [make_image(720, 1280, 1280, "F", 9), make_image(300, 900, 900, "F", 10)]
    angles = [k / 32 for k in range(1, 13)] * 2
    lst = [ims[0]] * 12 + [ims[1]] * 12
    params = [LONG if (k % 2) ^ (k >= 12) else (20, 600, 0.15, 1.01) for k in range(24)]
    per_slot = {}
    for a, p in zip(angles, params):
        per_slot.setdefault(a, set()).add(p)
    assert all(len(v) == 2 for v in per_slot.values())   # each slot holds both parameter sets
    d, c, builds = table_builds(gpu_face, lst, params, angles)
    assert builds == 1, builds
    assert_slices(d, c, [lone_scan(gpu_face, im, p, a) for im, p, a in zip(lst, params, angles)])
    assert c.sum() > 0


def test_keys_and_slots_past_the_bound_run_in_passes(gpu_face):
    """Three keys at eleven slots (33 tables of about 50 MB) and unrotated entries in between: several passes, every entry equal
    to a lone call."""
    ims = [make_image(720, 1280, 1280, "F", 9), make_image(300, 900, 900, "F", 10)]
    keys = [LONG, (24, 1000, 0.2, 1.01), (20, 800, 0.25, 1.012)]
    lst, prm, ang = [], [], []
    for s in range(11):
        for k, p in enumerate(keys):
            lst.append(ims[(s + k) % 2]); prm.append(p); ang.append((3 * s + 1) / 32)
        lst.append(ims[s % 2]); prm.append(keys[s % 3]); ang.append(0.0)
    d, c, builds = table_builds(gpu_face, lst, prm, ang)
    assert builds >= 2, builds
    assert_slices(d, c, [lone_scan(gpu_face, im, p, a) for im, p, a in zip(lst, prm, ang)])
    assert c.sum() > 0


def test_a_call_with_other_keys_does_not_reuse_a_cached_table(gpu_face, oracle_face):
    """One thread, so that the calls reuse one workspace: the same slots with other (MinSize, ScaleFactor) keys, and back."""
    ims = [make_image(400, 320, 320, "sample", 0), make_image(300, 900, 900, "F", 10)]
    angles = [0.05, 0.05, 0.25]
    lst = [ims[0], ims[1], ims[1]]
    found = 0
    for params in ([TEST_PARAMS] * 3, [(24, 1000, 0.2, 1.1), (20, 1000, 0.2, 1.25), (18, 700, 0.1, 1.1)], [TEST_PARAMS] * 3):
        d, c = run(gpu_face, lst, params, angles)
        assert_slices(d, c, [lone_scan(gpu_face, im, p, a) for im, p, a in zip(lst, params, angles)])
        o = oracle_face.run_cascade(ims[0].Pixels, 400, 320, 320, *params[0], angles[0])
        assert d[0, :c[0]].tobytes() == o.tobytes()
        found += len(o)
    assert found > 0


# ---- call forms ------------------------------------------------------------------------------------------------------------
def test_host_device_and_stream_forms_agree(gpu_face, mixed, mixed_params, mixed_angles):
    import torch
    ims, prm, ang = listing(mixed, "repeated", mixed_params, mixed_angles)
    hd, hc = run(gpu_face, ims, prm, ang)
    bufs = {}
    dev = []
    for im in ims:
        if id(im) not in bufs:
            bufs[id(im)] = torch.from_numpy(np.ascontiguousarray(im.Pixels).reshape(-1)[:im.Rows * im.Dim].copy()).cuda()
        dev.append((bufs[id(im)].data_ptr(), im.Rows, im.Cols, im.Dim))
    dd, dc = run(gpu_face, [ImageParams(p, r, c, d) for p, r, c, d in dev], prm, ang)
    assert np.array_equal(dc, hc) and dd.tobytes() == hd.tobytes() and hc.sum() > 0
    n, cap = len(ims), max(int(hc.max()), 1)
    out = torch.zeros((n, cap, 4), dtype=torch.int32, device="cuda")
    cnt = torch.zeros(n, dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for _ in range(2):   # back-to-back asynchronous calls reuse the same workspace
            gpu_face.run_cascade_images_params_device(dev, prm, ang, out.data_ptr(), cap, cnt.data_ptr(), st.cuda_stream)
    st.synchronize()
    o = out.cpu().numpy().view(np.uint8).reshape(n, cap, 16)
    assert np.array_equal(cnt.cpu().numpy(), hc)
    for i in range(n):
        assert o[i, :hc[i]].tobytes() == hd[i, :hc[i]].tobytes()


def test_capacity_error_reports_the_required_counts(gpu_face, mixed, mixed_params, mixed_angles):
    _, c = run(gpu_face, mixed, mixed_params, mixed_angles)
    assert c.max() > 2
    keep = [np.ascontiguousarray(im.Pixels) for im in mixed]
    desc = pigo_b200.image_descs([(k.ctypes.data, im.Rows, im.Cols, im.Dim) for k, im in zip(keep, mixed)])
    ang = np.array(mixed_angles, dtype=np.float64)
    out = np.zeros((len(mixed), 2), dtype=pigo_b200.DET_DTYPE)
    cnt = np.zeros(len(mixed), dtype=np.int32)
    rc = pigo_b200.lib().pigo_run_cascade_images_params(gpu_face._h, desc, len(mixed), pigo_b200.cascade_params_array(mixed_params), ang.ctypes.data,
                                                        out.ctypes.data, 2, cnt.ctypes.data, pigo_b200.MEM_HOST, None)
    assert rc == pigo_b200.PIGO_E_CAP
    assert np.array_equal(cnt, c)


@pytest.mark.parametrize("knobs", KNOBS)
def test_options_leave_the_outputs_unchanged(gpu_face, mixed, mixed_params, mixed_angles, knobs):
    ed, ec = run(gpu_face, mixed, mixed_params, mixed_angles)
    with options(**knobs):
        d, c = run(gpu_face, mixed, mixed_params, mixed_angles)
    assert np.array_equal(c, ec)
    for i in range(len(mixed)):
        assert d[i, :c[i]].tobytes() == ed[i, :ec[i]].tobytes(), i


def test_cascade_of_another_depth_takes_the_single_image_path(mixed, mixed_params, mixed_angles):
    face = pigo_b200.NewPigo().Unpack(synthetic_cascade(4, 9, seed=409))
    some, prm, ang = mixed[:12], mixed_params[:12], mixed_angles[:12]
    dets, cnt = run(face, some, prm, ang)
    assert_slices(dets, cnt, [lone_scan(face, im, p, a) for im, p, a in zip(some, prm, ang)])
    assert cnt.sum() > 0


# ---- pipeline ----------------------------------------------------------------------------------------------------------
EYE = 50


@pytest.fixture(scope="module")
def image_params(images):
    return [REFERENCE_SETTINGS[i % 4] if i % 3 else (20, 1000, 0.2, 1.1 + 0.02 * (i % 5)) for i in range(len(images))]


@pytest.fixture(scope="module")
def image_angles(images):
    rng = np.random.default_rng(17)
    return [float(rng.choice([0.0, 0.02, 0.03, 0.05, 0.25, math.nan, -0.2] if im.Cols >= im.Rows else [0.0, -0.2])) for im in images]


@pytest.fixture(scope="module")
def face_cap(gpu_face, cascades, images, image_params, image_angles):
    plc, flp, _, _ = cascades
    _, n, _ = pipeline.detect_images_params(gpu_face, plc, flp, cps_of(images, image_params), image_angles, face_cap=256, raw=True)
    return int(max(n.max(), 1))


def test_pipeline_each_image_equals_a_lone_detect_batch(gpu_face, cascades, images, image_params, image_angles, face_cap):
    plc, flp, _, _ = cascades
    rnd = randoms_for(len(images), face_cap, 47)
    got = pipeline.detect_images_params(gpu_face, plc, flp, cps_of(images, image_params), image_angles, face_cap=face_cap, randoms=rnd,
                                        eye_perturbs=EYE, raw=True)
    for i, (im, p, a) in enumerate(zip(images, image_params, image_angles)):
        one = lone_detect_batch(gpu_face, cascades, im, p, face_cap, rnd[i:i + 1], a, EYE)
        assert int(got[1][i]) == int(one[1][0]), i
        assert got[0][i].tobytes() == one[0][0].tobytes() and got[2][i].tobytes() == one[2][0].tobytes(), (i, p, a)
    faces, nfaces, _ = got
    refined = [i for i in range(len(images)) if (faces[i, :nfaces[i]]["scale"] > 50).any()]
    assert len(refined) >= 4 and len({image_params[i] for i in refined}) >= 2, refined
    assert any(image_angles[i] > 0 for i in refined), refined


@pytest.mark.parametrize("angle", [0.0, 0.03])
def test_pipeline_equal_parameters_equal_detect_images_angles(gpu_face, cascades, images, angle):
    plc, flp, _, _ = cascades
    ims = images if angle == 0.0 else [im for im in images if im.Cols >= im.Rows]
    angles = [angle] * len(ims)
    rnd = randoms_for(len(ims), 128, 49)
    for kw in ({"randoms": rnd}, {"rng_seed": 3}):
        a = pipeline.detect_images_angles_device(gpu_face, plc, flp, ims, cp_of(TEST_PARAMS), angles, face_cap=128, raw=True, **kw)
        b = pipeline.detect_images_params(gpu_face, plc, flp, cps_of(ims, [TEST_PARAMS] * len(ims)), angles, face_cap=128, raw=True, **kw)
        assert same(a, b) and (a[0]["scale"] > 50).sum() >= 2


def test_pipeline_capacity_errors_and_ignored_scan_fields(gpu_face, cascades, images, image_params, image_angles, face_cap):
    """The scan fields of the pipeline parameters are neither read nor checked (here they would fail pigo_run_cascade); the
    capacity errors report the required counts as pigo_detect_images does."""
    plc, flp, _, _ = cascades
    want = pipeline.detect_images_params(gpu_face, plc, flp, cps_of(images, image_params), image_angles, face_cap=face_cap, rng_seed=5, raw=True)
    need = want[1]
    assert need.max() > 1
    hs, fl = pipeline.landmark_call_arrays(flp)
    keep = [np.ascontiguousarray(im.Pixels) for im in images]
    desc = pigo_b200.image_descs([(k.ctypes.data, im.Rows, im.Cols, im.Dim) for k, im in zip(keep, images)])
    cprm = pigo_b200.cascade_params_array(image_params)
    ang = np.array(image_angles, dtype=np.float64)
    n = len(images)
    for fcap, det_cap, msg in ((face_cap, 0, None), (1, 0, "faces, face_cap is 1"), (face_cap, 2, "raw detections, det_cap is 2")):
        prm = pigo_b200.PipelineParams(-30, 10, math.nan, 1.0, 7.0, 0.1, 50, 50, 63, det_cap)
        faces = np.zeros((n, fcap), dtype=pigo_b200.DET_DTYPE)
        nfaces = np.zeros(n, dtype=np.int32)
        points = np.zeros((n, fcap, 2 + NCALLS), dtype=pigo_b200.POINT_DTYPE)
        rc = pigo_b200.lib().pigo_detect_images_params(gpu_face._h, plc._h, hs, fl.ctypes.data, NCALLS, desc, n, cprm, ang.ctypes.data, C.byref(prm),
                                                       None, 5, faces.ctypes.data, fcap, nfaces.ctypes.data, points.ctypes.data,
                                                       pigo_b200.MEM_HOST, None)
        if msg is None:
            assert rc == pigo_b200.PIGO_OK, pigo_b200.lib().pigo_last_error()
            assert same((faces, nfaces, points), want)
            continue
        assert rc == pigo_b200.PIGO_E_CAP
        assert msg in pigo_b200.lib().pigo_last_error().decode()
        if det_cap == 0:
            assert np.array_equal(nfaces, need)


def test_cpp_mirror_runs_a_list_of_calls():
    """tests/cpp/test_images_params.cpp (built by build()): entries under five of the reference's settings equal lone RunCascade
    calls, and the sample passes the reference's landmark assertions through DetectImagesParams."""
    run_cpp_mirror("test_images_params")
