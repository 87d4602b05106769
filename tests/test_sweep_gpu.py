"""pigo_run_cascade_images_sweep / pigo_detect_images_sweep: every image at every angle, one merged list per image.  Bar:
image i's clusters are pigo_cluster of the concatenation of its RunCascadeImagesAngles slices byte for byte, with the angle
indices of the largest-Q rule; on rotated samples and a 1080p frame they equal the oracle restatement (tests/sweep_oracle.py)
byte for byte and recover the tilt within one slot; the pipeline replays on the C oracle with eyes at each face's angle."""
import ctypes as C
import threading

import numpy as np
import pytest

import pigo_b200
import pipeline_oracle as P
import sweep_oracle as S
from mixed_images import (CLI_PARAMS, DOC_PARAMS, MIXED, NCALLS, TEST_PARAMS, cascades, cp_of, image_of, images, make_image,  # noqa: F401 (fixtures)
                          randoms_for, run_cpp_mirror, same)
from pigo_b200 import ImageParams, pipeline
from option_guard import options, options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)
from synthetic import synthetic_cascade

pytestmark = pytest.mark.gpu

ANGLES = S.sweep_angles()          # k/32, k = 0..31
TILTS = [0, 30, -45, 100]


@pytest.fixture(scope="module")
def mixed():
    """The mixed-size images split by shape: wide ones are swept at k/32, tall ones (whose rotated column clamp would read
    past the image, core/pigo.go:168,:171) at unrotated angles only."""
    ims = [make_image(r, c, d, k, 11 + i) for i, (r, c, d, k) in enumerate(MIXED)]
    return [im for im in ims if im.Cols >= im.Rows], [im for im in ims if im.Cols < im.Rows]


@pytest.fixture(scope="module")
def tilted():
    base = S.padded_sample()
    return [ImageParams(S.rotate(base, t), 520, 520, 520) for t in TILTS]


@pytest.fixture(scope="module")
def frame1080():
    return make_image(1080, 1920, 1920, "F", 3)


def reference_sweep(face, images, angles, params, iou):
    """pigo_cluster of each image's RunCascadeImagesAngles slices, concatenated in angle order, and the largest-Q tags."""
    ims = [im for im in images for _ in angles]
    dets, cnt = face.RunCascadeImagesAngles(ims, cp_of(params), [a for _ in images for a in angles], 4096)
    out = []
    for i in range(len(images)):
        parts = [dets[i * len(angles) + a, :cnt[i * len(angles) + a]] for a in range(len(angles))]
        out.append(S.merge(parts, iou, cluster=face.cluster_array))
    return out


def assert_sweep(got, expect):
    dets, idx, cnt = got
    assert len(cnt) == len(expect)
    for i, (cl, ix) in enumerate(expect):
        assert int(cnt[i]) == len(cl), (i, int(cnt[i]), len(cl))
        assert dets[i, :len(cl)].tobytes() == cl.tobytes(), i
        assert np.array_equal(idx[i, :len(cl)], ix), i


@pytest.mark.parametrize("params,iou", [(TEST_PARAMS, 0.1), (DOC_PARAMS, 0.2), (CLI_PARAMS, 0.1)])
def test_each_image_equals_the_cluster_of_its_angle_slices(gpu_face, mixed, params, iou):
    wide, tall = mixed
    for ims, angles in ((wide, ANGLES), (tall, [0.0, -0.1, float("nan")])):
        got = gpu_face.RunCascadeImagesSweep(ims, cp_of(params), angles, iou)
        expect = reference_sweep(gpu_face, ims, angles, params, iou)
        assert_sweep(got, expect)
    assert (got[2] > 0).sum() > 0


def test_rotated_samples_and_a_1080p_frame_equal_the_oracle(gpu_face, oracle_face, tilted, frame1080):
    ims = tilted + [frame1080]
    got = gpu_face.RunCascadeImagesSweep(ims, cp_of(TEST_PARAMS), ANGLES, 0.1)
    expect = [S.sweep_oracle(oracle_face, (im.Pixels, im.Rows, im.Cols, im.Dim), ANGLES, TEST_PARAMS, 0.1) for im in ims]
    assert_sweep(got, expect)
    for t, (cl, ix) in zip(TILTS, expect):
        assert S.slot_distance(S.strongest_slot(cl, ix, ANGLES), S.expected_slot(t)) <= 1, t


# ---- pipeline ----------------------------------------------------------------------------------------------------------
def sweep(gpu_face, cascades, ims, angles, **kw):
    plc, flp, _, _ = cascades
    return pipeline.detect_images_sweep_device(gpu_face, plc, flp, ims, cp_of(TEST_PARAMS), angles, raw=True, **kw)


def test_pipeline_replays_on_the_oracle(gpu_face, oracle_face, cascades, tilted, frame1080):
    """Faces and angle indices equal the oracle sweep; eyes replay on the C oracle at angles[face_angle], landmarks at 0."""
    ims = tilted + [frame1080]
    fcap, eye = 32, 50
    rnd = randoms_for(len(ims), fcap, 47)
    faces, nfaces, points, fangle = sweep(gpu_face, cascades, ims, ANGLES, face_cap=fcap, randoms=rnd, eye_perturbs=eye)
    cases = []
    for i, im in enumerate(ims):
        cl, ix = S.sweep_oracle(oracle_face, image_of(im), ANGLES, TEST_PARAMS, 0.1)
        assert np.array_equal(fangle[i, :len(cl)], ix), i
        cases.append((i, image_of(im), cl, [ANGLES[j] for j in ix]))
    _, rotated = P.replay(cascades[2:], cases, lambda i, k, slot: rnd[i, k, slot], eye, (faces, nfaces, points))
    assert rotated >= 2, rotated


@pytest.mark.parametrize("angle", [0.0, 0.03])
def test_one_angle_equals_detect_images_angles(gpu_face, cascades, images, angle):
    plc, flp, _, _ = cascades
    ims = images if angle == 0.0 else [im for im in images if im.Cols >= im.Rows]
    fcap = 128
    rnd = randoms_for(len(ims), fcap, 53)
    for kw in ({"randoms": rnd}, {"rng_seed": 3}):
        a = pipeline.detect_images_angles_device(gpu_face, plc, flp, ims, cp_of(TEST_PARAMS), [angle] * len(ims), face_cap=fcap, raw=True, **kw)
        b = sweep(gpu_face, cascades, ims, [angle], face_cap=fcap, **kw)
        assert same(a, b[:3])
        for i in range(len(ims)):
            assert (b[3][i, :b[1][i]] == 0).all(), i
        assert (a[0]["scale"] > 50).sum() >= 2


def test_decoded_images_through_the_device_arena(gpu_face, cascades, tilted):
    """pigo_gray_images then the sweep on the arena (PIGO_FRAMES_DEVICE): the same as the sweep of the host gray images."""
    srcs = [pigo_b200.DecodedImage.gray(np.ascontiguousarray(im.Pixels), im.Cols, im.Rows) for im in tilted]
    arena, dimgs = pigo_b200.gray_images(srcs)
    host = gpu_face.RunCascadeImagesSweep(tilted, cp_of(TEST_PARAMS), ANGLES, 0.1)
    dev = gpu_face.RunCascadeImagesSweep([ImageParams(*t) for t in dimgs], cp_of(TEST_PARAMS), ANGLES, 0.1)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(host, dev))
    a = sweep(gpu_face, cascades, tilted, ANGLES, rng_seed=5)
    b = sweep(gpu_face, cascades, [ImageParams(*t) for t in dimgs], ANGLES, rng_seed=5)
    assert same(a, b)
    del arena


def test_host_device_and_stream_forms_agree(gpu_face, cascades, tilted):
    import torch
    plc, flp, _, _ = cascades
    hd, hi, hc = gpu_face.RunCascadeImagesSweep(tilted, cp_of(TEST_PARAMS), ANGLES, 0.1)
    bufs = [torch.from_numpy(np.ascontiguousarray(im.Pixels).reshape(-1).copy()).cuda() for im in tilted]
    dev = [(b.data_ptr(), im.Rows, im.Cols, im.Dim) for b, im in zip(bufs, tilted)]
    n, cap = len(tilted), max(int(hc.max()), 1)
    out = torch.zeros((n, cap, 4), dtype=torch.int32, device="cuda")
    idx = torch.full((n, cap), -1, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(n, dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for _ in range(2):   # back-to-back asynchronous calls reuse the same workspace
            gpu_face.run_cascade_images_sweep_device(dev, ANGLES, *TEST_PARAMS, 0.1, 0, out.data_ptr(), idx.data_ptr(), cap, cnt.data_ptr(),
                                                     st.cuda_stream)
    st.synchronize()
    o = out.cpu().numpy().view(np.uint8).reshape(n, cap, 16)
    ix = idx.cpu().numpy()
    assert np.array_equal(cnt.cpu().numpy(), hc)
    for i in range(n):
        assert o[i, :hc[i]].tobytes() == hd[i, :hc[i]].tobytes() and np.array_equal(ix[i, :hc[i]], hi[i, :hc[i]]), i
    # pipeline: host images, device images with host outputs, device images with device outputs on a caller stream
    fcap = 8
    ha = sweep(gpu_face, cascades, tilted, ANGLES, face_cap=fcap, rng_seed=9)
    da = sweep(gpu_face, cascades, [ImageParams(*t) for t in dev], ANGLES, face_cap=fcap, rng_seed=9)
    assert same(ha, da)
    prm = pigo_b200.PipelineParams(*TEST_PARAMS, 0.0, 0.1, 50, 50, 63, 0)
    f = torch.zeros((n, fcap, 4), dtype=torch.int32, device="cuda")
    fa = torch.zeros((n, fcap), dtype=torch.int32, device="cuda")
    nf = torch.zeros(n, dtype=torch.int32, device="cuda")
    pts = torch.zeros((n, fcap, 2 + NCALLS, 4), dtype=torch.int32, device="cuda")
    with torch.cuda.stream(st):
        pipeline.detect_images_sweep_device_ptrs(gpu_face, plc, flp, dev, ANGLES, prm, f.data_ptr(), fa.data_ptr(), fcap, nf.data_ptr(),
                                                 pts.data_ptr(), rng_seed=9, stream=st.cuda_stream)
    st.synchronize()
    assert np.array_equal(nf.cpu().numpy(), ha[1])
    for i in range(n):
        k = int(ha[1][i])
        assert f.cpu().numpy().view(np.uint8).reshape(n, fcap, 16)[i, :k].tobytes() == ha[0][i, :k].tobytes(), i
        assert np.array_equal(fa.cpu().numpy()[i, :k], ha[3][i, :k]), i
    assert pts.cpu().numpy().view(np.uint8).reshape(n, fcap, 2 + NCALLS, 16).tobytes() == ha[2].tobytes()


def test_capacity_errors_report_the_required_counts(gpu_face, cascades, tilted):
    _, _, c = gpu_face.RunCascadeImagesSweep(tilted, cp_of(TEST_PARAMS), ANGLES, 0.1)
    assert c.max() > 1
    keep = [np.ascontiguousarray(im.Pixels) for im in tilted]
    desc = pigo_b200.image_descs([(k.ctypes.data, im.Rows, im.Cols, im.Dim) for k, im in zip(keep, tilted)])
    ang = np.array(ANGLES, dtype=np.float64)
    n, L = len(tilted), pigo_b200.lib()
    for cap, det_cap, msg in ((1, 0, "clusters, cap_per_image is 1"), (16, 2, "raw detections, det_cap is 2")):
        out = np.zeros((n, cap), dtype=pigo_b200.DET_DTYPE)
        idx = np.zeros((n, cap), dtype=np.int32)
        cnt = np.zeros(n, dtype=np.int32)
        rc = L.pigo_run_cascade_images_sweep(gpu_face._h, desc, n, ang.ctypes.data, len(ang), *TEST_PARAMS, 0.1, det_cap, out.ctypes.data,
                                             idx.ctypes.data, cap, cnt.ctypes.data, pigo_b200.MEM_HOST, None)
        assert rc == pigo_b200.PIGO_E_CAP
        assert msg in L.pigo_last_error().decode()
        if det_cap == 0:
            assert np.array_equal(cnt, c)
    plc, flp, _, _ = cascades
    need = sweep(gpu_face, cascades, tilted, ANGLES, face_cap=64)[1]
    assert need.max() > 1
    hs, fl = pipeline.landmark_call_arrays(flp)
    for fcap, det_cap, msg in ((1, 0, "faces, face_cap is 1"), (64, 2, "raw detections, det_cap is 2")):
        prm = pigo_b200.PipelineParams(*TEST_PARAMS, 0.0, 0.1, 50, 50, 63, det_cap)
        faces = np.zeros((n, fcap), dtype=pigo_b200.DET_DTYPE)
        fa = np.zeros((n, fcap), dtype=np.int32)
        nfaces = np.zeros(n, dtype=np.int32)
        points = np.zeros((n, fcap, 2 + NCALLS), dtype=pigo_b200.POINT_DTYPE)
        rc = L.pigo_detect_images_sweep(gpu_face._h, plc._h, hs, fl.ctypes.data, NCALLS, desc, n, ang.ctypes.data, len(ang), C.byref(prm), None, 0,
                                        faces.ctypes.data, fa.ctypes.data, fcap, nfaces.ctypes.data, points.ctypes.data, pigo_b200.MEM_HOST, None)
        assert rc == pigo_b200.PIGO_E_CAP
        assert msg in L.pigo_last_error().decode()
        if det_cap == 0:
            assert np.array_equal(nfaces, need)


@pytest.mark.parametrize("knobs", [{"scan_mode": 1}, {"rot_mode": 1}])
def test_fallback_scans_give_the_same_outputs(gpu_face, cascades, tilted, knobs):
    a = gpu_face.RunCascadeImagesSweep(tilted, cp_of(TEST_PARAMS), ANGLES, 0.1)
    pa = sweep(gpu_face, cascades, tilted, ANGLES, rng_seed=2)
    with options(**knobs):
        b = gpu_face.RunCascadeImagesSweep(tilted, cp_of(TEST_PARAMS), ANGLES, 0.1)
        pb = sweep(gpu_face, cascades, tilted, ANGLES, rng_seed=2)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    assert same(pa, pb)


def test_cascade_of_another_depth(tilted):
    face = pigo_b200.NewPigo().Unpack(synthetic_cascade(4, 9, seed=409))
    angles, params = ANGLES[::8], (60, 1000, 0.3, 1.2)   # a cascade that fires often: few windows keep the merged lists short
    got = face.RunCascadeImagesSweep(tilted[:2], cp_of(params), angles, 0.1)
    assert_sweep(got, reference_sweep(face, tilted[:2], angles, params, 0.1))
    assert got[2].sum() > 0


def test_concurrent_calls_on_one_classifier(gpu_face, tilted, frame1080):
    ims = tilted + [frame1080]
    subsets = [ims[i::3] for i in range(3)]
    expect = [gpu_face.RunCascadeImagesSweep(s, cp_of(TEST_PARAMS), ANGLES, 0.1) for s in subsets]
    errors = []

    def work(k):
        try:
            for _ in range(3):
                got = gpu_face.RunCascadeImagesSweep(subsets[k], cp_of(TEST_PARAMS), ANGLES, 0.1)
                if not all(x.tobytes() == y.tobytes() for x, y in zip(got, expect[k])):
                    errors.append(k)
        except Exception as e:   # noqa: BLE001
            errors.append(repr(e))

    ts = [threading.Thread(target=work, args=(k,)) for k in range(3)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert errors == []


def test_cpp_mirror_sweep():
    """tests/cpp/test_sweep.cpp (built by build()): the sample swept through DetectImagesSweep passes the reference's
    landmark assertions, and RunCascadeImagesSweep agrees with it and, at one angle, with ClusterDetections of RunCascade."""
    run_cpp_mirror("test_sweep")
