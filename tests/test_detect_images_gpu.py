"""pigo_detect_images: face -> cluster -> pupils -> 15 landmarks over images of different sizes in one call, and
pigo_puploc_run_images.  Bar: every image's slices equal a lone pigo_detect_batch(nframes=1) on that image byte for byte
with the same randoms, and up to 1080p the C oracle replays the sequence step by step."""
import ctypes as C
import threading

import numpy as np
import pytest

import oracle_lib as O
import pigo_b200
import pipeline_oracle as P
from mixed_images import (CLI_PARAMS, EYE, GEOMS, NCALLS, TEST_PARAMS, assert_same_outputs, cascades, cp_of, image_of, images,  # noqa: F401 (fixtures)
                          lone_detect_batch, make_image, randoms_for, run_cpp_mirror)
from pigo_b200 import CascadeParams, ImageParams, Puploc, pipeline, synth
from option_guard import options, options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def face_cap(gpu_face, cascades, images):
    """Room for every image's clusters (so that the randoms array covers them all)."""
    plc, flp, _, _ = cascades
    _, n, _ = pipeline.detect_images_device(gpu_face, plc, flp, images, cp_of(CLI_PARAMS), face_cap=256, raw=True)
    _, n2, _ = pipeline.detect_images_device(gpu_face, plc, flp, images, cp_of(TEST_PARAMS), face_cap=256, raw=True)
    return int(max(n.max(), n2.max(), 1))


@pytest.mark.parametrize("stage", [1, 2])
@pytest.mark.parametrize("angle", [0.0, 0.03])
@pytest.mark.parametrize("params", [TEST_PARAMS, CLI_PARAMS])
def test_each_image_equals_a_lone_detect_batch(gpu_face, oracle_face, cascades, images, face_cap, params, angle, stage):
    plc, flp, _, _ = cascades
    eye = EYE[params]
    rnd = randoms_for(len(images), face_cap, 17)
    with options(puploc_stage=stage):
        got = pipeline.detect_images_device(gpu_face, plc, flp, images, cp_of(params), face_cap=face_cap, randoms=rnd, angle=angle,
                                            eye_perturbs=eye, raw=True)
        for i, im in enumerate(images):
            assert_same_outputs(got, lone_detect_batch(gpu_face, cascades, im, params, face_cap, rnd[i:i + 1], angle, eye), [i], [0])
    faces, nfaces, _ = got
    refined = {GEOMS[i][:3] for i in range(len(images)) if (faces[i, :nfaces[i]]["scale"] > 50).any()}
    assert len(refined) >= 3, refined
    if stage == 2 and params == TEST_PARAMS:
        # step by step on the C oracle, each image with its own rows, cols and dim (images up to 1080p)
        cases = [(i, image_of(im), P.oracle_clusters(oracle_face, image_of(im), params, angle), angle)
                 for i, im in enumerate(images) if im.Rows * im.Cols <= 1080 * 1920]
        P.replay(cascades[2:], cases, lambda i, k, slot: rnd[i, k, slot], eye, got)


def test_one_geometry_with_the_library_generator_equals_detect_batch(gpu_face, cascades):
    plc, flp, _, _ = cascades
    frames = np.stack([synth.frame_faces(None, 540, 960, shift=(11 * i, 7 * i), noise_seed=90 + i) for i in range(4)])
    cpb = CascadeParams(ImageParams(None, 540, 960, 960), *TEST_PARAMS)
    ims = [ImageParams(f, 540, 960, 960) for f in frames]
    a = pipeline.detect_batch_device(gpu_face, plc, flp, frames, cpb, face_cap=16, rng_seed=5, raw=True)
    b = pipeline.detect_images_device(gpu_face, plc, flp, ims, cp_of(TEST_PARAMS), face_cap=16, rng_seed=5, raw=True)
    c = pipeline.detect_images_device(gpu_face, plc, flp, ims, cp_of(TEST_PARAMS), face_cap=16, rng_seed=5, raw=True)
    d = pipeline.detect_images_device(gpu_face, plc, flp, ims, cp_of(TEST_PARAMS), face_cap=16, rng_seed=6, raw=True)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    assert all(x.tobytes() == y.tobytes() for x, y in zip(b, c))
    assert b[0].tobytes() == d[0].tobytes() and b[1].tobytes() == d[1].tobytes() and b[2].tobytes() != d[2].tobytes()
    assert (b[0]["scale"] > 50).sum() >= 4


def test_host_device_and_stream_forms_agree(gpu_face, cascades, images, face_cap):
    import torch
    plc, flp, _, _ = cascades
    rnd = randoms_for(len(images), face_cap, 23)
    host = pipeline.detect_images_device(gpu_face, plc, flp, images, cp_of(TEST_PARAMS), face_cap=face_cap, randoms=rnd, raw=True)
    bufs = [torch.from_numpy(np.ascontiguousarray(im.Pixels).reshape(-1)[:im.Rows * im.Dim].copy()).cuda() for im in images]
    dev_ims = [ImageParams(b.data_ptr(), im.Rows, im.Cols, im.Dim) for b, im in zip(bufs, images)]
    dev = pipeline.detect_images_device(gpu_face, plc, flp, dev_ims, cp_of(TEST_PARAMS), face_cap=face_cap, randoms=rnd, raw=True)
    assert_same_outputs(host, dev)
    # device outputs (and device randoms) on a torch stream, two asynchronous calls back to back
    n = len(images)
    hs, fl = pipeline.landmark_call_arrays(flp)
    prm = pigo_b200.PipelineParams(*TEST_PARAMS[:2], *TEST_PARAMS[2:], 0.0, 0.1, 50, 50, 63, 0)
    desc = pigo_b200.image_descs([(b.data_ptr(), im.Rows, im.Cols, im.Dim) for b, im in zip(bufs, images)])
    d_rnd = torch.from_numpy(rnd).cuda()
    faces = torch.zeros((n, face_cap, 4), dtype=torch.int32, device="cuda")
    nfaces = torch.zeros(n, dtype=torch.int32, device="cuda")
    points = torch.zeros((n, face_cap, 2 + NCALLS, 4), dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for _ in range(2):
            rc = pigo_b200.lib().pigo_detect_images(gpu_face._h, plc._h, hs, fl.ctypes.data, NCALLS, desc, n, C.byref(prm), d_rnd.data_ptr(), 0,
                                                    faces.data_ptr(), face_cap, nfaces.data_ptr(), points.data_ptr(),
                                                    pigo_b200.FRAMES_DEVICE | pigo_b200.OUT_DEVICE, C.c_void_p(st.cuda_stream))
            assert rc == 0, pigo_b200.lib().pigo_last_error()
    st.synchronize()
    assert np.array_equal(nfaces.cpu().numpy(), host[1])
    assert faces.cpu().numpy().tobytes() == host[0].tobytes()
    assert points.cpu().numpy().tobytes() == host[2].tobytes()


def test_permuting_images_and_randoms_permutes_the_outputs(gpu_face, cascades, images, face_cap):
    plc, flp, _, _ = cascades
    rnd = randoms_for(len(images), face_cap, 29)
    base = pipeline.detect_images_device(gpu_face, plc, flp, images, cp_of(TEST_PARAMS), face_cap=face_cap, randoms=rnd, raw=True)
    perm = np.random.default_rng(4).permutation(len(images))
    got = pipeline.detect_images_device(gpu_face, plc, flp, [images[j] for j in perm], cp_of(TEST_PARAMS), face_cap=face_cap,
                                        randoms=rnd[perm], raw=True)
    assert_same_outputs(got, base, range(len(images)), perm)


def test_capacity_errors_report_the_required_counts(gpu_face, cascades, images, face_cap):
    plc, flp, _, _ = cascades
    _, need, _ = pipeline.detect_images_device(gpu_face, plc, flp, images, cp_of(TEST_PARAMS), face_cap=face_cap, raw=True)
    assert need.max() > 1
    hs, fl = pipeline.landmark_call_arrays(flp)
    keep = [np.ascontiguousarray(im.Pixels) for im in images]
    desc = pigo_b200.image_descs([(k.ctypes.data, im.Rows, im.Cols, im.Dim) for k, im in zip(keep, images)])
    n = len(images)
    for fcap, det_cap, msg in ((1, 0, "faces, face_cap is 1"), (face_cap, 2, "raw detections, det_cap is 2")):
        prm = pigo_b200.PipelineParams(*TEST_PARAMS[:2], *TEST_PARAMS[2:], 0.0, 0.1, 50, 50, 63, det_cap)
        faces = np.zeros((n, fcap), dtype=pigo_b200.DET_DTYPE)
        nfaces = np.zeros(n, dtype=np.int32)
        points = np.zeros((n, fcap, 2 + NCALLS), dtype=pigo_b200.POINT_DTYPE)
        rc = pigo_b200.lib().pigo_detect_images(gpu_face._h, plc._h, hs, fl.ctypes.data, NCALLS, desc, n, C.byref(prm), None, 0,
                                                faces.ctypes.data, fcap, nfaces.ctypes.data, points.ctypes.data, pigo_b200.MEM_HOST, None)
        assert rc == pigo_b200.PIGO_E_CAP
        assert msg in pigo_b200.lib().pigo_last_error().decode()
        if det_cap == 0:
            assert np.array_equal(nfaces, need)   # the required counts


def test_concurrent_calls_get_the_sequential_results(gpu_face, cascades, images, face_cap):
    plc, flp, _, _ = cascades
    subsets = [images[k::2] for k in range(2)]
    rnds = [randoms_for(len(s), face_cap, 31 + k) for k, s in enumerate(subsets)]
    expect = [pipeline.detect_images_device(gpu_face, plc, flp, s, cp_of(TEST_PARAMS), face_cap=face_cap, randoms=r, raw=True)
              for s, r in zip(subsets, rnds)]
    errors = []

    def work(k):
        try:
            for _ in range(2):
                got = pipeline.detect_images_device(gpu_face, plc, flp, subsets[k], cp_of(TEST_PARAMS), face_cap=face_cap, randoms=rnds[k], raw=True)
                if any(x.tobytes() != y.tobytes() for x, y in zip(got, expect[k])):
                    errors.append(k)
        except Exception as e:   # noqa: BLE001
            errors.append(repr(e))

    ts = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert errors == []


@pytest.mark.parametrize("knobs,angle", [({"scan_mode": 1}, 0.0), ({"rot_mode": 1}, 0.03)])
def test_universal_scan_options_give_the_same_results(gpu_face, cascades, images, face_cap, knobs, angle):
    """The images scan's own per-image fallback (universal gather kernel) under the pipeline."""
    plc, flp, _, _ = cascades
    some = [im for im in images if im.Rows * im.Cols <= 1080 * 1920]
    rnd = randoms_for(len(some), face_cap, 37)
    expect = pipeline.detect_images_device(gpu_face, plc, flp, some, cp_of(TEST_PARAMS), face_cap=face_cap, randoms=rnd, angle=angle, raw=True)
    with options(**knobs):
        got = pipeline.detect_images_device(gpu_face, plc, flp, some, cp_of(TEST_PARAMS), face_cap=face_cap, randoms=rnd, angle=angle, raw=True)
    assert_same_outputs(got, expect)
    assert expect[1].sum() > 0


@pytest.mark.parametrize("mode,stage", [(0, 0), (0, 1), (0, 2), (1, 0)])
def test_puploc_run_images_matches_the_oracle(mode, stage):
    """Both RunDetector kernels' image-table variants: seeds inside and past the borders of tall, wide and padded images,
    flips, Perturbs 0..63, rotated and not."""
    with options(puploc_mode=mode, puploc_stage=stage):
        _puploc_run_images_matches_the_oracle()


def _puploc_run_images_matches_the_oracle():
    ims = [make_image(700, 260, 272, "F", 3), make_image(300, 900, 912, "F", 4), make_image(333, 517, 531, "F", 5),
           ImageParams(synth.sample_gray(), 400, 320, 320), make_image(96, 128, 144, "S", 6)]
    rng = np.random.default_rng(77)
    for pkname in ("puploc", "lps/lp93"):
        pk = pigo_b200.load_cascade(pkname)
        plc = pigo_b200.NewPuplocCascade().UnpackCascade(pk)
        ora = O.OraclePuploc(pk)
        for ang in (0.0, 0.2, 0.93):
            seeds, which, flips, rnds = [], [], [], []
            for k in range(64):
                i = k % len(ims)
                im = ims[i]
                seeds.append(Puploc(int(rng.integers(-40, im.Rows + 40)), int(rng.integers(-40, im.Cols + 40)),
                                    float(np.float32(rng.uniform(2, 300))), k % 64))
                which.append(i)
                flips.append(bool(rng.integers(0, 2)))
                rnds.append(rng.random(189, dtype=np.float32))
            out = plc.run_detector_images(seeds, which, ims, ang, flips, np.stack(rnds))
            for s, i, f, r, o in zip(seeds, which, flips, rnds, out):
                im = ims[i]
                e = ora.run_detector(s.Row, s.Col, s.Scale, s.Perturbs, r, im.Pixels, im.Rows, im.Cols, im.Dim, ang, f)
                assert (o.Row, o.Col, np.float32(o.Scale)) == (e[0], e[1], np.float32(e[2])), (pkname, ang, i, s)


def test_cpp_mirror_detect_images():
    """tests/cpp/test_detect_images.cpp (built by build()): the reference's landmark assertions on the sample placed among
    other images, through DetectImages of include/pigo_b200.hpp, and its PIGO_E_CAP retry."""
    run_cpp_mirror("test_detect_images")
