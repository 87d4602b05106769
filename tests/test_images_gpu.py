"""pigo_run_cascade_images: RunCascade over images of different sizes in one call.  Bar: every image's slice equals a
lone pigo_run_cascade on that image byte for byte (emission order, bit-equal Q) and, up to 1080p, the C oracle."""
import threading

import numpy as np
import pytest

import pigo_b200
from mixed_images import CLI_PARAMS, DOC_PARAMS, KNOBS, MIXED, TEST_PARAMS, assert_slices, cp_of, lone_scan, make_image, run_cpp_mirror
from pigo_b200 import CascadeParams, ImageParams, synth
from option_guard import options, options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)
from synthetic import synthetic_cascade

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mixed():
    return [make_image(r, c, d, k, 11 + i) for i, (r, c, d, k) in enumerate(MIXED)]


@pytest.fixture(scope="module")
def wide(mixed):
    """Images with Cols >= Rows: the rotated scan clamps columns with Rows-1 (core/pigo.go:168,:171), which bites here, and
    never reads past the image (on tall images it can, where the reference itself would index out of range)."""
    return [im for im in mixed if im.Cols >= im.Rows] + [make_image(300, 900, 900, "F", 5), make_image(200, 1200, 1216, "S", 6)]


@pytest.mark.parametrize("params", [TEST_PARAMS, CLI_PARAMS, DOC_PARAMS])
def test_each_image_equals_a_lone_call_and_the_oracle(gpu_face, oracle_face, mixed, params):
    dets, cnt = gpu_face.RunCascadeImages(mixed, cp_of(params))
    expect = [lone_scan(gpu_face, im, params) for im in mixed]
    assert_slices(dets, cnt, expect)
    assert sum(len(e) for e in expect) > 0
    for i, im in enumerate(mixed):
        if im.Rows * im.Cols <= 1080 * 1920:
            o = oracle_face.run_cascade(im.Pixels, im.Rows, im.Cols, im.Dim, *params, 0.0)
            assert expect[i].tobytes() == o.tobytes(), f"image {i} differs from the oracle"


@pytest.mark.parametrize("angle", [1 / 32, 7 / 32, 16 / 32, 31 / 32, 1.0, 1.3])
def test_rotated_each_image_equals_a_lone_call(gpu_face, wide, angle):
    dets, cnt = gpu_face.RunCascadeImages(wide, cp_of(TEST_PARAMS), angle)
    assert_slices(dets, cnt, [lone_scan(gpu_face, im, TEST_PARAMS, angle) for im in wide])


@pytest.mark.parametrize("angle", [0.0, 0.25])
def test_one_geometry_equals_the_batch_call(gpu_face, angle):
    frames = synth.make_batch(5, 540, 960, "USF", seed0=31)
    bd, bc = gpu_face.RunCascadeBatch(frames, CascadeParams(ImageParams(None, 540, 960, 960), *TEST_PARAMS), angle, 256)
    dets, cnt = gpu_face.RunCascadeImages([ImageParams(f, 540, 960, 960) for f in frames], cp_of(TEST_PARAMS), angle, 256)
    assert np.array_equal(cnt, bc) and cnt.sum() > 0
    for i in range(5):
        assert dets[i, :cnt[i]].tobytes() == bd[i, :cnt[i]].tobytes()


def test_shuffled_order_permutes_the_outputs(gpu_face, mixed):
    d0, c0 = gpu_face.RunCascadeImages(mixed, cp_of(TEST_PARAMS))
    perm = np.random.default_rng(3).permutation(len(mixed))
    d1, c1 = gpu_face.RunCascadeImages([mixed[j] for j in perm], cp_of(TEST_PARAMS))
    for k, j in enumerate(perm):
        assert c1[k] == c0[j] and d1[k, :c1[k]].tobytes() == d0[j, :c0[j]].tobytes()


def test_host_device_and_stream_forms_agree(gpu_face, mixed):
    import torch
    hd, hc = gpu_face.RunCascadeImages(mixed, cp_of(TEST_PARAMS))
    bufs = [torch.from_numpy(np.ascontiguousarray(im.Pixels).reshape(-1)[:max(im.Rows * im.Dim, 1)].copy()).cuda() for im in mixed]
    dd, dc = gpu_face.RunCascadeImages([ImageParams(b.data_ptr(), im.Rows, im.Cols, im.Dim) for b, im in zip(bufs, mixed)],
                                       cp_of(TEST_PARAMS))
    assert np.array_equal(dc, hc)
    for i in range(len(mixed)):
        assert dd[i, :dc[i]].tobytes() == hd[i, :hc[i]].tobytes()
    n, cap = len(mixed), max(int(hc.max()), 1)
    out = torch.zeros((n, cap, 4), dtype=torch.int32, device="cuda")
    cnt = torch.zeros(n, dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for _ in range(2):   # back-to-back asynchronous calls reuse the same workspace
            gpu_face.run_cascade_images_device([(b.data_ptr(), im.Rows, im.Cols, im.Dim) for b, im in zip(bufs, mixed)], *TEST_PARAMS, 0.0,
                                               out.data_ptr(), cap, cnt.data_ptr(), st.cuda_stream)
    st.synchronize()
    o = out.cpu().numpy().view(np.uint8).reshape(n, cap, 16)
    assert np.array_equal(cnt.cpu().numpy(), hc)
    for i in range(n):
        assert o[i, :hc[i]].tobytes() == hd[i, :hc[i]].tobytes()


@pytest.mark.parametrize("knobs", KNOBS)
def test_options_leave_the_outputs_unchanged(gpu_face, wide, knobs):
    expect = {a: gpu_face.RunCascadeImages(wide, cp_of(TEST_PARAMS), a) for a in (0.0, 0.5)}
    with options(**knobs):
        for a, (ed, ec) in expect.items():
            d, c = gpu_face.RunCascadeImages(wide, cp_of(TEST_PARAMS), a)
            assert np.array_equal(c, ec), a
            for i in range(len(wide)):
                assert d[i, :c[i]].tobytes() == ed[i, :ec[i]].tobytes(), (a, i)


def test_cascade_of_another_depth_takes_the_single_image_path(mixed):
    face = pigo_b200.NewPigo().Unpack(synthetic_cascade(4, 9, seed=409))
    some = mixed[:12]
    dets, cnt = face.RunCascadeImages(some, cp_of(TEST_PARAMS), 0.0)
    assert_slices(dets, cnt, [lone_scan(face, im, TEST_PARAMS) for im in some])
    assert cnt.sum() > 0


def test_capacity_error_reports_the_required_counts(gpu_face, mixed):
    _, c = gpu_face.RunCascadeImages(mixed, cp_of(TEST_PARAMS))
    assert c.max() > 2
    desc = pigo_b200.image_descs([(im.Pixels.ctypes.data, im.Rows, im.Cols, im.Dim) for im in mixed])
    out = np.zeros((len(mixed), 2), dtype=pigo_b200.DET_DTYPE)
    cnt = np.zeros(len(mixed), dtype=np.int32)
    rc = pigo_b200.lib().pigo_run_cascade_images(gpu_face._h, desc, len(mixed), *TEST_PARAMS, 0.0, out.ctypes.data, 2, cnt.ctypes.data,
                                                 pigo_b200.MEM_HOST, None)
    assert rc == pigo_b200.PIGO_E_CAP
    assert np.array_equal(cnt, c)


@pytest.mark.parametrize("angle", [0.0, 0.4])
def test_mixed_calls_leave_the_uniform_plan_cache_alone(gpu_face, wide, angle):
    """One thread, so that the calls reuse one workspace: a uniform call, a mixed-size call with a longer ladder and the same
    rotation slot, the uniform call again -- each result unchanged."""
    frames = synth.make_batch(2, 360, 640, "FS", seed0=41)
    cpu = CascadeParams(ImageParams(None, 360, 640, 640), *TEST_PARAMS)
    d0, c0 = gpu_face.RunCascadeBatch(frames, cpu, angle, 1024)
    m0, k0 = gpu_face.RunCascadeImages(wide, cp_of(TEST_PARAMS), angle)
    d1, c1 = gpu_face.RunCascadeBatch(frames, cpu, angle, 1024)
    m1, k1 = gpu_face.RunCascadeImages(wide, cp_of(TEST_PARAMS), angle)
    assert np.array_equal(c0, c1) and d0.tobytes() == d1.tobytes()
    assert np.array_equal(k0, k1) and m0.tobytes() == m1.tobytes()
    assert_slices(m0, k0, [lone_scan(gpu_face, im, TEST_PARAMS, angle) for im in wide])


def test_concurrent_mixed_calls_on_one_classifier(gpu_face, mixed):
    subsets = [mixed[i::4] for i in range(4)]
    expect = [gpu_face.RunCascadeImages(s, cp_of(TEST_PARAMS)) for s in subsets]
    errors = []

    def work(k):
        try:
            for _ in range(3):
                d, c = gpu_face.RunCascadeImages(subsets[k], cp_of(TEST_PARAMS))
                ed, ec = expect[k]
                if not np.array_equal(c, ec) or any(d[i, :c[i]].tobytes() != ed[i, :ec[i]].tobytes() for i in range(len(c))):
                    errors.append(k)
        except Exception as e:   # noqa: BLE001
            errors.append(repr(e))

    ts = [threading.Thread(target=work, args=(k,)) for k in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert errors == []


def test_cluster_batch_on_the_output_equals_per_image_clustering(gpu_face, mixed):
    d, c = gpu_face.RunCascadeImages(mixed, cp_of(TEST_PARAMS))
    cl, k = gpu_face.cluster_batch_array(d.copy(), c, 0.1)
    for i in range(len(mixed)):
        _, e = gpu_face.cluster_array(d[i, :c[i]].copy(), 0.1)
        assert int(k[i]) == len(e) and cl[i, :k[i]].tobytes() == e.tobytes(), i


def test_cpp_mirror_sample_inside_a_mixed_batch():
    """tests/cpp/test_images.cpp (built by build()): the reference's >= 1 face assertion on the sample image placed inside a
    mixed-size batch, through include/pigo_b200.hpp."""
    run_cpp_mirror("test_images")
