"""pigo_blur_faces and pigo_blur_decoded on the H100: every byte of every plane, row padding included, equals the C oracle
(tests/blur_oracle.c) over formats, YCbCr ratios and origins, sizes, face placements and radii, host and device planes and
faces, the library's and a caller's stream; pigo_blur_decoded's faces equal gray_images -> RunCascadeImagesParams ->
ClusterDetections and its planes pigo_blur_faces on those faces."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import blur_oracle as B
import pigo_b200
from decoded_sources import face_gray
from option_guard import options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)
from pigo_b200 import DET_DTYPE, PIGO_E_CAP, PIGO_E_INVALID, BlurParams, CascadeParams

pytestmark = pytest.mark.gpu

FACEBLUR = (5.0, 0.5, 0.0, 15)


def pack(face_lists, cap=None):
    """[N][cap] DET_DTYPE and counts [N] of per-entry face arrays."""
    cap = max([len(f) for f in face_lists] + [1]) if cap is None else cap
    out = np.zeros((len(face_lists), max(cap, 1)), dtype=DET_DTYPE)
    for i, f in enumerate(face_lists):
        out[i, :min(cap, len(f))] = f[:cap]
    return out, np.array([len(f) for f in face_lists], dtype=np.int32)


def blur_lib(srcs, faces, counts, params, device_sources=False, device_faces=False, stream=None):
    """pigo_blur_faces on copies of srcs; returns them with their planes (whole buffers) back on the host."""
    work = [s.copy() for s in srcs]
    bp = BlurParams(*params)
    if device_sources:
        planes = [[torch.from_numpy(p).cuda() for p in s.planes] for s in work]
        decoded = [s.decoded(pl) for s, pl in zip(work, planes)]
    else:
        decoded = [s.decoded() for s in work]
    f, c = faces, counts
    if device_faces:
        f = torch.from_numpy(np.ascontiguousarray(faces).view(np.int32).reshape(len(srcs), -1, 4).copy()).cuda()
        c = torch.from_numpy(np.ascontiguousarray(counts, dtype=np.int32)).cuda()
    torch.cuda.synchronize()
    pigo_b200.blur_faces(decoded, f, c, bp, stream=stream, device_sources=device_sources, device_faces=device_faces)
    if stream is not None:
        stream.synchronize()
    if device_sources:
        for s, pl in zip(work, planes):
            s.planes = [p.cpu().numpy() for p in pl]
    return work


def blur_want(srcs, faces, counts, params):
    cap = faces.shape[1]
    return [B.blur_c(s, faces[i, :min(max(int(counts[i]), 0), cap)], *params) for i, s in enumerate(srcs)]


def assert_planes(got, want, what=""):
    for i, (g, w) in enumerate(zip(got, want)):
        for k, (a, b) in enumerate(zip(g.planes, w.planes)):
            assert np.array_equal(a, b), (what, i, k, g.fmt, g.w, g.h, int(np.count_nonzero(a != b)))


def seeded_batch(n=60, base=0):
    cases = [B.random_case(base + s) for s in range(n)]
    srcs = [c[0] for c in cases]
    faces, counts = pack([c[1] for c in cases])
    return srcs, faces, counts


@pytest.mark.parametrize("device_sources,device_faces,caller_stream", [(False, False, False), (True, False, False), (False, True, True),
                                                                       (True, True, True), (True, False, True)])
def test_seeded_batch_equals_the_c_oracle(device_sources, device_faces, caller_stream):
    srcs, faces, counts = seeded_batch()
    assert {s.fmt for s in srcs} == set(B.FORMATS)
    for params in (FACEBLUR, (5.0, 1.0, 0.5, 0), (-math.inf, 0.3, 2.0, 3)):
        st = torch.cuda.Stream() if caller_stream else None
        got = blur_lib(srcs, faces, counts, params, device_sources, device_faces, st)
        assert_planes(got, blur_want(srcs, faces, counts, params), params)


def edge_faces(w, h):
    """Faces inside, straddling the edges and centred outside; a point disc, R 0, R past the image, R clamped at 1023,
    overlapping discs of different R, a repeated face, q == min_q, NaN q, and the skipped bounds."""
    big = 1 << 24
    L = [(h // 2, w // 2, 8, 9.0), (0, w - 1, 12, 6.0), (-5, w // 3, 16, 7.0), (h + 3, -4, 20, 8.0), (h // 3, w // 4, 1, 9.0),
         (h // 2, w // 2, 0, 9.0), (h - 1, 0, 10, 5.0), (h // 2, w // 2 + 3, 30, 5.5), (h // 2, w // 2 + 3, 30, 5.5),
         (h // 4, w // 2, 6, float("nan")), (h // 2, w // 2, big + 1, 9.0), (big + 1, 0, 5, 9.0), (0, -big - 1, 5, 9.0),
         (h // 2, w // 2, -3, 9.0), (2 * h, 2 * w, 4 * max(w, h), 6.0)]
    return np.array(L, dtype=DET_DTYPE)


def geometry_sources():
    rng = np.random.default_rng(7)
    srcs = []
    for fmt in B.FORMATS:
        for (w, h) in ((1, 1), (37, 1), (1, 29), (17, 33)):
            srcs.append(B.make_src(fmt, w, h, rng, sub=(w + h) % 6, min_x=w % 5, min_y=h % 3, pad=3))
    for sub in range(6):
        srcs.append(B.make_src(0, 61, 45, rng, sub=sub, min_x=2 * sub + 1, min_y=sub % 2 + 1, pad=5))
    srcs.append(B.make_src(0, 1920, 1080, rng, sub=2, min_x=3, min_y=1, pad=16, luma=face_gray(1080, 1920, 3)))
    srcs.append(B.make_src(1, 1920, 1080, rng, pad=4))
    return srcs


@pytest.mark.parametrize("params", [FACEBLUR, (5.0, 0.5, 16.0, 0), (5.0, 1.0, 0.0, 1023), (-math.inf, 0.0, 0.0, 7)])
def test_geometries_and_face_placements(params):
    srcs = geometry_sources()
    faces, counts = pack([edge_faces(s.w, s.h) for s in srcs])
    got = blur_lib(srcs, faces, counts, params)
    assert_planes(got, blur_want(srcs, faces, counts, params), params)


def test_counts_are_clamped_to_face_cap():
    srcs, faces, counts = seeded_batch(12, base=500)
    counts = counts.copy()
    counts[::3] = faces.shape[1] + 40
    counts[1::3] = -7
    got = blur_lib(srcs, faces, counts, FACEBLUR, device_faces=True)
    assert_planes(got, blur_want(srcs, faces, counts, FACEBLUR))
    assert_planes(blur_lib(srcs, faces, counts, FACEBLUR), blur_want(srcs, faces, counts, FACEBLUR))


def test_a_4k_crowd_and_a_face_covering_4k():
    rng = np.random.default_rng(11)
    src = B.make_src(0, 3840, 2160, rng, sub=2, pad=8)
    crowd = np.zeros(2000, dtype=DET_DTYPE)
    crowd["row"], crowd["col"] = rng.integers(-20, 2180, 2000), rng.integers(-20, 3860, 2000)
    crowd["scale"], crowd["q"] = rng.integers(20, 160, 2000), rng.uniform(4, 12, 2000)
    faces, counts = pack([crowd])
    for params in (FACEBLUR, (5.0, 0.5, 0.25, 2)):
        assert_planes(blur_lib([src], faces, counts, params, device_sources=True), blur_want([src], faces, counts, params), "crowd")
    whole, counts = pack([np.array([(1080, 1920, 8000, 9.0)], dtype=DET_DTYPE)])
    params = (5.0, 0.5, 0.0, 1023)
    assert_planes(blur_lib([src], whole, counts, params), blur_want([src], whole, counts, params), "whole")


def test_a_capturing_stream_is_refused():
    srcs, faces, counts = seeded_batch(3)
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    decoded = [x.decoded() for x in srcs]
    with torch.cuda.graph(g, stream=s, capture_error_mode="relaxed"):
        rc = pigo_b200.lib().pigo_blur_faces(pigo_b200.decoded_descs(decoded), 3, faces.ctypes.data, faces.shape[1], counts.ctypes.data,
                                             C.byref(BlurParams(*FACEBLUR)), 0, s.cuda_stream)
    assert rc == PIGO_E_INVALID


# ---- pigo_blur_decoded ------------------------------------------------------------------------------------------------------
def face_sources():
    """Mixed formats with face content, per-image CascadeParams and angles (two rotated)."""
    rng = np.random.default_rng(21)
    shapes = [(0, 640, 480, 2, 1, 1), (1, 500, 400, 0, 0, 0), (2, 600, 360, 0, 0, 0), (3, 540, 420, 0, 0, 0), (8, 480, 480, 0, 0, 0),
              (0, 961, 541, 5, 3, 0)]
    srcs = [B.make_src(fmt, w, h, rng, sub=sub, min_x=mx, min_y=my, pad=7, luma=face_gray(h, w, 30 + k))
            for k, (fmt, w, h, sub, mx, my) in enumerate(shapes)]
    cps = [(20, 1000, 0.1, 1.1), (30, 800, 0.15, 1.1), (20, 1000, 0.2, 1.2), (20, 1000, 0.1, 1.1), (24, 600, 0.1, 1.15), (20, 1000, 0.1, 1.1)]
    angles = [0.0, 0.0, 0.05, 0.0, 0.0, 0.1]
    return srcs, cps, angles


def composition(gpu_face, srcs, cps, angles, iou):
    arena, images = pigo_b200.gray_images([s.decoded() for s in srcs])
    dets, cnt = gpu_face.RunCascadeImagesParams([CascadeParams(im, *cp) for im, cp in zip(images, cps)], angles)
    clusters, ncl = gpu_face.cluster_batch_array(dets, cnt, iou)
    del arena
    return clusters, ncl


def blur_decoded_raw(gpu_face, srcs, cps, angles, iou, params, face_cap, det_cap=0, stream=None):
    work = [s.copy() for s in srcs]
    faces = np.zeros((len(srcs), max(face_cap, 1)), dtype=DET_DTYPE)
    n_faces = np.zeros(len(srcs), dtype=np.int32)
    rc = pigo_b200.lib().pigo_blur_decoded(gpu_face._h, pigo_b200.decoded_descs([s.decoded() for s in work]), len(srcs),
                                           pigo_b200.cascade_params_array(cps), np.ascontiguousarray(angles, dtype=np.float64).ctypes.data, iou,
                                           det_cap, C.byref(BlurParams(*params)), faces.ctypes.data, face_cap, n_faces.ctypes.data, 0, stream)
    return rc, work, faces, n_faces


def test_blur_decoded_is_the_composition(gpu_face):
    srcs, cps, angles = face_sources()
    want_cl, want_n = composition(gpu_face, srcs, cps, angles, 0.1)
    assert (want_n > 0).sum() >= 3
    face_cap = int(want_n.max()) + 2
    pigo_b200.set_option("timing", 1)
    try:
        before = pigo_b200.launch_count()
        rc, got, faces, n_faces = blur_decoded_raw(gpu_face, srcs, cps, angles, 0.1, FACEBLUR, face_cap)
        assert rc == 0
        assert pigo_b200.get_option("t_blur_n") == 6 and pigo_b200.launch_count() - before > 6
    finally:
        pigo_b200.set_option("timing", 0)
    assert n_faces.tolist() == want_n.tolist()
    for i in range(len(srcs)):
        assert faces[i, :n_faces[i]].tobytes() == want_cl[i, :want_n[i]].tobytes()
        assert not faces[i, n_faces[i]:].view(np.uint8).any()
    assert_planes(got, blur_lib(srcs, faces, n_faces, FACEBLUR), "blur_faces")
    assert_planes(got, blur_want(srcs, faces, n_faces, FACEBLUR), "oracle")
    assert any(not np.array_equal(g.planes[0], s.planes[0]) for g, s in zip(got, srcs))
    # the mirror, on device planes and a caller's stream
    work = [s.copy() for s in srcs]
    planes = [[torch.from_numpy(p).cuda() for p in s.planes] for s in work]
    st = torch.cuda.Stream()
    lists = gpu_face.BlurDecoded([s.decoded(pl) for s, pl in zip(work, planes)], [CascadeParams(None, *cp) for cp in cps], angles, 0.1,
                                 BlurParams(*FACEBLUR), device_sources=True, stream=st)
    st.synchronize()
    assert [len(x) for x in lists] == want_n.tolist()
    for s, pl in zip(work, planes):
        s.planes = [p.cpu().numpy() for p in pl]
    assert_planes(work, got, "device planes")


def test_blur_decoded_capacity_errors(gpu_face):
    srcs, cps, angles = face_sources()
    _, full, faces_full, n_full = blur_decoded_raw(gpu_face, srcs, cps, angles, 0.1, FACEBLUR, 64)
    # more clusters than face_cap: every cluster is still blurred, n_faces holds the required counts
    small = int(n_full.max()) - 1
    rc, got, faces, n_faces = blur_decoded_raw(gpu_face, srcs, cps, angles, 0.1, FACEBLUR, small)
    assert rc == PIGO_E_CAP and n_faces.tolist() == n_full.tolist()
    assert faces[:, :small].tobytes() == faces_full[:, :small].tobytes()
    assert_planes(got, full, "face_cap")
    # more raw detections than det_cap: the entry is named and no plane is written
    rc, got, _, _ = blur_decoded_raw(gpu_face, srcs, cps, angles, 0.1, FACEBLUR, 64, det_cap=1)
    assert rc == PIGO_E_CAP and b"raw detections" in pigo_b200.lib().pigo_last_error()
    assert_planes(got, srcs, "det_cap")
    # the mirror retries det_cap and returns every face list
    lists = gpu_face.BlurDecoded([s.copy().decoded() for s in srcs], [CascadeParams(None, *cp) for cp in cps], angles, 0.1, BlurParams(*FACEBLUR),
                                 det_cap=1)
    assert [len(x) for x in lists] == n_full.tolist()
    # a capturing stream is refused
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s, capture_error_mode="relaxed"):
        rc = blur_decoded_raw(gpu_face, srcs, cps, angles, 0.1, FACEBLUR, 8, stream=s.cuda_stream)[0]
    assert rc == PIGO_E_INVALID
