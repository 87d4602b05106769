"""pigo_blur_faces / pigo_blur_decoded without a device: the C and numpy restatements of the blur agree byte for byte, the
Rmax rule and the chroma anchoring on hand-computed cases, and every argument the calls reject fails with PIGO_E_INVALID
before any device work."""
import ctypes as C
import math

import numpy as np
import pytest

import blur_oracle as B
from abi_cases import FAKE
import pigo_b200
from pigo_b200 import DET_DTYPE, PIGO_E_INVALID, BlurParams, DecodedImage


def both(src, faces, params):
    return B.blur_c(src, faces, *params), B.blur_np(src, faces, *params)


def test_c_and_numpy_restatements_agree_on_seeded_cases():
    changed = 0
    for seed in range(300):
        src, faces, params = B.random_case(seed)
        c, n = both(src, faces, params)
        for k, (a, b) in enumerate(zip(c.planes, n.planes)):
            assert np.array_equal(a, b), (seed, k)
        changed += any(not np.array_equal(a, s) for a, s in zip(c.planes, src.planes))
    assert changed > 100   # the cases blur something


def test_rmax_rule_on_a_row():
    """Two discs on a 9x1 Gray row share pixel 3: it takes the larger box (R 3, not 1), in either face order."""
    row = np.array([90, 0, 0, 0, 0, 0, 0, 0, 30], np.uint8)
    src = B.BlurSrc(3, 9, 1, [row.copy()], (9, 0))
    faces = np.array([(0, 2, 2, 6.0), (0, 6, 6, 6.0)], dtype=DET_DTYPE)   # d 1, R 1 and d 3, R 3
    want = [90, 30, 0, 13, 0, 4, 9, 13, 17]
    for f in (faces, faces[::-1]):
        for out in both(src, f, (5.0, 0.5, 0.5, 0)):
            assert out.planes[0].tolist() == want


def test_chroma_samples_follow_their_anchor():
    """4:2:0 at origin (1, 1), 4x2: the chroma columns anchor at luma columns 0, 1 and 3 (the last clamped into the
    rectangle), so a point disc at column 3 blurs chroma column 2 and one at column 2 blurs no chroma sample."""
    y = np.array([[1, 2, 3, 4], [5, 6, 7, 8]], np.uint8)
    cb = np.array([[10, 20, 30], [40, 50, 60]], np.uint8)
    cr = np.array([[100, 110, 120], [130, 140, 150]], np.uint8)
    src = B.BlurSrc(0, 4, 2, [y.reshape(-1).copy(), cb.reshape(-1).copy(), cr.reshape(-1).copy()], (4, 3), sub=2, min_x=1, min_y=1)
    assert src.chroma() == (2, 3)
    params = (5.0, 0.5, 0.0, 2)   # scale 1: d 0, R 2 (chroma radii 1, 1)
    for out in both(src, np.array([(0, 3, 1, 9.0)], dtype=DET_DTYPE), params):
        assert out.planes[0].reshape(2, 4).tolist() == [[1, 2, 3, 5], [5, 6, 7, 8]]
        assert out.planes[1].reshape(2, 3).tolist() == [[10, 20, 37], [40, 50, 60]]
        assert out.planes[2].reshape(2, 3).tolist() == [[100, 110, 127], [130, 140, 150]]
    for out in both(src, np.array([(0, 2, 1, 9.0)], dtype=DET_DTYPE), params):
        assert out.planes[0].reshape(2, 4).tolist() == [[1, 2, 4, 4], [5, 6, 7, 8]]
        assert np.array_equal(out.planes[1], src.planes[1]) and np.array_equal(out.planes[2], src.planes[2])


def test_face_selection_rules():
    """q == min_q is blurred, NaN q and the out-of-range faces are not; min_q = -inf blurs every non-NaN face."""
    rng = np.random.default_rng(5)
    src = B.make_src(3, 20, 20, rng)
    one = lambda r, c, s, q: np.array([(r, c, s, q)], dtype=DET_DTYPE)
    p = (5.0, 0.5, 0.0, 2)
    assert not np.array_equal(B.blur_np(src, one(10, 10, 8, 5.0), *p).planes[0], src.planes[0])
    for f in (one(10, 10, 8, np.nan), one(10, 10, -1, 9.0), one(10, 10, (1 << 24) + 1, 9.0), one((1 << 24) + 1, 10, 8, 9.0),
              one(10, -(1 << 24) - 1, 8, 9.0), one(10, 10, 8, 4.99)):
        for out in both(src, f, p):
            assert np.array_equal(out.planes[0], src.planes[0]), f
    assert not np.array_equal(B.blur_np(src, one(10, 10, 8, -1e30), -math.inf, 0.5, 0.0, 2).planes[0], src.planes[0])


# ---- argument checks (no device needed) --------------------------------------------------------------------------------------
def _sources():
    rng = np.random.default_rng(1)
    return [B.make_src(0, 40, 29, rng, sub=2, min_x=1, min_y=1), B.make_src(1, 5, 7, rng, pad=3), B.make_src(2, 5, 6, rng),
            B.make_src(3, 1, 1, rng), B.make_src(8, 6, 3, rng)]


def _blur(decoded, params=BlurParams(5.0, 0.5, 0.0, 15), face_cap=2, n=None, faces=True, counts=True):
    L = pigo_b200.lib()
    k = len(decoded)
    f = np.zeros((max(k, 1), max(face_cap, 1)), dtype=DET_DTYPE)
    c = np.zeros(max(k, 1), dtype=np.int32)
    return L.pigo_blur_faces(pigo_b200.decoded_descs(decoded), k if n is None else n, f.ctypes.data if faces else None, face_cap,
                             c.ctypes.data if counts else None, C.byref(params) if params is not None else None, 0, None)


@pytest.fixture
def face():
    """A Pigo whose handle the argument checks never dereference (each call fails on an earlier argument)."""
    clf = pigo_b200.NewPigo()
    clf._h = FAKE
    yield clf
    clf._h = None


def _blur_decoded(face, decoded, params=BlurParams(5.0, 0.5, 0.0, 15), face_cap=2, cps=None, det_cap=0, handle=True, n_faces=True):
    L = pigo_b200.lib()
    k = len(decoded)
    cp = pigo_b200.cascade_params_array(cps if cps is not None else [(20, 1000, 0.1, 1.1)] * max(k, 1))
    f = np.zeros((max(k, 1), max(face_cap, 1)), dtype=DET_DTYPE)
    c = np.zeros(max(k, 1), dtype=np.int32)
    return L.pigo_blur_decoded(face._h if handle else None, pigo_b200.decoded_descs(decoded), k, cp, None, 0.1, det_cap,
                               C.byref(params) if params is not None else None, f.ctypes.data, face_cap, c.ctypes.data if n_faces else None, 0, None)


def _bad_source(**kw):
    s = _sources()[kw.pop("which", 0)].decoded()
    d = dict(format=s.format, width=s.width, height=s.height, planes=s.planes, strides=s.strides, subsample=s.subsample, min_x=s.min_x, min_y=s.min_y)
    d.update(kw)
    return DecodedImage(**d)


BAD_SOURCES = [dict(format=4), dict(format=-1), dict(subsample=6), dict(min_x=-1), dict(width=0), dict(height=0), dict(strides=(39, 21)),
               dict(strides=(40, 19)), dict(which=1, strides=(19, 0)), dict(planes=(None, np.zeros(8, np.uint8), np.zeros(8, np.uint8))),
               dict(which=3, planes=(None,)), dict(which=4, strides=(23, 0)),
               # decodable, but not blurred: Gray16, RGBA64, NRGBA64 and Paletted
               dict(which=3, format=5, strides=(2, 0)), dict(which=1, format=6, strides=(40, 0)), dict(which=1, format=7, strides=(40, 0)),
               dict(which=3, format=9, planes=(np.zeros(1, np.uint8), np.zeros(4, np.uint8)), strides=(1, 1))]
BAD_PARAMS = [None, BlurParams(5.0, 0.5, 0.0, -1), BlurParams(5.0, 0.5, 0.0, 1024), BlurParams(5.0, math.nan, 0.0, 15),
              BlurParams(5.0, 0.5, math.nan, 15), BlurParams(5.0, -0.1, 0.0, 15), BlurParams(5.0, 0.5, -1e-9, 15),
              BlurParams(5.0, 16.5, 0.0, 15), BlurParams(5.0, 0.5, 17.0, 15), BlurParams(math.nan, 0.5, 0.0, 15)]


@pytest.mark.parametrize("bad", BAD_SOURCES)
def test_invalid_sources_fail_without_a_device(face, bad):
    decoded = [s.decoded() for s in _sources()] + [_bad_source(**bad)]
    assert _blur(decoded) == PIGO_E_INVALID
    assert _blur_decoded(face, decoded) == PIGO_E_INVALID


@pytest.mark.parametrize("k", range(len(BAD_PARAMS)))
def test_invalid_parameters_fail_without_a_device(face, k):
    decoded = [s.decoded() for s in _sources()]
    assert _blur(decoded, params=BAD_PARAMS[k]) == PIGO_E_INVALID
    assert _blur_decoded(face, decoded, params=BAD_PARAMS[k]) == PIGO_E_INVALID


def test_invalid_calls_fail_without_a_device(face):
    decoded = [s.decoded() for s in _sources()]
    L = pigo_b200.lib()
    repeated = decoded + [decoded[2]]
    assert _blur(repeated) == PIGO_E_INVALID and _blur_decoded(face, repeated) == PIGO_E_INVALID
    assert _blur(decoded, face_cap=-1) == PIGO_E_INVALID and _blur_decoded(face, decoded, face_cap=-1) == PIGO_E_INVALID
    assert _blur(decoded, n=-1) == PIGO_E_INVALID and _blur(decoded * 13108, n=65536) == PIGO_E_INVALID
    assert _blur(decoded, faces=False) == PIGO_E_INVALID and _blur(decoded, counts=False) == PIGO_E_INVALID
    assert L.pigo_blur_faces(None, 1, None, 0, None, C.byref(BlurParams(5.0, 0.5, 0.0, 15)), 0, None) == PIGO_E_INVALID
    assert _blur_decoded(face, decoded, handle=False) == PIGO_E_INVALID
    assert _blur_decoded(face, decoded, n_faces=False) == PIGO_E_INVALID
    assert _blur_decoded(face, decoded, det_cap=-1) == PIGO_E_INVALID
    # the scan's own checks on the decoded geometry: a ladder pigo_run_cascade rejects, named by its entry
    bad = [(20, 1000, 0.1, 1.1)] * 4 + [(-30, 10, 0.2, 1.1)]   # a negative window size
    assert _blur_decoded(face, decoded, cps=bad) == PIGO_E_INVALID
    assert b"image 4" in L.pigo_last_error()
    cp = pigo_b200.cascade_params_array([(20, 1000, 0.1, 1.1)] * 5)
    assert L.pigo_blur_decoded(face._h, pigo_b200.decoded_descs(decoded), len(decoded), None, None, 0.1, 0, C.byref(BlurParams(5.0, 0.5, 0.0, 15)),
                               None, 0, (C.c_int * 5)(), 0, None) == PIGO_E_INVALID
    assert L.pigo_blur_decoded(face._h, pigo_b200.decoded_descs(decoded), len(decoded), cp, None, 0.1, 0, C.byref(BlurParams(5.0, 0.5, 0.0, 15)),
                               None, 3, (C.c_int * 5)(), 0, None) == PIGO_E_INVALID   # null faces with face_cap > 0
