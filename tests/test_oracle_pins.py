"""Pins the CPU oracle (oracle/pigo_oracle.c) against everything the reference's own tests assert for
this path (SURVEY.md section 8c) -- they are existential, not numeric -- against the independently written
numpy restatement (oracle/np_oracle.py) and against the committed oracle-generated vectors.

"parity unpinned": the reference is Go, no Go toolchain exists here, and core/*_test.go hold no goldens."""
import numpy as np
import pytest

import oracle_lib as O
import pigo_b200
from oracle import np_oracle as NP
from pigo_b200 import synth
from synthetic import synthetic_cascade

TEST_PARAMS = (20, 1000, 0.2, 1.1)  # core/pigo_test.go:44-50


def test_unpack_geometry(facefinder_bytes, oracle_face):
    assert (oracle_face.depth, oracle_face.ntrees) == (6, 468)
    assert len(facefinder_bytes) == 16 + 468 * 512
    pl = O.OraclePuploc(pigo_b200.load_cascade("puploc"))
    assert (pl.stages, pl.trees, pl.depth) == (5, 20, 10) and abs(pl.scales - 0.8) < 1e-6
    lp = O.OraclePuploc(pigo_b200.load_cascade("lps/lp42"))
    assert (lp.stages, lp.trees, lp.depth) == (6, 20, 9) and abs(lp.scales - 0.7) < 1e-6


def test_reference_assertion_face_detected(oracle_face, sample_gray):
    """core/pigo_test.go:68-84: len(ClusterDetections(RunCascade(...), 0.1)) > 0."""
    d = oracle_face.run_cascade(sample_gray, 400, 320, 320, *TEST_PARAMS, 0.0)
    _, cl = O.cluster(d, 0.1)
    assert len(cl) > 0
    # core/puploc_test.go:55-80 and flploc_test.go:150-153 imply exactly one face with Scale > 50
    assert sum(1 for c in cl if c["scale"] > 50) == 1


def test_reference_assertion_15_landmark_points(oracle_face, sample_gray):
    """core/flploc_test.go:75-154: 2*5 + 4 + 1 landmark points with Row>0 && Col>0 (randoms injected)."""
    d = oracle_face.run_cascade(sample_gray, 400, 320, 320, *TEST_PARAMS, 0.0)
    _, cl = O.cluster(d, 0.1)
    plc = O.OraclePuploc(pigo_b200.load_cascade("puploc"))
    rng = np.random.default_rng(123)
    pts = 0
    for det in cl:
        if det["scale"] <= 50:
            continue
        row = int(det["row"]) - int(np.float32(0.075) * np.float32(det["scale"]))
        sc = float(np.float32(det["scale"]) * np.float32(0.25))
        lc = int(det["col"]) - int(np.float32(0.175) * np.float32(det["scale"]))
        rc = int(det["col"]) + int(np.float32(0.185) * np.float32(det["scale"]))
        le = plc.run_detector(row, lc, sc, 50, rng.random(189, dtype=np.float32), sample_gray, 400, 320, 320)
        re_ = plc.run_detector(row, rc, sc, 50, rng.random(189, dtype=np.float32), sample_gray, 400, 320, 320)
        assert le[0] > 0 and le[1] > 0 and re_[0] > 0 and re_[1] > 0
        calls = [(e, f) for e in ("lp46", "lp44", "lp42", "lp38", "lp312") for f in (False, True)]
        calls += [(m, False) for m in ("lp93", "lp84", "lp82", "lp81")] + [("lp84", True)]
        for name, flip in calls:
            fl = O.OraclePuploc(pigo_b200.load_cascade("lps/" + name))
            r0, c0, s0 = O.landmark_seed(le[0], le[1], re_[0], re_[1])
            p = fl.run_detector(r0, c0, float(s0), 63, rng.random(189, dtype=np.float32), sample_gray, 400, 320, 320, 0.0, flip)
            if p[0] > 0 and p[1] > 0:
                pts += 1
    assert pts == 2 * 5 + 4 + 1


@pytest.mark.parametrize("angle", [0.0, 0.2, 0.55, 1.0])
def test_c_and_numpy_restatements_agree_on_sample(facefinder_bytes, oracle_face, sample_gray, angle):
    npf = NP.FaceCascade(facefinder_bytes)
    a = oracle_face.run_cascade(sample_gray, 400, 320, 320, 20, 1000, 0.1, 1.1, angle)
    b = npf.run_cascade(sample_gray, 400, 320, 320, 20, 1000, 0.1, 1.1, angle)
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert (x["row"], x["col"], x["scale"]) == (y[0], y[1], y[2]) and x["q"] == y[3]


def test_c_and_numpy_agree_on_noise_and_strided_frames(facefinder_bytes, oracle_face):
    npf = NP.FaceCascade(facefinder_bytes)
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, size=(97, 160), dtype=np.uint8)   # Dim (160) != Cols (131): Q7
    for ang in (0.0, 0.7):
        a = oracle_face.run_cascade(img, 97, 131, 160, 12, 90, 0.1, 1.2, ang)
        b = npf.run_cascade(img, 97, 131, 160, 12, 90, 0.1, 1.2, ang)
        assert [(x["row"], x["col"], x["scale"], x["q"]) for x in a] == [(y[0], y[1], y[2], y[3]) for y in b]
    # per-window scores incl. rejected ones
    rr, cc = NP.grid(97, 131, 24, 0.1)
    R, Cc = np.meshgrid(rr, cc, indexing="ij")
    q = npf.classify(R.ravel(), Cc.ravel(), 24, img, 97, 131, 160)
    for k in range(0, q.size, 7):
        assert q[k] == oracle_face.classify_region(int(R.ravel()[k]), int(Cc.ravel()[k]), 24, img, 160)


def test_rotation_slot_32_equals_unrotated_sampling(oracle_face, sample_gray):
    """angle 1.0 -> table slot 32 = (cos 256, sin 0): same sample points as the unrotated path wherever no
    clamp applies (core/pigo.go:156-171)."""
    a = oracle_face.run_cascade(sample_gray, 400, 320, 320, *TEST_PARAMS, 0.0)
    b = oracle_face.run_cascade(sample_gray, 400, 320, 320, *TEST_PARAMS, 1.0)
    assert [tuple(x) for x in a] == [tuple(x) for x in b]


def test_cluster_c_vs_numpy(oracle_face):
    fr = synth.frame_faces(None, 720, 1280, noise_seed=3)
    d = oracle_face.run_cascade(fr, 720, 1280, 1280, *TEST_PARAMS, 0.0)
    assert len(d) > 10
    for thr in (0.0, 0.1, 0.2, 0.5):
        srt, cl = O.cluster(d, thr)
        s2, c2 = NP.cluster_detections([tuple(x) for x in d], thr)
        assert [tuple(x) for x in srt] == [(a[0], a[1], a[2], a[3]) for a in s2]
        assert [tuple(x) for x in cl] == [(a[0], a[1], a[2], a[3]) for a in c2]


def test_puploc_c_vs_numpy(sample_gray):
    pk = pigo_b200.load_cascade("puploc")
    a, b = O.OraclePuploc(pk), NP.PuplocCascade(pk)
    rnd = np.random.default_rng(11).random(189, dtype=np.float32)
    for (r, c, s, ang, fl) in [(180, 110, 60.0, 0.0, False), (180, 200, 55.5, 0.0, True), (185, 120, 70.0, 0.3, False),
                               (10, 5, 90.0, 0.0, False), (395, 318, 80.0, 0.9, True)]:
        x = a.classify(np.float32(r), np.float32(c), np.float32(s), sample_gray, 400, 320, 320, ang, fl)
        y = b.classify(r, c, s, sample_gray, 400, 320, 320, ang, fl)
        assert x == y
    for P in (63, 50, 7, 0):
        x = a.run_detector(180, 110, 60.0, P, rnd, sample_gray, 400, 320, 320, 0.0, False)
        y = b.run_detector(180, 110, 60.0, P, rnd, sample_gray, 400, 320, 320, 0.0, False)
        assert x == y
    with pytest.raises(ValueError):
        a.run_detector(180, 110, 60.0, 64, np.zeros(192, np.float32), sample_gray, 400, 320, 320)


def test_committed_vectors_still_reproduce(golden, oracle_face, sample_gray):
    d = oracle_face.run_cascade(sample_gray, 400, 320, 320, *TEST_PARAMS, 0.0)
    assert d.tobytes() == golden["sample_test_dets"].tobytes()
    assert O.cluster(d, 0.1)[1].tobytes() == golden["sample_test_clusters"].tobytes()
    assert oracle_face.run_cascade(sample_gray, 400, 320, 320, 20, 1000, 0.1, 1.1).tobytes() == golden["sample_doc_dets"].tobytes()
    for k in (1, 5, 8, 16, 27, 32):
        assert oracle_face.run_cascade(sample_gray, 400, 320, 320, *TEST_PARAMS, k / 32.0).tobytes() == golden[f"sample_rot{k}_dets"].tobytes()
    f1080 = synth.frame_faces(sample_gray, 1080, 1920)
    assert oracle_face.run_cascade(f1080, 1080, 1920, 1920, *TEST_PARAMS, 0.0).tobytes() == golden["f1080_test_dets"].tobytes()
    pl = O.OraclePuploc(pigo_b200.load_cascade("puploc"))
    for row in golden["puploc_cases"]:
        r0, cc, sc, P, ang, fl, o0, o1, o2 = row
        o = pl.run_detector(int(r0), int(cc), float(sc), int(P), golden["puploc_randoms"], sample_gray, 400, 320, 320, float(ang), bool(fl))
        assert (o[0], o[1]) == (int(o0), int(o1)) and np.float32(o[2]) == np.float32(o2)


def test_grayscale_restatements_agree():
    rgba = np.random.default_rng(2).integers(0, 256, size=(50, 40, 4), dtype=np.uint8)
    rgba[..., 3] = 255
    assert np.array_equal(O.rgba_to_gray(rgba), NP.rgb_to_grayscale(rgba[..., :3]))


@pytest.mark.parametrize("depth,ntrees", [(6, 3), (6, 40), (4, 9), (1, 2), (8, 5), (6, 1)])
def test_c_and_numpy_agree_on_random_cascades_of_any_depth(depth, ntrees):
    """Both restatements are generic in tree depth and count (core/pigo.go:113-147 reads them from the packet): random
    cascades, extreme codes (-128 / 127) included, unrotated and rotated, same detections and bit-equal scores."""
    from pigo_b200 import synth
    pk = synthetic_cascade(depth, ntrees, seed=depth * 100 + ntrees)
    c_or, np_or = O.OracleFace(pk), NP.FaceCascade(pk)
    assert (c_or.depth, c_or.ntrees) == (depth, ntrees) == (np_or.depth, np_or.ntrees)
    img = synth.frame_smooth(150, 210, seed=depth + ntrees, sigma=3.0)
    total = 0
    for ang in (0.0, 0.4):
        a = c_or.run_cascade(img, 150, 210, 210, 20, 120, 0.2, 1.2, ang, cap=1 << 16)
        b = np_or.run_cascade(img, 150, 210, 210, 20, 120, 0.2, 1.2, ang)
        assert [(x["row"], x["col"], x["scale"], x["q"]) for x in a] == [(y[0], y[1], y[2], y[3]) for y in b]
        total += len(a)
    assert total > 0


def test_ycbcr_restatement_is_within_one_of_the_reference_tests_formula():
    """core/image_test.go:92-148 restates the YCbCr->RGB conversion with ROUNDING ((yy<<16 + 91881*cr + 1<<15) >> 16) and accepts
    a difference of 1 against ImgToNRGBA (color.YCbCrToRGB, which truncates after multiplying y by 0x10101): the oracle's
    restatement of the latter must satisfy the same pin for the six subsample ratios the test covers."""
    import oracle_lib as O
    for sub in range(6):
        for (w, h, mx, my) in ((16, 16, 0, 0), (31, 17, 2, 3)):
            y, cb, cr = O.make_ycbcr_planes(7 * sub + w, sub, w, h, mx, my)
            got = O.ycbcr_to_nrgba(y, cb, cr, sub, w, h, mx, my).astype(np.int64)
            xd = {0: 1, 1: 2, 2: 2, 3: 1, 4: 4, 5: 4}[sub]
            yd = {0: 1, 1: 1, 2: 2, 3: 2, 4: 1, 5: 2}[sub]
            for dy in range(h):
                for dx in range(w):
                    yy = int(y[dy, dx])
                    ci, cj = (my + dy) // yd - my // yd, (mx + dx) // xd - mx // xd
                    b_, r_ = int(cb[ci, cj]) - 128, int(cr[ci, cj]) - 128
                    r = min(255, max(0, (yy * 65536 + 91881 * r_ + 32768) >> 16))
                    g = min(255, max(0, (yy * 65536 - 22554 * b_ - 46802 * r_ + 32768) >> 16))
                    b = min(255, max(0, (yy * 65536 + 116130 * b_ + 32768) >> 16))
                    assert abs(got[dy, dx, 0] - r) <= 1 and abs(got[dy, dx, 1] - g) <= 1 and abs(got[dy, dx, 2] - b) <= 1
                    assert got[dy, dx, 3] == 255


def test_c_and_numpy_restatements_agree_on_random_calls(facefinder_bytes, oracle_face, sample_gray):
    """The two independently written restatements (C, window-vectorised numpy) on 14 random calls -- geometry, stride, size range,
    ShiftFactor, ScaleFactor, angle, content -- from the same generator the GPU fuzz uses (tests/test_gpu_parity.py::_fuzz_case):
    identical detections, bit-equal scores.  Half of the cases contain the sample face rotated by the call's angle."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("gpu_parity_cases", os.path.join(os.path.dirname(__file__), "test_gpu_parity.py"))
    src = open(spec.origin).read()
    a, b = src.index("def _fuzz_case"), src.index("def test_random_geometry_and_parameter_fuzz")
    ns = {"np": np}
    exec(src[a:b], ns)                       # only the case generator (the module itself is GPU-marked)
    npf = NP.FaceCascade(facefinder_bytes)
    rng = np.random.default_rng(77)
    total = 0
    for case in range(14):
        buf, rows, cols, dim, prm, ang, kind = ns["_fuzz_case"](rng, sample_gray, case)
        x = oracle_face.run_cascade(buf, rows, cols, dim, *prm, ang)
        y = npf.run_cascade(buf, rows, cols, dim, *prm, ang)
        assert [(d["row"], d["col"], d["scale"], d["q"]) for d in x] == [(d[0], d[1], d[2], d[3]) for d in y], (case, rows, cols, dim, prm, ang)
        total += len(x)
    assert total > 50
