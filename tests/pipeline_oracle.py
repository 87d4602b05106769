"""Step-by-step replay of the face -> cluster -> pupils -> 15 landmarks pipeline on the C oracle (core/flploc_test.go:75-154):
eye seeds -> RunDetector x2 -> landmark seed -> 15 x RunDetector per face of scale > 50, with the randoms the library was
given, against the library's (faces, n_faces, points) outputs."""
import numpy as np

import oracle_lib as O
import pigo_b200
from pigo_b200 import pipeline


def oracle_cascades():
    """(puploc, {name: landmark cascade}) on the C oracle."""
    names = sorted(set(pipeline.EYE_CASCADES + pipeline.MOUTH_CASCADES))
    return O.OraclePuploc(pigo_b200.load_cascade("puploc")), {n: O.OraclePuploc(pigo_b200.load_cascade("lps/" + n)) for n in names}


def oracle_clusters(oracle_face, image, params, angle, iou=0.1):
    """ClusterDetections(RunCascade) of image = (pixels, rows, cols, dim) on the C oracle."""
    return O.cluster(oracle_face.run_cascade(*image, *params, angle), iou)[1]


def oracle_points(oracle, image, clusters, angles, randoms, eye):
    """The 2 eyes and 15 landmarks of every face of `clusters` on the oracle: the eyes at angles[k] with randoms(k, 0) and
    randoms(k, 1), landmark call c at angle 0 with randoms(k, 2 + c).  Faces of scale <= 50 keep zero points."""
    oplc, oflp = oracle
    angles = np.broadcast_to(np.asarray(angles, dtype=np.float64), len(clusters))
    calls = pipeline.landmark_calls()
    out = np.zeros((len(clusters), 2 + len(calls)), dtype=pigo_b200.POINT_DTYPE)
    for k, f in enumerate(clusters):
        if f["scale"] <= 50:
            continue
        ls, rs = pipeline.eye_seeds(int(f["row"]), int(f["col"]), int(f["scale"]), eye)
        le = oplc.run_detector(ls.Row, ls.Col, ls.Scale, eye, randoms(k, 0), *image, angles[k])
        re_ = oplc.run_detector(rs.Row, rs.Col, rs.Scale, eye, randoms(k, 1), *image, angles[k])
        out[k, 0], out[k, 1] = le[:3] + (0,), re_[:3] + (0,)
        for ci, (name, flip) in enumerate(calls):
            out[k, 2 + ci] = oracle_landmark(oflp[name], le, re_, randoms(k, 2 + ci), image, flip)[:3] + (0,)
    return out


def oracle_landmark(cascade, left_eye, right_eye, randoms, image, flip):
    """GetLandmarkPoint on the oracle: RunDetector from the landmark seed of the eyes' (row, col), Perturbs 63, angle 0."""
    r0, c0, s0 = O.landmark_seed(left_eye[0], left_eye[1], right_eye[0], right_eye[1])
    return cascade.run_detector(r0, c0, float(s0), 63, randoms, *image, 0.0, flip)


def face_arrays(face_lists):
    """The (faces, n_faces, points) arrays of per-image Face lists (pipeline.detect_batch's form); a face without eyes has
    zero points."""
    n, cap = len(face_lists), max([len(fl) for fl in face_lists] + [1])
    faces = np.zeros((n, cap), dtype=pigo_b200.DET_DTYPE)
    points = np.zeros((n, cap, 2 + len(pipeline.landmark_calls())), dtype=pigo_b200.POINT_DTYPE)
    for i, fl in enumerate(face_lists):
        for k, fc in enumerate(fl):
            faces[i, k] = fc.det
            if fc.left_eye is not None:
                points[i, k] = [(p.Row, p.Col, p.Scale, p.Perturbs) for p in [fc.left_eye, fc.right_eye] + fc.landmarks]
    return faces, np.array([len(fl) for fl in face_lists]), points


def replay(oracle, cases, randoms, eye, got):
    """cases: (i, image, clusters, angles) per image to check: i its index in the call, image = (pixels, rows, cols, dim),
    clusters the expected faces, angles the eye angle of each face (or one angle for all).  randoms(i, k, slot) is the
    randoms array of one RunDetector call; got = (faces, n_faces, points) of the library.  Asserts the faces byte for byte,
    every point of a refined face in (row, col, float32 scale), and zero points for every other face.  Returns the number of
    refined faces and of those refined at an angle > 0."""
    faces, nfaces, points = got
    refined = rotated = 0
    for i, image, clusters, angles in cases:
        angles = np.broadcast_to(np.asarray(angles, dtype=np.float64), len(clusters))
        assert int(nfaces[i]) == len(clusters), i
        assert faces[i, :len(clusters)].tobytes() == clusters.tobytes(), i
        want = oracle_points(oracle, image, clusters, angles, lambda k, slot: randoms(i, k, slot), eye)
        for k, f in enumerate(clusters):
            pts = points[i, k]
            if f["scale"] <= 50:
                assert not pts.tobytes().strip(b"\0"), (i, k)
                continue
            refined += 1
            rotated += angles[k] > 0
            for c, (p, e) in enumerate(zip(pts, want[k])):
                assert (int(p["row"]), int(p["col"]), np.float32(p["scale"])) == (e["row"], e["col"], e["scale"]), (i, k, c)
    return refined, rotated
