"""CPU restatement of an angle sweep merged per image (pigo_run_cascade_images_sweep), on the C oracle.

For one image and a host list of angles: D = RunCascade at angles[0] ++ ... ++ RunCascade at angles[-1] (each list in
emission order), the clusters are ClusterDetections(D, iou) with a stable sort by Q (oracle_lib.cluster), and each
cluster's angle index is the tag of its member with the largest Q, the earliest in D among equal Q.  Also the numpy
rotation the sweep tests tilt the sample with (scipy.ndimage.rotate(order=1, reshape=False, mode="nearest") restated).
"""
from __future__ import annotations

import numpy as np

import oracle_lib as O
from pigo_b200 import synth


def sweep_angles(n: int = 32):
    return [k / n for k in range(n)]


def expected_slot(tilt_deg: float, n: int = 32) -> int:
    return int(round(n * tilt_deg / 360.0)) % n


def padded_sample() -> np.ndarray:
    """The 400x320 sample edge-padded to 520x520, so that a rotation keeps the face inside the frame."""
    return np.pad(synth.sample_gray(), ((60, 60), (100, 100)), mode="edge")


def rotate(img: np.ndarray, deg: float) -> np.ndarray:
    """scipy.ndimage.rotate(img, deg, order=1, reshape=False, mode="nearest") in numpy: output pixel o reads the input at
    R @ (o - centre) + centre, R = [[cos, sin], [-sin, cos]], bilinear, coordinates clamped to the border, rounded to uint8."""
    rows, cols = img.shape
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    cr, cc = (rows - 1) / 2.0, (cols - 1) / 2.0
    orow, ocol = np.meshgrid(np.arange(rows, dtype=np.float64), np.arange(cols, dtype=np.float64), indexing="ij")
    ir = np.clip(c * (orow - cr) + s * (ocol - cc) + cr, 0, rows - 1)
    ic = np.clip(-s * (orow - cr) + c * (ocol - cc) + cc, 0, cols - 1)
    r0, c0 = np.floor(ir).astype(np.int64), np.floor(ic).astype(np.int64)
    r1, c1 = np.minimum(r0 + 1, rows - 1), np.minimum(c0 + 1, cols - 1)
    fr, fc = ir - r0, ic - c0
    f = img.astype(np.float64)
    v = (f[r0, c0] * (1 - fr) * (1 - fc) + f[r0, c1] * (1 - fr) * fc + f[r1, c0] * fr * (1 - fc) + f[r1, c1] * fr * fc)
    return np.clip(np.floor(v + 0.5), 0, 255).astype(np.uint8)


def _iou(d: np.ndarray, i: int) -> np.ndarray:
    """IoU of detection i with every detection of d, float64 in the reference's operation order (core/pigo.go:268-278)."""
    r, c, s = d["row"].astype(np.float64), d["col"].astype(np.float64), d["scale"].astype(np.float64)
    r1, c1, s1 = r[i], c[i], s[i]
    over_r = np.maximum(0.0, np.minimum(r1 + s1 / 2, r + s / 2) - np.maximum(r1 - s1 / 2, r - s / 2))
    over_c = np.maximum(0.0, np.minimum(c1 + s1 / 2, c + s / 2) - np.maximum(c1 - s1 / 2, c - s / 2))
    return (over_r * over_c) / ((s1 * s1 + s * s) - over_r * over_c)


def merge(parts, iou: float, cluster=O.cluster):
    """parts[a] = angle a's detections (DET_DTYPE).  Returns (clusters, angle_index) of their concatenation D, the clusters
    from cluster(D, iou) -> (sorted D, clusters): the C oracle's, or the library's (Pigo.cluster_array)."""
    D = np.concatenate([np.asarray(p, dtype=O.DET_DTYPE) for p in parts]) if parts else np.zeros(0, O.DET_DTYPE)
    tags = np.concatenate([np.full(len(p), a, dtype=np.int32) for a, p in enumerate(parts)]) if parts else np.zeros(0, np.int32)
    _, clusters = cluster(D.copy(), iou)   # (the library's clustering sorts its argument in place)
    order = np.argsort(D["q"], kind="stable")
    d, t = D[order], tags[order]
    n = len(d)
    assigned = np.zeros(n, dtype=bool)
    index = []
    for i in range(n):                       # core/pigo.go:282-301
        if assigned[i]:
            continue
        members = _iou(d, i) > iou
        assigned |= members
        q = d["q"][members]
        first_max = np.flatnonzero(members)[np.flatnonzero(q == q.max())[0]]
        index.append(int(t[first_max]))
    assert len(index) == len(clusters), (len(index), len(clusters))
    return clusters, np.array(index, dtype=np.int32)


def sweep_oracle(face: O.OracleFace, image, angles, params, iou: float):
    """image = (pixels, rows, cols, dim); params = (min_size, max_size, shift, scale).  Returns (clusters, angle_index)."""
    px, rows, cols, dim = image
    return merge([face.run_cascade(px, rows, cols, dim, *params, a) for a in angles], iou)


def strongest_slot(clusters: np.ndarray, index: np.ndarray, angles) -> int:
    k = int(np.argmax(clusters["q"]))
    return int(round(angles[index[k]] * len(angles))) % len(angles)


def slot_distance(a: int, b: int, n: int = 32) -> int:
    d = abs(a - b) % n
    return min(d, n - d)
