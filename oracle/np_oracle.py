"""numpy restatement of esimov/pigo's detection path -- ORACLE #2 (test infrastructure only).

Written independently of oracle/pigo_oracle.c (vectorised over windows instead of
window-at-a-time) so that the two restatements check each other; neither is the
product.  Follows:

  core/pigo.go:51-110   Unpack                -> FaceCascade.__init__
  core/pigo.go:113-147  classifyRegion        -> FaceCascade.classify(..., angle=0)
  core/pigo.go:150-191  classifyRotatedRegion -> FaceCascade.classify(..., angle>0)
  core/pigo.go:212-258  RunCascade            -> FaceCascade.run_cascade
  core/pigo.go:262-308  ClusterDetections     -> cluster_detections
  core/puploc.go:38-103 UnpackCascade         -> PuplocCascade.__init__
  core/puploc.go:106-217 classifyRegion/Rotated -> PuplocCascade.classify
  core/puploc.go:239-277 RunDetector          -> PuplocCascade.run_detector
  core/flploc.go:36-57  GetLandmarkPoint      -> landmark_seed
  core/grayscale.go:8-23 RgbToGrayscale       -> rgb_to_grayscale

"parity unpinned": see the header of pigo_oracle.c -- no Go toolchain, and the
reference's tests carry no numeric goldens.  Only tests/ and tools/ import this.
"""
from __future__ import annotations

import math

import numpy as np

QCOS = np.array([256, 251, 236, 212, 181, 142, 97, 49, 0, -49, -97, -142, -181, -212, -236, -251, -256,
                 -251, -236, -212, -181, -142, -97, -49, 0, 49, 97, 142, 181, 212, 236, 251, 256], dtype=np.int64)
QSIN = np.array([0, 49, 97, 142, 181, 212, 236, 251, 256, 251, 236, 212, 181, 142, 97, 49, 0,
                 -49, -97, -142, -181, -212, -236, -251, -256, -251, -236, -212, -181, -142, -97, -49, 0], dtype=np.int64)


def scale_ladder(min_size: int, max_size: int, scale_factor: float) -> list[int]:
    """core/pigo.go:226,:255 -- float64 arithmetic with truncation."""
    out, s = [], int(min_size)
    while s <= max_size:
        out.append(s)
        s = int(float(s) + max(2.0, float(s) * scale_factor - float(s)))
    return out


def grid(rows: int, cols: int, s: int, shift: float):
    """core/pigo.go:227-231: (row values, col values) for scale s."""
    step = int(max(shift * float(s), 1.0))
    off = s // 2 + 1
    return np.arange(off, rows - off + 1, step, dtype=np.int64), np.arange(off, cols - off + 1, step, dtype=np.int64)


def count_windows(rows, cols, min_size, max_size, shift, scale_factor) -> int:
    n = 0
    for s in scale_ladder(min_size, max_size, scale_factor):
        rr, cc = grid(rows, cols, s, shift)
        n += len(rr) * len(cc)
    return n


class FaceCascade:
    def __init__(self, packet: bytes):
        buf = np.frombuffer(packet, dtype=np.uint8)
        self.depth = int(np.frombuffer(packet, dtype="<u4", count=1, offset=8)[0])
        self.ntrees = int(np.frombuffer(packet, dtype="<u4", count=1, offset=12)[0])
        L = 1 << self.depth
        per = 4 * L - 4 + 4 * L + 4
        body = buf[16:16 + self.ntrees * per].reshape(self.ntrees, per)
        codes = np.zeros((self.ntrees, L, 4), dtype=np.int8)           # node idx (1-based heap) -> 4 codes
        codes.reshape(self.ntrees, 4 * L)[:, 4:] = body[:, :4 * L - 4].view(np.int8)
        self.codes = codes
        self.preds = body[:, 4 * L - 4:4 * L - 4 + 4 * L].copy().view("<f4").reshape(self.ntrees, L)
        self.thresh = body[:, -4:].copy().view("<f4").reshape(self.ntrees)
        self.leaves = L

    def classify(self, r, c, s: int, pixels: np.ndarray, rows: int, cols: int, dim: int, angle: float = 0.0,
                 return_ntrees: bool = False):
        """Vectorised classifyRegion / classifyRotatedRegion for window centres r[], c[] at one scale."""
        r = np.asarray(r, dtype=np.int64)
        c = np.asarray(c, dtype=np.int64)
        flat = np.ascontiguousarray(pixels).reshape(-1)
        n = r.shape[0]
        out = np.zeros(n, dtype=np.float32)
        result = np.full(n, -1.0, dtype=np.float32)
        ntre = np.zeros(n, dtype=np.int32)
        alive = np.arange(n)
        rotated = angle > 0.0
        if rotated:
            a = min(angle, 1.0)
            qsin = s * int(QSIN[int(32.0 * a)])
            qcos = s * int(QCOS[int(32.0 * a)])
        for t in range(self.ntrees):
            if alive.size == 0:
                break
            ra, ca = r[alive], c[alive]
            idx = np.ones(alive.size, dtype=np.int64)
            tc = self.codes[t].astype(np.int64)
            for _ in range(self.depth):
                cd = tc[idx]
                if not rotated:
                    x1 = ((ra * 256 + cd[:, 0] * s) >> 8) * dim + ((ca * 256 + cd[:, 1] * s) >> 8)
                    x2 = ((ra * 256 + cd[:, 2] * s) >> 8) * dim + ((ca * 256 + cd[:, 3] * s) >> 8)
                else:
                    lim = rows - 1  # pigo.go:168,:171 clamp BOTH coordinates with nrows-1
                    r1 = np.abs(np.minimum(lim, np.maximum(0, 65536 * ra + qcos * cd[:, 0] - qsin * cd[:, 1]) >> 16))
                    c1 = np.abs(np.minimum(lim, np.maximum(0, 65536 * ca + qsin * cd[:, 0] + qcos * cd[:, 1]) >> 16))
                    r2 = np.abs(np.minimum(lim, np.maximum(0, 65536 * ra + qcos * cd[:, 2] - qsin * cd[:, 3]) >> 16))
                    c2 = np.abs(np.minimum(lim, np.maximum(0, 65536 * ca + qsin * cd[:, 2] + qcos * cd[:, 3]) >> 16))
                    x1, x2 = r1 * dim + c1, r2 * dim + c2
                idx = 2 * idx + (flat[x1] <= flat[x2])
            out[alive] = out[alive] + self.preds[t][idx - self.leaves]   # float32 add, tree order
            ntre[alive] += 1
            keep = ~(out[alive] <= self.thresh[t])   # core/pigo.go:139-141: a NaN sum or threshold does not reject
            alive = alive[keep]
        if self.ntrees > 0:
            result[alive] = out[alive] - self.thresh[self.ntrees - 1]
        else:
            result[:] = 0.0
        return (result, ntre) if return_ntrees else result

    def run_cascade(self, pixels, rows, cols, dim, min_size, max_size, shift, scale_factor, angle=0.0,
                    return_stats: bool = False):
        """Returns an (n,4) float64 array of (row, col, scale, q) in the reference's emission order."""
        dets = []
        hist = np.zeros(self.ntrees + 1, dtype=np.int64)
        for s in scale_ladder(min_size, max_size, scale_factor):
            rr, cc = grid(rows, cols, s, shift)
            if len(rr) == 0 or len(cc) == 0:
                continue
            R, C = np.meshgrid(rr, cc, indexing="ij")
            q, ntre = self.classify(R.ravel(), C.ravel(), s, pixels, rows, cols, dim, angle, return_ntrees=True)
            hist += np.bincount(ntre, minlength=self.ntrees + 1)
            sel = np.nonzero(q > 0.0)[0]
            for i in sel:
                dets.append((int(R.ravel()[i]), int(C.ravel()[i]), s, np.float32(q[i])))
        return (dets, hist) if return_stats else dets


def q_sort_key(q):
    """The library's order of Q: ascending, -0 equal to +0 (float comparison), every NaN after +inf and equal to each
    other.  With a stable sort this is np.argsort(q, kind="stable")."""
    q = float(np.float32(q))
    return (1, 0.0) if q != q else (0, q)


def _trunc_div(a: int, k: int) -> int:
    """Go's integer division: truncates toward zero."""
    m = abs(a) // k
    return m if a >= 0 else -m


def cluster_detections(dets, iou_threshold: float):
    """core/pigo.go:262-308.  dets: list of (row, col, scale, q).  Stable sort by q_sort_key."""
    d = sorted(dets, key=lambda x: q_sort_key(x[3]))  # python's sort is stable
    n = len(d)
    assigned = [False] * n

    def iou(a, b):
        r1, c1, s1 = float(a[0]), float(a[1]), float(a[2])
        r2, c2, s2 = float(b[0]), float(b[1]), float(b[2])
        orow = max(0.0, min(r1 + s1 / 2, r2 + s2 / 2) - max(r1 - s1 / 2, r2 - s2 / 2))
        ocol = max(0.0, min(c1 + s1 / 2, c2 + s2 / 2) - max(c1 - s1 / 2, c2 - s2 / 2))
        den = s1 * s1 + s2 * s2 - orow * ocol
        # the denominator is 0 only for two zero scales, where the overlap is 0 too: IEEE 0/0 (Python would raise)
        return orow * ocol / den if den != 0.0 else float("nan")

    clusters = []
    with np.errstate(over="ignore", invalid="ignore"):   # float32 Q sums may overflow to inf, or meet inf - inf
        for i in range(n):
            if assigned[i]:
                continue
            r = c = s = k = 0
            q = np.float32(0.0)
            for j in range(n):
                if iou(d[i], d[j]) > iou_threshold:
                    assigned[j] = True
                    r += int(d[j][0]); c += int(d[j][1]); s += int(d[j][2])
                    q = np.float32(q + np.float32(d[j][3]))
                    k += 1
            if k > 0:
                clusters.append((_trunc_div(r, k), _trunc_div(c, k), _trunc_div(s, k), q))
    return d, clusters


class PuplocCascade:
    def __init__(self, packet: bytes):
        self.stages = int(np.frombuffer(packet, dtype="<u4", count=1, offset=0)[0])
        self.scales = np.frombuffer(packet, dtype="<f4", count=1, offset=4)[0]
        self.trees = int(np.frombuffer(packet, dtype="<u4", count=1, offset=8)[0])
        self.depth = int(np.frombuffer(packet, dtype="<u4", count=1, offset=12)[0])
        L = 1 << self.depth
        per = 4 * L - 4 + 8 * L
        nt = self.stages * self.trees
        body = np.frombuffer(packet, dtype=np.uint8, count=nt * per, offset=16).reshape(nt, per)
        self.codes = body[:, :4 * L - 4].copy().view(np.int8).reshape(nt, L - 1, 4)   # node idx 0-based heap
        self.preds = body[:, 4 * L - 4:].copy().view("<f4").reshape(nt, L, 2)
        self.leaves = L

    def classify(self, r, c, s, pixels, rows, cols, dim, angle=0.0, flipv=False):
        """One perturbation; r, c, s are float32 scalars.  Returns float32 (r, c, s)."""
        f32 = np.float32
        r, c, s = f32(r), f32(c), f32(s)
        flat = np.ascontiguousarray(pixels).reshape(-1)
        rotated = angle > 0.0
        if rotated:
            a = min(angle, 1.0)
            qsin = int(f32(s * f32(QSIN[int(32.0 * a)])))   # int(qsin) truncation, puploc.go:188
            qcos = int(f32(s * f32(QCOS[int(32.0 * a)])))
        L = self.leaves
        for i in range(self.stages):
            dr, dc = f32(0), f32(0)
            for j in range(self.trees):
                t = i * self.trees + j
                idx = 0
                for _ in range(self.depth):
                    cd = [int(v) for v in self.codes[t, idx]]
                    if flipv:   # int8 negation wraps: -(-128) == -128
                        cd[1] = int(np.int8(np.uint8((-cd[1]) & 0xFF)))
                        cd[3] = int(np.int8(np.uint8((-cd[3]) & 0xFF)))
                    ir, ic = _go_int(r), _go_int(c)
                    if not rotated:
                        rs = int(_go_round(float(s)))
                        r1 = min(rows - 1, max(0, (256 * ir + cd[0] * rs) >> 8))
                        r2 = min(rows - 1, max(0, (256 * ir + cd[2] * rs) >> 8))
                        c1 = min(cols - 1, max(0, (256 * ic + cd[1] * rs) >> 8))
                        c2 = min(cols - 1, max(0, (256 * ic + cd[3] * rs) >> 8))
                        bit = 1 if flat[r1 * dim + c1] > flat[r2 * dim + c2] else 0
                    else:
                        r1 = min(rows - 1, max(0, 65536 * ir + qcos * cd[0] - qsin * cd[1]) >> 16)
                        c1 = min(cols - 1, max(0, 65536 * ic + qsin * cd[0] + qcos * cd[1]) >> 16)
                        r2 = min(rows - 1, max(0, 65536 * ir + qcos * cd[2] - qsin * cd[3]) >> 16)
                        c2 = min(cols - 1, max(0, 65536 * ic + qsin * cd[2] + qcos * cd[3]) >> 16)
                        bit = 1 if flat[r1 * dim + c1] <= flat[r2 * dim + c2] else 0
                    idx = 2 * idx + 1 + bit
                leaf = idx - (L - 1)
                dr = f32(dr + self.preds[t, leaf, 0])
                dc = f32(dc + (-self.preds[t, leaf, 1] if flipv else self.preds[t, leaf, 1]))
            r = f32(r + f32(dr * s))
            c = f32(c + f32(dc * s))
            s = f32(s * self.scales)
        return r, c, s

    def run_detector(self, row, col, scale, perturbs, randoms, pixels, rows, cols, dim, angle=0.0, flipv=False):
        f32 = np.float32
        assert 0 <= perturbs <= 63
        pr, pc, ps = np.zeros(63, f32), np.zeros(63, f32), np.zeros(63, f32)
        rnd = np.asarray(randoms, dtype=f32).reshape(-1, 3)
        for i in range(perturbs):
            t1 = f32(f32(scale) * f32(0.15))
            rowf = f32(f32(row) + f32(t1 * f32(f32(0.5) - rnd[i, 0])))
            colf = f32(f32(col) + f32(t1 * f32(f32(0.5) - rnd[i, 1])))
            sc = f32(f32(scale) * f32(f32(0.925) + f32(f32(0.15) * rnd[i, 2])))
            pr[i], pc[i], ps[i] = self.classify(rowf, colf, sc, pixels, rows, cols, dim, angle, flipv)
        mid = int(_go_round(perturbs / 2))
        return _to_i32(_pool_median(pr, mid)), _to_i32(_pool_median(pc, mid)), _pool_median(ps, mid)


def _go_int(v) -> int:
    """int(r) as the sample arithmetic sees it: truncation toward zero; Go on amd64 gives the int64 minimum for NaN and
    out-of-range values, and 256 * (or 65536 *) that minimum wraps to 0."""
    return int(v) if abs(float(v)) < 2.0 ** 63 else 0


def _pool_median(pool, mid):
    """Entry `mid` of the 63-slot pool in RunDetector's order (core/puploc.go:267-269): numbers ascending (-0 == +0), every
    NaN above every number, ties by slot -- the total order the library picks where Go's order with NaNs is an accident."""
    order = sorted(range(63), key=lambda k: (bool(np.isnan(pool[k])), 0.0 if np.isnan(pool[k]) else float(pool[k]), k))
    return pool[order[mid]]


def _to_i32(v) -> int:
    """int() into the 32-bit Row / Col field: truncation, saturated at the int32 range, NaN -> 0."""
    if np.isnan(v):
        return 0
    return int(min(max(float(v), -2.0 ** 31), 2.0 ** 31 - 1))


def _go_round(x: float) -> float:
    """core/utils.go:33-39 / math.Round: half away from zero."""
    t = math.trunc(x)
    if abs(x - t) >= 0.5:
        return t + math.copysign(1.0, x)
    return float(t)


def landmark_seed(lrow, lcol, rrow, rcol):
    """core/flploc.go:37-50."""
    dist = math.sqrt(float((lrow - rrow) ** 2 + (lcol - rcol) ** 2))
    row = float(lrow + rrow) / 2.0 + 0.25 * dist
    col = float(lcol + rcol) / 2.0 + 0.15 * dist
    return int(row), int(col), np.float32(3.0 * dist)


def rgb_to_grayscale(rgb: np.ndarray) -> np.ndarray:
    """core/grayscale.go:8-23 for an opaque image: 8-bit channels expand to v*0x101 (RGBA())."""
    v = rgb.astype(np.float64) * 257.0
    g = (0.299 * v[..., 0] + 0.587 * v[..., 1] + 0.114 * v[..., 2]) / 256
    return g.astype(np.uint8)
