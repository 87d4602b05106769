"""Synthetic depth-6 face cascades for the tests of the face scan's deep queue (tests/test_scan_cases_cpu.py,
tests/test_scan_overflow_gpu.py), and a restatement of the queue's sizing and hand-over points.

Cascade families (facefinder binary layout, core/pigo.go:51-110):
  * survivor S(n, k): random leaves that are not dyadic (summation order matters); the first n - k trees have threshold
    -inf, so every window walks them; the last k trees have thresholds calibrated on noise so that about 3 % of the windows
    are detected.  A call then hands every window over to the deep queue, far more than it holds.
  * flat-prefix F(n): in each of the first n - 1 trees all 64 leaves are equal and the threshold is -inf, so every window
    reaches the last tree with the same float32 partial sum C (formed in tree order); the last tree detects about one window
    in eight.  F(n) gives exactly the output of its two-tree collapsed cascade (tree 0: every leaf C, threshold -inf; tree 1:
    F's last tree), which the oracle walks 2 trees per window instead of n.
  * ties: leaves in {+-0.5, +-0.25, 0} and thresholds on the same lattice, so that acc == thr (a rejection) happens at trees
    in every range and q == 0 (no detection) at the last tree.
  * special values: NaN / +-inf leaves and thresholds and -0.0 leaves at chosen trees.
"""
import os

import numpy as np

DEPTH = 6
LEAVES = 1 << DEPTH
NODE_BYTES = 4 * LEAVES - 4
HEADER = b"\x03\x00\x00\x00\x81\x7f\x81\x7f"

# ---- restated constants (checked against the sources by tests/test_scan_cases_cpu.py) --------------------------------------
TILE_KS = 48            # host.h tile_ks: cascade trees resident in the fused kernel's shared memory
GATHER_KS = 32          # host.h gather_ks: resident trees of the gather-v2 kernel
QUEUE_MAX = 1 << 26     # cap on the deep queue's items per pipeline group
SMALL_CALL = 4_000_000  # windows: a "small call" (8-window gather blocks, 32 deep lanes, per-item deep order)
MID_CALL = 40_000_000   # windows: unrotated calls up to this size hand over after 8 trees
IMAGES_GROUP_WINDOWS = 128 * 894448


def run_scan_queue_cap(group_windows: int) -> int:
    """Q2 items of one pipeline group of a uniform batch (run_scan, classic tile role)."""
    return min(group_windows // 16 + group_windows // 32 + 65536, QUEUE_MAX)


def images_queue_cap(group_windows: int) -> int:
    """Q2 items of one group of a mixed-size call (run_scan_images)."""
    return min(group_windows // 32 + 65536, QUEUE_MAX)


def schedule(call_windows: int, rot: bool, large_limit: int) -> dict:
    """images_schedule at default options: gather_limit (trees a gather-role window walks before it is handed over),
    deep_group (lanes per deep window) and deep_ordered (the deep queue is sorted into image order).  large_limit: 16 for
    run_scan, 24 for the mixed-size scan."""
    small = call_windows <= SMALL_CALL
    glimit = (8 if small else 24) if rot else (8 if call_windows <= MID_CALL else large_limit)
    return {"gather_limit": glimit, "deep_group": 32 if small else 8, "deep_ordered": call_windows > SMALL_CALL}


def gather_v2_handover(ntrees: int, gather_limit: int) -> int:
    """Trees a gather-v2 window walks before its hand-over (its resident prefix); ntrees or more: no hand-over."""
    return min(GATHER_KS, gather_limit, ntrees)


def predict_queue(hist, handover: int, cap: int) -> dict:
    """From the oracle's tree histogram (hist[k]: windows that walked exactly k trees) of the windows of one queue: how many
    windows outlive `handover` trees (each of them is offered to the queue), whether they overflow a queue of `cap` items,
    and a lower bound on the hand-over attempts a gather role makes when a refused window asks again after every later tree
    (what it did before it stopped after its warp's first refusal): the `cap` windows that get in ask once (the bound puts
    the longest-lived ones there), every other window asks after each of its trees handover .. min(k, n - 1)."""
    hist = np.asarray(hist, dtype=np.int64)
    n = len(hist) - 1
    if handover >= n:
        return {"survivors": 0, "overflow": False, "attempts": 0}
    k = np.arange(n + 1)
    per = np.where(k > handover, k - handover, 0).astype(np.int64)   # attempts of a refused window that walked k trees
    survivors = int(hist[handover + 1:].sum())
    queued = min(cap, survivors)
    left, attempts = queued, queued
    for kk in range(n, handover, -1):   # the queued ones: the longest-lived first (lower bound)
        take = min(left, int(hist[kk]))
        left -= take
        attempts += (int(hist[kk]) - take) * int(per[kk])
    return {"survivors": survivors, "overflow": survivors > cap, "attempts": attempts}


# ---- cascade construction -----------------------------------------------------------------------------------------------
def pack(codes, leaves, thresh) -> bytes:
    """codes [n, 252] int8, leaves [n, 64] float32, thresh [n] float32 -> cascade bytes."""
    codes = np.asarray(codes, dtype=np.int8)
    leaves = np.asarray(leaves, dtype="<f4")
    thresh = np.asarray(thresh, dtype="<f4")
    n = len(thresh)
    out = bytearray(HEADER) + np.uint32(DEPTH).tobytes() + np.uint32(n).tobytes()
    for t in range(n):
        out += codes[t].tobytes() + leaves[t].tobytes() + thresh[t].tobytes()
    return bytes(out)


def unpack(pk: bytes):
    n = int(np.frombuffer(pk, dtype="<u4", count=1, offset=12)[0])
    body = np.frombuffer(pk, dtype=np.uint8, offset=16).reshape(n, NODE_BYTES + 4 * LEAVES + 4)
    codes = body[:, :NODE_BYTES].view(np.int8).copy()
    leaves = body[:, NODE_BYTES:NODE_BYTES + 4 * LEAVES].copy().view("<f4")
    thresh = body[:, -4:].copy().view("<f4").reshape(n)
    return codes, leaves, thresh


def random_codes(rng, n):
    return rng.integers(-128, 128, size=(n, NODE_BYTES), dtype=np.int8)


def noise_frame(rows, cols, seed):
    return np.random.default_rng(seed).integers(0, 256, size=(rows, cols), dtype=np.uint8)


def _calibration_windows():
    """A sample of unrotated windows (centre row, col, size) on a 256 x 256 noise frame, for threshold calibration."""
    frame = noise_frame(256, 256, 4242)
    rng = np.random.default_rng(4243)
    s = rng.integers(20, 120, size=3000)
    r = rng.integers(s // 2 + 1, 256 - s // 2 - 1)
    c = rng.integers(s // 2 + 1, 256 - s // 2 - 1)
    return frame, r.astype(np.int64), c.astype(np.int64), s.astype(np.int64)


def leaf_values(codes, leaves, t, frame, r, c, s):
    """Leaf value of tree t for every window (classifyRegion's walk, core/pigo.go:121-137)."""
    dim = frame.shape[1]
    flat = frame.reshape(-1)
    cd = codes[t].astype(np.int64).reshape(-1, 4)   # node i (1-based heap) at row i - 1
    idx = np.ones(len(r), dtype=np.int64)
    for _ in range(DEPTH):
        q = cd[idx - 1]
        x1 = ((r * 256 + q[:, 0] * s) >> 8) * dim + ((c * 256 + q[:, 1] * s) >> 8)
        x2 = ((r * 256 + q[:, 2] * s) >> 8) * dim + ((c * 256 + q[:, 3] * s) >> 8)
        idx = 2 * idx + (flat[x1] <= flat[x2])
    return leaves[t][idx - LEAVES]


def _calibrate(codes, leaves, first, pass_rate, lattice=None):
    """Thresholds: -inf for trees < first; for the later trees the quantile of the calibration windows' partial sums that
    keeps `pass_rate` of those still alive (given a `lattice`: rounded down onto it, then one step lower, so that a lattice
    point that holds many windows does not reject them all)."""
    n = len(leaves)
    thresh = np.full(n, -np.inf, dtype=np.float32)
    frame, r, c, s = _calibration_windows()
    acc = np.zeros(len(r), dtype=np.float32)
    alive = np.ones(len(r), dtype=bool)
    for t in range(n):
        acc = (acc + leaf_values(codes, leaves, t, frame, r, c, s)).astype(np.float32)
        if t >= first and alive.any():
            thr = np.quantile(acc[alive].astype(np.float64), 1.0 - pass_rate)
            thr = (np.floor(thr / lattice) - 1) * lattice if lattice else thr
            thresh[t] = np.float32(thr)
            alive &= acc > thresh[t]
    return thresh


def survivor_cascade(n: int, k: int, seed: int, detect=0.03) -> bytes:
    """S(n, k): every window walks the first n - k trees; about `detect` of them are detected after the last k."""
    rng = np.random.default_rng(seed)
    codes = random_codes(rng, n)
    leaves = rng.uniform(-1.0, 1.0, size=(n, LEAVES)).astype(np.float32)
    return pack(codes, leaves, _calibrate(codes, leaves, n - k, detect ** (1.0 / k)))


def flat_prefix_cascade(n: int, seed: int):
    """(F(n), its collapsed two-tree cascade, C)."""
    rng = np.random.default_rng(seed)
    codes = random_codes(rng, n)
    v = rng.uniform(-0.05, 0.05, size=n - 1).astype(np.float32)
    leaves = np.empty((n, LEAVES), dtype=np.float32)
    leaves[:n - 1] = v[:, None]
    leaves[n - 1] = rng.uniform(-1.0, 1.0, size=LEAVES).astype(np.float32)
    C = np.float32(0.0)
    for x in v:                          # the kernels' and the oracle's float32 sum, in tree order
        C = np.float32(C + x)
    assert C != 0 and np.isfinite(C)     # (C = -0 would not survive 0 + C in the collapsed cascade)
    thresh = np.full(n, -np.inf, dtype=np.float32)
    frame, r, c, s = _calibration_windows()
    last = (C + leaf_values(codes, leaves, n - 1, frame, r, c, s)).astype(np.float32)
    thresh[n - 1] = np.float32(np.quantile(last.astype(np.float64), 7.0 / 8.0))
    full = pack(codes, leaves, thresh)
    collapsed = pack(np.stack([codes[0], codes[n - 1]]), np.stack([np.full(LEAVES, C, dtype=np.float32), leaves[n - 1]]),
                     np.array([-np.inf, thresh[n - 1]], dtype=np.float32))
    return full, collapsed, C


def tie_cascade(n: int, seed: int) -> bytes:
    """Leaves from {+-0.5, +-0.25, 0}, thresholds on the 0.25 lattice: each tree rejects about 1.5 % of the windows still
    alive (many of them at acc == thr), and the last tree's lattice threshold gives q == 0 to many windows."""
    rng = np.random.default_rng(seed)
    codes = random_codes(rng, n)
    leaves = rng.choice(np.array([-0.5, -0.25, 0.0, 0.25, 0.5], dtype=np.float32), size=(n, LEAVES))
    thresh = _calibrate(codes, leaves, 0, 0.985, lattice=0.25)
    thresh[n - 1] = _calibrate(codes, leaves, n - 1, 0.2, lattice=0.25)[n - 1]
    return pack(codes, leaves, thresh)


def special_cascade(n: int, seed: int, at: dict) -> bytes:
    """S(n, 4) with special values: at = {tree: kind}, kinds "nan_leaf", "pinf_leaf", "ninf_leaf", "negzero_leaves"
    (on some leaves of the tree), "nan_thr", "pinf_thr", "ninf_thr" (the tree's threshold)."""
    pk = survivor_cascade(n, 4, seed)
    codes, leaves, thresh = unpack(pk)
    rng = np.random.default_rng(seed + 1)
    for t, kind in at.items():
        some = rng.choice(LEAVES, size=5, replace=False)
        if kind == "nan_leaf":
            leaves[t, some[:2]] = np.nan
        elif kind == "pinf_leaf":
            leaves[t, some[:2]] = np.inf
        elif kind == "ninf_leaf":
            leaves[t, some[:2]] = -np.inf
        elif kind == "negzero_leaves":
            leaves[t, some] = -0.0
        elif kind == "nan_thr":
            thresh[t] = np.nan
        elif kind == "pinf_thr":
            thresh[t] = np.inf
        elif kind == "ninf_thr":
            thresh[t] = -np.inf
        else:
            raise ValueError(kind)
    return pack(codes, leaves, thresh)


# Special-value placements: tree 0, around the fused kernel's resident prefix (KS = 48), at the gather hand-overs (8, 16, 24),
# inside the deep range and at the last tree of a 100-tree cascade.
SPECIALS = {
    "leaves": {0: "negzero_leaves", 7: "nan_leaf", 8: "pinf_leaf", 16: "ninf_leaf", 24: "nan_leaf", 47: "pinf_leaf",
               48: "negzero_leaves", 49: "ninf_leaf", 70: "nan_leaf", 99: "pinf_leaf"},
    # a NaN threshold rejects nothing (acc <= NaN is false), also at the first calibrated tree (96)
    "thresholds": {0: "nan_thr", 8: "nan_thr", 16: "ninf_thr", 24: "nan_thr", 47: "nan_thr", 48: "ninf_thr", 49: "nan_thr",
                   70: "nan_thr", 80: "negzero_leaves", 96: "nan_thr"},
    # +inf sums (q = +inf detections), +inf + -inf = NaN (walks to the end, never detected), NaN sums from tree 30 on
    "inf_q": {3: "pinf_leaf", 30: "nan_leaf", 61: "pinf_leaf", 62: "ninf_leaf", 98: "pinf_leaf", 99: "negzero_leaves"},
    # a +inf threshold rejects every window but the NaN ones (tree 10), which are never detected
    "pinf_thr": {10: "nan_leaf", 52: "pinf_thr"},
}


def sources_text(name: str) -> str:
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "pigo_b200", "csrc", name)) as f:
        return f.read()
