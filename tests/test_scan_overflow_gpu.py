"""The depth-6 face scan against the C oracle on synthetic cascades (tests/scan_cases.py) whose windows overflow the deep
queue Q2 by themselves, at the call sizes where the schedule switches: per-warp tiles and per-item deep order (one 1080p
frame), the region role (3 frames), the ordered deep queue (6 frames), scan_mode=3, rotated uniform batches, the mixed-size
entry points, and forced deep lane groups.  Every window of a survivor or flat-prefix cascade outlives the hand-over point,
so the queue refuses most of them and they finish in place: in the tile roles' overflow mode, or in the gather role's walk
on the global tables.  Each case checks that the launches are the kernels it names, that the predictor
(scan_cases.predict_queue, from the oracle's tree histogram) says Q2 overflowed, and every output byte against the oracle.

The counter-wrap cases run F(4096) on two 1080p images, where a gather role that asked the queue again after every tree
would make more than 2^32 hand-over attempts and wrap the u32 queue count onto queued items."""
import concurrent.futures as cf
import ctypes as C
import os

import numpy as np
import pytest

import oracle_lib as O
import pigo_b200
import scan_cases as SC
from option_guard import options, options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)
from pigo_b200 import CascadeParams, ImageParams

pytestmark = pytest.mark.gpu

PRM = (20, 1000, 0.2, 1.1)
R, Cc = 1080, 1920
R2, C2 = 720, 1280
ANGLE = 0.25
NTHREADS = max(1, os.cpu_count() or 1)
WA = O.count_windows(R, Cc, *PRM)
WB = O.count_windows(R2, C2, *PRM)

# survivor cascades S(n, k): every remainder of n mod 8 past the resident prefix of 48 trees, and the hand-overs at 8, 24, 48
S_TREES = [1, 8, 9, 24, 25, 47, 48, 49] + list(range(50, 57)) + [100, 468]


def _k(n):
    return min(n, 1 + n % 4)


CASCADES = {f"S({n},{_k(n)})": (lambda n=n: SC.survivor_cascade(n, _k(n), 500 + n)) for n in S_TREES}
CASCADES.update({"ties(60)": lambda: SC.tie_cascade(60, 61), "ties(200)": lambda: SC.tie_cascade(200, 62)})
CASCADES.update({f"special-{k}": (lambda k=k: SC.special_cascade(100, 70 + i, SC.SPECIALS[k])) for i, k in enumerate(SC.SPECIALS)})


@pytest.fixture(scope="module")
def frames():
    return {"a": SC.noise_frame(R, Cc, 1), "b": SC.noise_frame(R2, C2, 2)}


@pytest.fixture(scope="module")
def expected(frames):
    """The oracle's detections and tree histogram of every cascade on frame a (unrotated and at ANGLE) and b (unrotated):
    computed once per distinct frame, in parallel (the C oracle releases the GIL)."""
    packs = {name: make() for name, make in CASCADES.items()}
    jobs = [(name, key, ang) for name in packs for key, ang in (("a", 0.0), ("a", ANGLE), ("b", 0.0))]
    jobs.sort(key=lambda j: -SC.unpack(packs[j[0]])[2].shape[0])

    def one(job):
        name, key, ang = job
        f = frames[key]
        return job, O.OracleFace(packs[name]).run_cascade(f, f.shape[0], f.shape[1], f.shape[1], *PRM, ang, with_hist=True)

    with cf.ThreadPoolExecutor(NTHREADS) as ex:
        res = dict(ex.map(one, jobs))
    return packs, {(n, k, a): v for (n, k, a), v in res.items()}


def timed(fn):
    with options(timing=1):
        out = fn()
        launches = {k: pigo_b200.get_option(k) for k in ("t_tiled_n", "t_region_n", "t_gather_n", "t_deep_n")}
    return out, launches


def batch(clf, frame, nf, angle, cap=1024):
    """pigo_run_cascade_batch of nf copies of `frame` (host), outputs prefilled with 0xa5: (rc, dets[nf, cap], counts)."""
    frs = np.ascontiguousarray(np.broadcast_to(frame, (nf,) + frame.shape))
    out = np.full(nf * cap * 16, 0xa5, dtype=np.uint8).view(pigo_b200.DET_DTYPE).reshape(nf, cap)
    cnt = np.full(nf, -7, dtype=np.int32)
    rows, cols = frame.shape
    rc = pigo_b200.lib().pigo_run_cascade_batch(clf._h, C.c_void_p(frs.ctypes.data), nf, rows * cols, rows, cols, cols, *PRM, angle,
                                                out.ctypes.data, cap, cnt.ctypes.data, pigo_b200.MEM_HOST, None)
    return rc, out, cnt


def assert_slices(out, cnt, want, what, prefilled=True):
    """Every slice equals the oracle byte for byte; slots past a slice's count up to the largest count are zero, those past
    the largest count are the caller's (0xa5) when the output was prefilled."""
    copied = min(int(cnt.max(initial=0)), out.shape[1])
    for i, w in enumerate(want):
        assert cnt[i] == len(w), f"{what}: slice {i}: {cnt[i]} detections vs oracle {len(w)}"
        assert out[i, :cnt[i]].tobytes() == w.tobytes(), f"{what}: slice {i}"
        assert not out[i, cnt[i]:copied].tobytes().strip(b"\0"), f"{what}: slice {i}: padding past the count is not zero"
        if prefilled:
            assert not out[i, copied:].tobytes().strip(b"\xa5"), f"{what}: slice {i}: slots past the largest count were written"


def run_batch_checked(clf, frame, nf, angle, want, what):
    rc, out, cnt = batch(clf, frame, nf, angle)
    if rc == pigo_b200.PIGO_E_CAP:
        assert list(cnt) == [len(want)] * nf, what
        rc, out, cnt = batch(clf, frame, nf, angle, int(cnt.max()))
    assert rc == 0, f"{what}: {pigo_b200.lib().pigo_last_error().decode()}"
    assert_slices(out, cnt, [want] * nf, what)


def names(launches):
    """The kernels a call ran: "region" / "tiles" (fused kernel and its tile role), "gather" (gather-v2), "deep"."""
    k = []
    if launches["t_tiled_n"]:
        k.append("region" if launches["t_region_n"] == launches["t_tiled_n"] else "tiles")
    if launches["t_gather_n"]:
        k.append("gather")
    if launches["t_deep_n"]:
        k.append("deep")
    return " ".join(k)


# Paths: (name, options, kernels, call).  call(clf, frames, want) runs the call and checks it against `want`, and returns
# (the oracle result whose histogram its windows follow, the queue cap as a function of the windows of a group, and the
# hand-over point of an n-tree cascade on that path).
def _uniform(nf, angle):
    def call(clf, fr, want, ntrees):
        key = ("a", angle)
        run_batch_checked(clf, fr["a"], nf, angle, want[key], f"{nf} x 1080p angle {angle}")
        w = nf * WA
        sch = SC.schedule(w, angle > 0, 16)
        h = SC.gather_v2_handover(ntrees, sch["gather_limit"]) if angle > 0 else min(SC.TILE_KS, ntrees)
        return key, SC.run_scan_queue_cap, h
    return call


def _mode3(clf, fr, want, ntrees):
    run_batch_checked(clf, fr["a"], 1, 0.0, want[("a", 0.0)], "scan_mode 3")
    return ("a", 0.0), SC.run_scan_queue_cap, SC.gather_v2_handover(ntrees, 8)


def _images(order):
    def call(clf, fr, want, ntrees):
        ims = [ImageParams(fr[k], *fr[k].shape, fr[k].shape[1]) for k in order]
        dets, cnt = clf.RunCascadeImages(ims, CascadeParams(ims[0], *PRM), 0.0)
        assert_slices(dets, cnt, [want[(k, 0.0)] for k in order], f"images {order}", prefilled=False)
        w = sum(WA if k == "a" else WB for k in order)
        sch = SC.schedule(w, False, 24)
        return ("a", 0.0), SC.images_queue_cap, SC.gather_v2_handover(ntrees, sch["gather_limit"])
    return call


def _angles(clf, fr, want, ntrees):
    keys = [("a", ANGLE), ("b", 0.0), ("a", 0.0)]
    ims = [ImageParams(fr[k], *fr[k].shape, fr[k].shape[1]) for k, _ in keys]
    dets, cnt = clf.RunCascadeImagesAngles(ims, CascadeParams(ims[0], *PRM), [a for _, a in keys])
    assert_slices(dets, cnt, [want[k] for k in keys], "images angles", prefilled=False)
    return ("a", ANGLE), SC.images_queue_cap, SC.gather_v2_handover(ntrees, 8)


def _params(clf, fr, want, ntrees):
    keys = [("b", 0.0), ("a", ANGLE), ("a", 0.0)]
    cps = [CascadeParams(ImageParams(fr[k], *fr[k].shape, fr[k].shape[1]), *PRM) for k, _ in keys]
    dets, cnt = clf.RunCascadeImagesParams(cps, [a for _, a in keys])
    assert_slices(dets, cnt, [want[k] for k in keys], "images params", prefilled=False)
    return ("a", ANGLE), SC.images_queue_cap, SC.gather_v2_handover(ntrees, 8)


MIXED_ORDERED = ["a", "b", "a", "b", "a", "a"]   # 4.4 M windows: the ordered deep queue on the mixed-size path
PATHS = [
    ("1x1080p", {}, "tiles deep", _uniform(1, 0.0)),
    ("3x1080p", {}, "region deep", _uniform(3, 0.0)),
    ("6x1080p", {}, "region deep", _uniform(6, 0.0)),
    ("scan_mode3", {"scan_mode": 3}, "gather deep", _mode3),
    ("rot1", {}, "gather deep", _uniform(1, ANGLE)),
    ("rot6", {}, "gather deep", _uniform(6, ANGLE)),
    ("images", {}, "gather deep", _images(["a", "b", "a"])),
    ("images-angles", {}, "gather deep", _angles),
    ("images-params", {}, "gather deep", _params),
] + [(f"6x1080p-deep{g}", {"deep_group": g}, "region deep", _uniform(6, 0.0)) for g in (8, 16, 32)] \
  + [(f"images-ordered-deep{g}", {"deep_group": g}, "gather deep", _images(MIXED_ORDERED)) for g in (8, 16, 32)]


def test_restated_schedule_covers_the_switches():
    """The call sizes above reach both deep orders, both gather hand-overs of the rotated scan and both tile roles."""
    assert not SC.schedule(WA, False, 16)["deep_ordered"] and SC.schedule(6 * WA, False, 16)["deep_ordered"]
    assert SC.schedule(4 * WA + 2 * WB, False, 24)["deep_ordered"] and not SC.schedule(2 * WA + WB, False, 24)["deep_ordered"]
    assert SC.schedule(WA, True, 16)["gather_limit"] == 8 and SC.schedule(6 * WA, True, 16)["gather_limit"] == 24
    plans = [pigo_b200.describe_plan(R, Cc, *PRM, nframes=n)["region"] for n in (1, 3, 6)]
    assert plans == [0, 1, 1]


@pytest.mark.parametrize("cascade", list(CASCADES))
def test_scan_paths_against_oracle(expected, frames, cascade):
    packs, res = expected
    pk = packs[cascade]
    ntrees = SC.unpack(pk)[2].shape[0]
    clf = pigo_b200.NewPigo().Unpack(pk)
    want = {(k, a): res[(cascade, k, a)][0] for k, a in (("a", 0.0), ("a", ANGLE), ("b", 0.0))}
    overflowed = 0
    for name, opts, kernels, call in PATHS:
        with options(**opts):
            (key, cap, h), launches = timed(lambda: call(clf, frames, want, ntrees))
        assert names(launches) == kernels, f"{cascade} {name}: ran {launches}, expected {kernels}"
        if kernels.startswith(("tiles", "region")):
            nf = 1 if name == "1x1080p" else 3 if name == "3x1080p" else 6
            assert pigo_b200.describe_plan(R, Cc, *PRM, nframes=nf)["region"] == (kernels.startswith("region"))
        # the windows of frame a against a queue sized for frame a alone: sufficient for the whole call, whose queue grows
        # by less than one item per window it adds
        hist = res[(cascade,) + key][1]
        per_frame = SC.predict_queue(hist, h, cap(WA))
        if cascade.startswith("S(") and ntrees - _k(ntrees) > h:
            assert per_frame["overflow"], f"{cascade} {name}: {per_frame}, hand-over {h}"
        overflowed += per_frame["overflow"]
    if cascade.startswith("S(") and ntrees > 50:
        assert overflowed == len(PATHS)
    total = sum(len(v) for v in want.values())
    if cascade != "special-pinf_thr":
        assert total > 0, cascade


# ---- the counter wrap ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def wrap_case():
    """F(4096), its collapsed cascade's oracle results on two distinct 1080p noise images (unrotated and at ANGLE)."""
    full, collapsed, _ = SC.flat_prefix_cascade(4096, 4096)
    ora = O.OracleFace(collapsed)
    ims = [SC.noise_frame(R, Cc, 11), SC.noise_frame(R, Cc, 12)]
    want = {(i, a): ora.run_cascade(ims[i], R, Cc, Cc, *PRM, a, with_hist=True) for i in range(2) for a in (0.0, ANGLE)}
    return pigo_b200.NewPigo().Unpack(full), ims, want


def _full_hist(hist2, n):
    """The collapsed cascade's histogram in F(n)'s trees: walking tree 1 of the collapse is walking all n trees."""
    h = np.zeros(n + 1, dtype=np.int64)
    h[1], h[n] = hist2[1], hist2[2]
    return h


def test_counter_wrap_mixed_size_call(wrap_case):
    clf, ims, want = wrap_case
    w = 2 * WA
    cap = SC.images_queue_cap(w)
    h = SC.gather_v2_handover(4096, SC.schedule(w, False, 24)["gather_limit"])
    hist = _full_hist(want[(0, 0.0)][1], 4096) + _full_hist(want[(1, 0.0)][1], 4096)
    p = SC.predict_queue(hist, h, cap)
    assert p["overflow"] and p["attempts"] > 2 ** 32, p
    imp = [ImageParams(im, R, Cc, Cc) for im in ims]
    (dets, cnt), launches = timed(lambda: clf.RunCascadeImages(imp, CascadeParams(imp[0], *PRM), 0.0))
    assert names(launches) == "gather deep", launches
    assert_slices(dets, cnt, [want[(0, 0.0)][0], want[(1, 0.0)][0]], "F(4096) images", prefilled=False)


def test_counter_wrap_rotated_batch(wrap_case):
    clf, ims, want = wrap_case
    w = 2 * WA
    cap = SC.run_scan_queue_cap(w)
    h = SC.gather_v2_handover(4096, SC.schedule(w, True, 16)["gather_limit"])
    hist = _full_hist(want[(0, ANGLE)][1], 4096) + _full_hist(want[(1, ANGLE)][1], 4096)
    p = SC.predict_queue(hist, h, cap)
    assert p["overflow"] and p["attempts"] > 2 ** 32, p
    frs = np.stack(ims)
    (dets, cnt), launches = timed(lambda: clf.RunCascadeBatch(frs, CascadeParams(ImageParams(None, R, Cc, Cc), *PRM), ANGLE))
    assert names(launches) == "gather deep", launches
    assert_slices(dets, cnt, [want[(0, ANGLE)][0], want[(1, ANGLE)][0]], "F(4096) rotated batch", prefilled=False)


# ---- capacity ------------------------------------------------------------------------------------------------------------
def test_capacity_with_overflowing_queue(expected, frames):
    """cap_per_frame below the detections of S(56, 1) on 2 x 1080p: PIGO_E_CAP with every frame's required count equal to
    the oracle's, and the retry equal to the oracle."""
    packs, res = expected
    clf = pigo_b200.NewPigo().Unpack(packs["S(56,1)"])
    want = res[("S(56,1)", "a", 0.0)][0]
    assert len(want) > 100
    for angle in (0.0, ANGLE):
        want = res[("S(56,1)", "a", angle)][0]
        rc, out, cnt = batch(clf, frames["a"], 2, angle, cap=50)
        assert rc == pigo_b200.PIGO_E_CAP and list(cnt) == [len(want)] * 2, (rc, list(cnt), len(want))
        rc, out, cnt = batch(clf, frames["a"], 2, angle, cap=int(cnt.max()))
        assert rc == 0
        assert_slices(out, cnt, [want] * 2, f"capacity retry angle {angle}")
