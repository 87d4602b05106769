"""The deep-queue fixtures of tests/scan_cases.py on the CPU: the C and numpy oracles agree byte for byte on every cascade
family, unrotated and at several rotation slots; a flat-prefix cascade F(n) gives exactly its collapsed two-tree cascade;
the families do what their tests rely on (survivor and detection rates, ties at every tree range); and the restated queue
sizes, hand-over points and schedule match pigo_b200/csrc."""
import numpy as np
import pytest

import oracle_lib as O
from oracle import np_oracle
import scan_cases as SC

PRM = (20, 70, 0.2, 1.1)
ANGLES = [0.0, 3 / 32.0, 0.5, 0.97]


def _np_dets(pk, frame, prm, angle):
    rows, cols = frame.shape
    dets = np_oracle.FaceCascade(pk).run_cascade(frame, rows, cols, cols, *prm, angle)
    return np.array(dets, dtype=O.DET_DTYPE)


FAMILIES = {
    "S(9,3)": lambda: SC.survivor_cascade(9, 3, 1),
    "S(53,4)": lambda: SC.survivor_cascade(53, 4, 2),
    "S(100,1)": lambda: SC.survivor_cascade(100, 1, 3),
    "F(64)": lambda: SC.flat_prefix_cascade(64, 4)[0],
    "ties(60)": lambda: SC.tie_cascade(60, 5),
    **{f"special-{k}": (lambda k=k: SC.special_cascade(100, 6, SC.SPECIALS[k])) for k in SC.SPECIALS},
}


@pytest.mark.filterwarnings("ignore:invalid value encountered:RuntimeWarning")   # inf + -inf in the special cascades
@pytest.mark.parametrize("family", list(FAMILIES))
def test_c_and_numpy_oracles_agree(family):
    pk = FAMILIES[family]()
    ora = O.OracleFace(pk)
    frame = SC.noise_frame(90, 130, 77)
    total = 0
    for angle in ANGLES:
        c = ora.run_cascade(frame, 90, 130, 130, *PRM, angle)
        n = _np_dets(pk, frame, PRM, angle)
        assert c.tobytes() == n.tobytes(), f"{family} angle {angle}: {len(c)} vs {len(n)} detections"
        total += len(c)
    if family != "special-pinf_thr":
        assert total > 0, family


@pytest.mark.parametrize("n", [2, 9, 64, 300])
def test_flat_prefix_equals_collapsed_cascade(n):
    full, collapsed, C = SC.flat_prefix_cascade(n, 100 + n)
    assert C != 0 and np.signbit(C) == (C < 0)
    of, oc = O.OracleFace(full), O.OracleFace(collapsed)
    assert (of.ntrees, oc.ntrees) == (n, 2)
    frame = SC.noise_frame(200, 300, n)
    windows = O.count_windows(200, 300, 20, 200, 0.1, 1.1)
    for angle in ANGLES:
        a, hist = of.run_cascade(frame, 200, 300, 300, 20, 200, 0.1, 1.1, angle, with_hist=True)
        b, hist2 = oc.run_cascade(frame, 200, 300, 300, 20, 200, 0.1, 1.1, angle, with_hist=True)
        assert a.tobytes() == b.tobytes(), f"n {n} angle {angle}"
        assert hist[n] == hist2[2] == windows and hist.sum() == windows     # every window walks every tree
        assert 0.05 < len(a) / windows < 0.2, len(a) / windows              # about one window in eight detects


@pytest.mark.parametrize("n,k", [(9, 1), (56, 8), (468, 6)])
def test_survivor_cascade_rates(n, k):
    """Every window walks the first n - k trees; 0.5 .. 10 % are detected (on a 1080p-like noise crop)."""
    pk = SC.survivor_cascade(n, k, 7 + n)
    frame = SC.noise_frame(240, 320, 9)
    dets, hist = O.OracleFace(pk).run_cascade(frame, 240, 320, 320, 20, 1000, 0.2, 1.1, with_hist=True)
    windows = O.count_windows(240, 320, 20, 1000, 0.2, 1.1)
    assert hist[:n - k].sum() == 0 and hist.sum() == windows
    assert 0.005 <= len(dets) / windows <= 0.10, len(dets) / windows
    codes, leaves, thresh = SC.unpack(pk)
    assert np.isneginf(thresh[:n - k]).all() and np.isfinite(thresh[n - k:]).all()
    assert (leaves != np.round(leaves * 2 ** 10) / 2 ** 10).mean() > 0.99            # not dyadic: summation order matters


def _walk_sums(pk, frame, scale):
    """Partial sums after every tree of every window of one scale (no rejection), and the thresholds."""
    codes, leaves, thresh = SC.unpack(pk)
    rows, cols = frame.shape
    rr, cc = np_oracle.grid(rows, cols, scale, 0.1)
    R, Cc = np.meshgrid(rr, cc, indexing="ij")
    r, c = R.ravel().astype(np.int64), Cc.ravel().astype(np.int64)
    s = np.full(len(r), scale, dtype=np.int64)
    acc = np.zeros(len(r), dtype=np.float32)
    sums = np.empty((len(thresh), len(r)), dtype=np.float32)
    for t in range(len(thresh)):
        acc = (acc + SC.leaf_values(codes, leaves, t, frame, r, c, s)).astype(np.float32)
        sums[t] = acc
    return sums, thresh


def test_tie_cascade_hits_ties_in_every_range():
    """acc == thr on windows still alive at trees of the tile prefix (< 8), the gather prefix, around the resident prefix
    (48), in the deep range, and q == 0 at the last tree: each is a rejection, and the oracles agree on it."""
    n = 200
    pk = SC.tie_cascade(n, 11)
    frame = SC.noise_frame(200, 200, 12)
    ties = np.zeros(n, dtype=np.int64)
    for scale in (24, 40, 70):
        sums, thresh = _walk_sums(pk, frame, scale)
        alive = np.ones(sums.shape[1], dtype=bool)
        for t in range(n):
            ties[t] += int((alive & (sums[t] == thresh[t])).sum())
            alive &= ~(sums[t] <= thresh[t])
    for lo, hi in [(0, 8), (8, 48), (48, 56), (56, n - 1), (n - 1, n)]:
        assert ties[lo:hi].sum() > 0, (lo, hi, ties[lo:hi])
    dets = O.OracleFace(pk).run_cascade(frame, 200, 200, 200, 20, 1000, 0.1, 1.1)
    assert len(dets) > 0 and (dets["q"] > 0).all()


def test_special_cascade_values_are_placed():
    for name, at in SC.SPECIALS.items():
        codes, leaves, thresh = SC.unpack(SC.special_cascade(100, 6, at))
        for t, kind in at.items():
            if kind.endswith("_thr"):
                v = {"nan_thr": np.nan, "pinf_thr": np.inf, "ninf_thr": -np.inf}[kind]
                assert np.array_equal(thresh[t], np.float32(v), equal_nan=True), (name, t)
            elif kind == "negzero_leaves":
                assert ((leaves[t] == 0) & np.signbit(leaves[t])).sum() == 5, (name, t)
            else:
                v = {"nan_leaf": np.nan, "pinf_leaf": np.inf, "ninf_leaf": -np.inf}[kind]
                assert 0 < np.isclose(leaves[t], v, equal_nan=True).sum() < 64, (name, t)


# ---- restated constants --------------------------------------------------------------------------------------------------
def test_queue_constants_match_sources():
    drv, host, api, deep, common = (SC.sources_text(f) for f in ("scan_driver.cu", "host.h", "api.cu", "deep.cu", "common.cuh"))
    assert "std::min<uint64_t>(total_windows / 16 + total_windows / (g_opt.tile_ptab.load() != 0 ? 16 : 32) + 65536, 1ull << 26)" in drv
    assert "std::min<uint64_t>(group_windows / 32 + 65536, 1ull << 26)" in drv
    assert "const bool small = call_windows <= 4000000ull;" in drv
    assert "if (glimit <= 0) glimit = rot ? (small ? 8 : 24) : (call_windows <= 40000000ull ? 8 : large_limit);" in drv
    assert "if (P.deep_group != 8 && P.deep_group != 16 && P.deep_group != 32) P.deep_group = small ? 32 : 8;" in drv
    assert "static bool deep_ordered(uint64_t call_windows) { return call_windows > 4000000ull; }" in drv
    assert "images_schedule(call_windows, rot, 16)" in drv and "images_schedule(pass_windows, !p.tables.empty(), 24)" in api
    assert "G.ks = round_ks(std::min<long long>(g_opt.gather_ks.load(), T.gather_limit));" in drv
    assert "std::min<long long>(g_opt.gather_ks.load(), P.gather_limit)" in drv
    assert "std::atomic<long long> tile_ks{48};" in host and "std::atomic<long long> gather_ks{32};" in host
    assert "kImagesGroupWindows = 128ull * 894448ull;" in api
    assert "if (sub <= 0) sub = resident ? 128 : 64;" in api
    assert deep.count("const uint32_t qn = min(*A.long_count, A.long_cap);") >= 3     # consumers clamp the count to the cap
    assert "unsigned int* long_count;" in common and "uint32_t long_cap;" in common      # a u32 count: it can wrap
    assert SC.run_scan_queue_cap(894448) == 894448 // 16 + 894448 // 32 + 65536
    assert SC.run_scan_queue_cap(1 << 31) == SC.images_queue_cap(1 << 32) == 1 << 26
    assert SC.schedule(894448, False, 16) == {"gather_limit": 8, "deep_group": 32, "deep_ordered": False}
    assert SC.schedule(6 * 894448, True, 16) == {"gather_limit": 24, "deep_group": 8, "deep_ordered": True}
    assert SC.schedule(50_000_000, False, 24)["gather_limit"] == 24


def test_gather_role_stops_asking_after_a_refusal():
    """The gather role's hand-over is skipped once the queue refused one of the lane's windows, so the u32 count passes the
    cap by at most one refusal per lane instead of growing by one per refused window and tree."""
    src = SC.sources_text("scan_tiled.cu")
    body = src[src.index("__device__ __forceinline__ void gather_role("):src.index("// Stages the first KS tree records")]
    assert "else if (tbo[u] >= casc_end && S.longq != nullptr && !queue_full) {" in body
    refusal = body[body.index("if (pos < S.long_cap) {"):]
    assert refusal.index("} else {") < refusal.index("queue_full = true;") < refusal.index("}\n", refusal.index("queue_full = true;"))


def test_predictor_and_the_wrap_figures():
    """The predictor on hand-made histograms, and the counter-wrap sizes of tests/test_scan_overflow_gpu.py: F(4096) over
    two 1080p images makes more than 2^32 hand-over attempts when refused windows ask after every tree."""
    h = np.zeros(11, dtype=np.int64)
    h[[1, 5, 9, 10]] = [100, 7, 3, 4]   # 7 windows outlive 4 trees
    assert SC.predict_queue(h, 4, 5) == {"survivors": 14, "overflow": True, "attempts": 5 + 2 * 5 + 7 * 1}
    assert SC.predict_queue(h, 10, 5)["survivors"] == 0 and not SC.predict_queue(h, 4, 14)["overflow"]
    w = 2 * O.count_windows(1080, 1920, 20, 1000, 0.2, 1.1)
    assert w == 1_788_896
    hist = np.zeros(4097, dtype=np.int64)
    hist[4096] = w
    cap = SC.images_queue_cap(w)
    glimit = SC.schedule(w, False, 24)["gather_limit"]
    p = SC.predict_queue(hist, SC.gather_v2_handover(4096, glimit), cap)
    assert cap == 121_439 and p["overflow"] and p["attempts"] == cap + (w - cap) * (4096 - 8)
    assert p["attempts"] > 1.5 * 2 ** 32
    rot = SC.predict_queue(hist, SC.gather_v2_handover(4096, SC.schedule(w, True, 16)["gather_limit"]), SC.run_scan_queue_cap(w))
    assert rot["attempts"] > 1.4 * 2 ** 32
