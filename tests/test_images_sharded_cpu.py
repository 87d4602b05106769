"""The split of the sharded mixed-size calls (pigo_shard_plan) and their argument checks, without a device.  The split
must be contiguous, cover every entry once, be deterministic and reach the least largest-shard cost any contiguous split
reaches under the cost model count_windows x (rotated ? 1.4 : 1) + 4096 per entry."""
import ctypes as C
import functools
import math

import numpy as np
import pytest

import pigo_b200
from abi_cases import IMAGE_CASES, PIPELINE_CASES, descs, detect, scan
from pigo_b200 import CascadeParams, ImageParams

TEST_PARAMS = (20, 1000, 0.2, 1.1)   # core/pigo_test.go:44-50
ROT, UNROT, IMG = 14, 10, 4096 * 10   # the cost model in tenths of a window (pigo_b200/csrc/api.cu)


def geoms(seed, n):
    rng = np.random.default_rng(seed)
    shapes = [(1, 1), (10, 10), (22, 22), (400, 320), (480, 640), (1080, 1920), (2160, 3840), (97, 131), (45, 1200), (900, 41)]
    out = []
    for _ in range(n):
        if rng.random() < 0.5:
            r, c = shapes[rng.integers(len(shapes))]
        else:
            r, c = int(rng.integers(1, 1200)), int(rng.integers(1, 1600))
        out.append((r, c, c + int(rng.integers(0, 3))))
    return out


def costs(g, angles=None, params=TEST_PARAMS):
    out = []
    for k, (r, c, _) in enumerate(g):
        w = pigo_b200.count_windows(r, c, *params)
        rot = angles is not None and angles[k] > 0
        out.append(w * (ROT if rot else UNROT) + IMG)
    return out


def best_bottleneck(cost, k):
    """Least largest-range cost of a split of cost[] into at most k contiguous ranges (exhaustive DP)."""
    n = len(cost)
    pre = np.concatenate([[0], np.cumsum(cost, dtype=np.int64)])

    @functools.lru_cache(maxsize=None)
    def f(i, s):   # entries i.. into at most s ranges
        if i == n:
            return 0
        if s == 0:
            return math.inf
        return min(max(int(pre[j] - pre[i]), f(j, s - 1)) for j in range(i + 1, n + 1))
    return f(0, k)


def plan(g, nshards, angles=None, params=TEST_PARAMS):
    return pigo_b200.shard_plan([(0, r, c, d) for r, c, d in g], *params, angles=angles, nshards=nshards)


def shard_costs(first, cost):
    return [sum(cost[first[s]:first[s + 1]]) for s in range(len(first) - 1)]


@pytest.mark.parametrize("seed,n,k", [(1, 12, 2), (2, 12, 3), (3, 17, 4), (4, 9, 8), (5, 25, 5), (6, 30, 7)])
def test_ranges_are_contiguous_cover_everything_and_reach_the_best_bottleneck(seed, n, k):
    g = geoms(seed, n)
    angles = [float(a) for a in np.random.default_rng(seed).choice([0.0, 0.0, 0.25, 1.0, -0.5], size=n)]
    for ang in (None, angles):
        first = plan(g, k, ang)
        assert first[0] == 0 and first[-1] == n
        assert len(first) - 1 == min(k, n)
        assert all(a < b for a, b in zip(first, first[1:])), first   # non-empty, in caller order
        cost = costs(g, ang)
        worst = max(shard_costs(first, cost))
        best = best_bottleneck(cost, k)
        assert worst <= best + max(cost)   # the bound the split promises ...
        assert worst == best               # ... and what the bottleneck search reaches


def test_the_plan_is_deterministic():
    g = geoms(7, 200)
    angles = [0.1 * (k % 4) for k in range(200)]
    a = plan(g, 8, angles)
    assert all(plan(g, 8, angles) == a for _ in range(5))


def test_a_4k_image_among_thumbnails_gets_a_shard_of_its_own():
    g = [(120, 160, 160)] * 20 + [(2160, 3840, 3840)] + [(120, 160, 160)] * 20
    first = plan(g, 4)
    assert 20 in first and 21 in first, first
    costs_ = shard_costs(first, costs(g))
    assert max(costs_) == costs(g)[20]
    # the count-based split would have put the 4K image with ten thumbnails
    assert len(first) == 5


def test_balance_is_on_cost_not_on_count():
    g = [(1080, 1920, 1920)] * 4 + [(100, 100, 100)] * 12
    first = plan(g, 2)
    assert first == [0, 2, 16], first


@pytest.mark.parametrize("n,k", [(0, 3), (1, 4), (3, 8), (5, 5)])
def test_more_shards_than_entries_use_one_shard_per_entry(n, k):
    g = geoms(8, n)
    first = plan(g, k)
    assert first == list(range(n + 1))


def test_rotated_entries_weigh_more():
    g = [(480, 640, 640)] * 10
    assert plan(g, 2) == [0, 5, 10]
    # the first four rotated: 4 x 1.4 = 5.6 image-costs on the left, so the cut moves left
    first = plan(g, 2, [0.25] * 4 + [0.0] * 6)
    assert first[1] < 5, first
    first = plan(g, 2, [0.0] * 6 + [0.5] * 4)
    assert first[1] > 5, first
    # NaN and negative angles scan unrotated and weigh the same as 0
    assert plan(g, 2, [math.nan, -1.0] * 2 + [0.0] * 6) == [0, 5, 10]


def test_nshards_zero_follows_the_option_and_else_the_devices():
    g = geoms(9, 10)
    old = pigo_b200.get_option("shard_split")
    try:
        pigo_b200.set_option("shard_split", 4)
        assert len(plan(g, 0)) == 5
        pigo_b200.set_option("shard_split", 0)
        assert 2 <= len(plan(g, 0)) <= 17   # one shard per selected device (the default device when none was selected)
    finally:
        pigo_b200.set_option("shard_split", old)


def test_plan_argument_errors():
    L = pigo_b200.lib()
    n = C.c_int()
    first = (C.c_int * 4)()
    d = pigo_b200.image_descs([(0, 10, 10, 10)])
    assert L.pigo_shard_plan(d, -1, None, *TEST_PARAMS, 2, first, C.byref(n)) == pigo_b200.PIGO_E_INVALID
    assert L.pigo_shard_plan(None, 1, None, *TEST_PARAMS, 2, first, C.byref(n)) == pigo_b200.PIGO_E_INVALID
    assert L.pigo_shard_plan(d, 1, None, *TEST_PARAMS, -2, first, C.byref(n)) == pigo_b200.PIGO_E_INVALID
    assert L.pigo_shard_plan(d, 1, None, *TEST_PARAMS, 2, first, None) == pigo_b200.PIGO_E_INVALID
    bad = pigo_b200.image_descs([(0, 10, 10, 9)])
    assert L.pigo_shard_plan(bad, 1, None, *TEST_PARAMS, 2, first, C.byref(n)) == pigo_b200.PIGO_E_INVALID
    assert L.pigo_shard_plan(d, 1, None, 20, 1000, 0.2, 1.1, 2, None, C.byref(n)) == 0 and n.value == 1


# ---- argument errors of the four calls: all reached before any device work ---------------------------------------------
def test_run_cascade_images_sharded_argument_errors():
    for case, images, nimages, kw, msg in IMAGE_CASES + [("valid images", descs((40, 40, 40), (30, 50, 50)), 2, {}, "null cascade")]:
        rc, err = scan("pigo_run_cascade_images_sharded", images, nimages, angles=False, **kw)
        assert rc == pigo_b200.PIGO_E_INVALID, case
        assert msg in err, (case, err)


def test_detect_images_sharded_argument_errors():
    for case, images, nimages, kw, msg in PIPELINE_CASES + [("valid images", descs((40, 40, 40), (30, 50, 50)), 2, {}, "null cascade")]:
        rc, err = detect("pigo_detect_images_sharded", images, nimages, angles=False, **kw)
        assert rc == pigo_b200.PIGO_E_INVALID, case
        assert msg in err, (case, err)


def test_decoded_sharded_argument_errors():
    pix = np.zeros(40 * 30 * 8, dtype=np.uint8)
    good = pigo_b200.DecodedImage(pigo_b200.DECODED_GRAY, 40, 30, (pix,), (40, 0))
    bad_fmt = pigo_b200.DecodedImage(4, 40, 30, (pix,), (40, 0))
    short = pigo_b200.DecodedImage(pigo_b200.DECODED_RGBA64, 40, 30, (pix,), (100, 0))
    no_plane = pigo_b200.DecodedImage(pigo_b200.DECODED_GRAY, 40, 30, (None,), (40, 0))
    empty = pigo_b200.DecodedImage(pigo_b200.DECODED_GRAY, 0, 30, (pix,), (40, 0))
    one = pigo_b200.decoded_descs([good])
    cases = [([good, bad_fmt], 2, "source 1: unknown format 4"), ([good, short], 2, "source 1: stride 100 below the row"),
             ([no_plane, good], 2, "source 0: null plane"), ([empty], 1, "source 0: bad size 0x30"),
             ([good], -1, "-1 sources: outside 0..65535"), ([good], 70000, "70000 sources: outside 0..65535"), (None, 1, "null src"),
             ([good, good], 2, "null cascade")]   # the last: valid sources, null cascade
    for srcs, n, msg in cases:
        desc = pigo_b200.decoded_descs(srcs) if srcs is not None else None
        for entry, call in (("pigo_run_cascade_decoded_sharded", scan), ("pigo_detect_decoded_sharded", detect)):
            rc, err = call(entry, desc, n, angles=False)
            assert rc == pigo_b200.PIGO_E_INVALID and msg in err, (entry, msg, err)
    for entry, call, kw, msg in (("pigo_run_cascade_decoded_sharded", scan, {"with_out": False}, "null out"),
                                 ("pigo_run_cascade_decoded_sharded", scan, {"with_n_out": False}, "null n_out"),
                                 ("pigo_detect_decoded_sharded", detect, {"params": False}, "null params"),
                                 ("pigo_detect_decoded_sharded", detect, {"face_cap": 0}, "face_cap")):
        rc, err = call(entry, one, 1, angles=False, **kw)
        assert rc == pigo_b200.PIGO_E_INVALID and msg in err, (entry, msg, err)


def test_mirrors_check_the_angle_count():
    clf = pigo_b200.Pigo()
    clf._h = C.c_void_p(1)   # never reaches the library
    with pytest.raises(ValueError):
        clf.run_cascade_images_sharded([ImageParams(np.zeros(4, np.uint8), 2, 2, 2)], CascadeParams(ImageParams(), *TEST_PARAMS), angles=[0.0, 0.1])
    clf._h = None
