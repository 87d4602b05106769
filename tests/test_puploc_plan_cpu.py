"""The RunDetector fixtures of tests/test_puploc_fuzz_gpu.py on the CPU: the C and numpy oracles agree on synthetic pupil /
landmark cascades of every shape the GPU module runs, the numpy restatement of the library generator is pinned, and the
restated launch plan (tests/puploc_cases.py) is checked against the constants of pigo_b200/csrc/puploc.cu and api.cu."""
import os
import re

import numpy as np
import pytest

import oracle_lib as O
from oracle import np_oracle as NP
from pigo_b200 import synth
from puploc_cases import (M64, growth, library_randoms, mix64, pair_launch, patch_stages, puploc_cascade, standalone_kernel)

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pigo_b200", "csrc")

# (depth, trees, stages, scales): depths 1, 2, 9, 10, 12; trees 0, 1, 20, 33, 64; stages 0, 1, 7; scales 0.7, 1.0, 1.3, -0.8
SHAPES = [(1, 1, 1, 0.7), (2, 33, 7, 1.3), (9, 20, 7, 0.7), (10, 64, 1, -0.8), (12, 1, 7, 1.0), (10, 0, 7, 0.7), (9, 20, 0, 0.7),
          (2, 64, 7, -0.8), (1, 33, 7, 1.3), (12, 20, 1, 1.0)]
# every rotation slot once over the shapes, plus unrotated, slot 0 through an angle in (0, 1/32) and an angle above 1
ANGLES = [0.0, 0.01, 1.7] + [k / 32 for k in range(1, 33)]


def _image():
    img = np.full((120, 160), 0x5A, dtype=np.uint8)
    img[:, :150] = synth.frame_smooth(120, 150, seed=4, sigma=2.0) ^ synth.frame_noise(120, 150, 5) // 8
    return img


@pytest.mark.parametrize("k,shape", list(enumerate(SHAPES)))
def test_c_and_numpy_oracles_agree_on_synthetic_cascades(k, shape):
    depth, trees, stages, scales = shape
    pk = puploc_cascade(depth, trees, stages, scales, seed=k)
    a, b = O.OraclePuploc(pk), NP.PuplocCascade(pk)
    assert (a.stages, a.trees, a.depth) == (b.stages, b.trees, b.depth) == (stages, trees, depth)
    img = _image()
    rng = np.random.default_rng(k)
    angles = ANGLES[k::len(SHAPES)]
    for j, ang in enumerate(angles):
        fl = bool((j + k) % 2)
        r, c, s = float(rng.uniform(-20, 140)), float(rng.uniform(-20, 170)), float(rng.uniform(1, 300))
        x = a.classify(np.float32(r), np.float32(c), np.float32(s), img, 120, 150, 160, ang, fl)
        y = b.classify(r, c, s, img, 120, 150, 160, ang, fl)
        assert [v.tobytes() for v in x] == [v.tobytes() for v in y], (shape, ang, fl)
    rnd = rng.random(189, dtype=np.float32)
    for P in (0, 1, 2, 63) if depth * max(trees, 1) * stages <= 300 else (0, 2):
        x = a.run_detector(60, 70, 40.0, P, rnd, img, 120, 150, 160, angles[0], k % 2 == 1)
        y = b.run_detector(60, 70, 40.0, P, rnd, img, 120, 150, 160, angles[0], k % 2 == 1)
        assert (x[0], x[1], x[2].tobytes()) == (y[0], y[1], y[2].tobytes()), (shape, P)


def test_oracles_order_nan_and_signed_zero_pools_alike():
    """A pool with NaNs (NaN leaf predictions) and with -0 against the pool's +0 slots (scale 0 times scales < 0): both
    oracles pick the same entry, NaN above every number and ties by slot, and int(NaN) is 0."""
    img = _image()
    pk = puploc_cascade(4, 6, 2, -0.8, seed=3, pred=0.5, nan_leaves=0.05)
    a, b = O.OraclePuploc(pk), NP.PuplocCascade(pk)
    rnd = np.random.default_rng(1).random(189, dtype=np.float32)
    nan_seen = 0
    for P in (63, 40, 9):
        for scale in (0.0, 30.0):
            x = a.run_detector(50, 60, scale, P, rnd, img, 120, 150, 160)
            y = b.run_detector(50, 60, scale, P, rnd, img, 120, 150, 160)
            assert (x[0], x[1], x[2].tobytes()) == (y[0], y[1], y[2].tobytes()), (P, scale)
        pool = [a.classify(np.float32(50), np.float32(60), np.float32(30.0 * (0.925 + 0.15 * u)), img, 120, 150, 160) for u in rnd[2:3 * P:3]]
        nan_seen += sum(bool(np.isnan(p[0])) for p in pool)
    assert nan_seen > 0
    assert NP._to_i32(np.float32("nan")) == 0 and NP._to_i32(np.float32(3e9)) == 2 ** 31 - 1 and NP._to_i32(np.float32(-7.9)) == -7


def test_library_generator_restatement_is_pinned():
    """mix64 and the draw keys of both kernels, restated in numpy, pinned to constants; the kernel source must still hold
    the keys and constants restated here, so that a change on either side fails on the CPU first."""
    assert (mix64(0), mix64(1), mix64(M64), mix64(123456789)) == (14819496, 9505325, 14997873, 2243700)
    assert [hex(v) for v in library_randoms(0, 0)[0].view("u4")] == ["0x3f6220a8", "0x3f110a2d", "0x3f175835"]
    assert [hex(v) for v in library_randoms(7, 1000)[5].view("u4")] == ["0x39171000", "0x3f437938", "0x3f04449f"]
    assert [hex(v) for v in library_randoms(M64, 3)[62].view("u4")] == ["0x3f27e597", "0x3ef83e20", "0x3b805e00"]
    d = library_randoms(11, 5)
    assert d.dtype == np.float32 and (d >= 0).all() and (d < 1).all() and len(set(d.ravel().tolist())) == d.size
    src = open(os.path.join(CSRC, "puploc.cu")).read()
    for const in ("0x9E3779B97F4A7C15ull", "(x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull", "(x ^ (x >> 27)) * 0x94D049BB133111EBull", "x ^= x >> 31",
                  "(uint32_t)(x >> 40)", "rng_seed * 0xD1342543DE82EF95ull + (uint64_t)sidx * 64 + i",
                  "W.rng_seed * 0xD1342543DE82EF95ull + ((uint64_t)slot + W.slot_base) * 64 + tid", "mix64(key * 3 + 2) * (1.0f / 16777216.0f)"):
        assert const in src, const


def test_launch_plan_restatement_matches_the_source_and_its_boundaries():
    """pair_launch restates launch_puploc_pairs: depth 10 with 20 / 24 / 25 trees is patch / staged only / unstaged under
    puploc_stage 2, 203 trees still run the pair kernel and 204 do not; a launch is sized by its largest cascade."""
    src = open(os.path.join(CSRC, "puploc.cu")).read()
    for frag in ("if (leaf > 100 * 1024) return -1;", "const size_t kBudget = 110 * 1024;", "leaf + codes_max + 4096 <= kBudget",
                 "std::min<size_t>(48 * 1024, kBudget - leaf - codes_max)", "(size_t)T.trees * (4 * (size_t)T.leaves + 8)",
                 "(a >> 1) + 2", "((iqs < 0 ? -iqs : iqs) + (iqc < 0 ? -iqc : iqc)) >> 9) + 2", "min(max(s_box[2], 0), clim) & ~15",
                 "((long long)c1 - c0 + 16) & ~15ll", "(dim() & 15) || (reinterpret_cast<uintptr_t>(pixels) & 15)"):
        assert frag in src, frag
    assert [pair_launch([(t, 10)], 2) for t in (20, 24, 25)] == [(True, 20480), (True, 0), (False, 0)]
    assert [pair_launch([(20, 10)], s) for s in (0, 1)] == [(False, 0), (True, 0)]
    assert pair_launch([(203, 4)], 2) == (False, 0) and pair_launch([(204, 4)], 2) is None
    assert pair_launch([(20, 10), (33, 5), (204, 1)], 1) is None
    assert pair_launch([(20, 10), (25, 10)], 2) == (False, 0)
    api = open(os.path.join(CSRC, "api.cu")).read()
    assert "std::fabs((double)scale) * growth <= 16384.0" in api and "puploc_growth(cidx < 0 ? puploc : flp[cidx]) > 512.0" in api
    assert growth(0, 3.0) == growth(1, 3.0) == growth(20, 0.7) == growth(9, -1.0) == 1.0 and growth(19, 2.0) == 2.0 ** 18
    small = puploc_cascade(3, 4, 20, 2.0, seed=1)
    assert standalone_kernel(small, [0.03], 0) == "pair" and standalone_kernel(small, [0.04], 0) == "warp"   # 0.04 * 2^19 > 16384
    assert standalone_kernel(small, [0.03], 1) == "warp"
    assert standalone_kernel(puploc_cascade(1, 204, 1, 0.7, seed=1), [10.0], 0) == "warp"


def test_patch_restatement_on_hand_built_cases():
    """Small seeds in the middle of an aligned image are served from the patch at every stage; the same call on an
    unaligned base, or with a seed whose sample box exceeds the cap, gathers from global memory; Perturbs 0 never stages."""
    img = _image()
    pk = puploc_cascade(5, 8, 4, 0.8, seed=2)
    rnd = np.random.default_rng(3).random((63, 3), dtype=np.float32)
    im = (img, 120, 150, 160)
    assert patch_stages(pk, (60, 70, 12.0, 30), rnd, im, 0.0, False, 20480, True) == (4, 0)
    assert patch_stages(pk, (60, 70, 12.0, 30), rnd, im, 0.0, False, 20480, False) == (0, 4)
    assert patch_stages(pk, (60, 70, 12.0, 0), rnd, im, 0.0, False, 20480, True) == (0, 4)
    assert patch_stages(pk, (60, 70, 12.0, 30), rnd, im, 0.3, True, 0, True) == (0, 4)
    big = patch_stages(pk, (60, 70, 400.0, 30), rnd, im, 0.0, False, 1024, True)
    assert big[0] < 4 and sum(big) == 4
