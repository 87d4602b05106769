"""GPU parity tests: libpigo_b200 (through the C-ABI, via the ctypes mirror of the Go API) against the CPU
oracle on identical grayscale buffers.  Bar: (row, col, scale) integer-exact AND in the reference's emission
order, Q bit-equal (float32 adds happen in tree order on both sides) -- stronger than the 1e-4 asked."""
import numpy as np
import pytest

import oracle_lib as O
import pigo_b200
from pigo_b200 import CascadeParams, ImageParams, Puploc, synth
import pipeline_oracle as P
from mixed_images import cascades, run_cpp_mirror   # noqa: F401 (fixture)
from option_guard import options, options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)
from synthetic import synthetic_cascade

pytestmark = pytest.mark.gpu

TEST_PARAMS = (20, 1000, 0.2, 1.1)   # core/pigo_test.go:44-50
DOC_PARAMS = (20, 1000, 0.1, 1.1)    # README
CLI_PARAMS = (20, 1000, 0.15, 1.15)  # cmd/pigo/main.go:110-111


def cp_of(img, rows, cols, dim, params):
    return CascadeParams(ImageParams(img, rows, cols, dim), params[0], params[1], params[2], params[3])


def assert_same(gpu: np.ndarray, ora: np.ndarray):
    assert len(gpu) == len(ora), f"{len(gpu)} detections vs oracle {len(ora)}"
    assert gpu.tobytes() == ora.tobytes()   # row, col, scale, and the float32 bits of q, in order


@pytest.mark.parametrize("params", [TEST_PARAMS, DOC_PARAMS, CLI_PARAMS])
def test_sample_image(gpu_face, oracle_face, sample_gray, params, golden):
    g = gpu_face.run_cascade_array(cp_of(sample_gray, 400, 320, 320, params), 0.0)
    assert_same(g, oracle_face.run_cascade(sample_gray, 400, 320, 320, *params, 0.0))
    if params == TEST_PARAMS:
        assert g.tobytes() == golden["sample_test_dets"].tobytes()
        # the reference's own assertion (core/pigo_test.go:68-84) through the mirrored API
        dets = gpu_face.RunCascade(cp_of(sample_gray, 400, 320, 320, params), 0.0)
        assert len(gpu_face.ClusterDetections(dets, 0.1)) > 0


@pytest.mark.parametrize("k", [1, 3, 8, 13, 16, 21, 27, 31, 32, 40])
def test_rotated_sample(gpu_face, oracle_face, sample_gray, k):
    a = k / 32.0   # every quadrant of the table; 40/32 > 1 exercises the clamp to 1.0 (core/pigo.go:233-235)
    g = gpu_face.run_cascade_array(cp_of(sample_gray, 400, 320, 320, TEST_PARAMS), a)
    assert_same(g, oracle_face.run_cascade(sample_gray, 400, 320, 320, *TEST_PARAMS, a))


def test_rotated_wide_frame_column_clamp_quirk(gpu_face, oracle_face, sample_gray):
    """cols > rows: the reference clamps COLUMNS with nrows-1 (core/pigo.go:168,:171)."""
    fr = synth.frame_faces(sample_gray, 300, 900, noise_seed=1)
    for a in (0.05, 0.5, 0.97):
        g = gpu_face.run_cascade_array(cp_of(fr, 300, 900, 900, TEST_PARAMS), a)
        assert_same(g, oracle_face.run_cascade(fr, 300, 900, 900, *TEST_PARAMS, a))


def test_strided_and_odd_geometry(gpu_face, oracle_face):
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, size=(97, 160), dtype=np.uint8)
    for ang in (0.0, 0.7):
        g = gpu_face.run_cascade_array(cp_of(img, 97, 131, 160, (12, 90, 0.1, 1.2)), ang)   # Dim != Cols (Q7)
        assert_same(g, oracle_face.run_cascade(img, 97, 131, 160, 12, 90, 0.1, 1.2, ang))
    patch = synth.frame_faces(None, 333, 517, shift=(11, 7))
    buf = np.zeros((333, 531), dtype=np.uint8)
    buf[:, :517] = patch
    g = gpu_face.run_cascade_array(cp_of(buf, 333, 517, 531, DOC_PARAMS), 0.0)
    o = oracle_face.run_cascade(buf, 333, 517, 531, *DOC_PARAMS, 0.0)
    assert len(o) > 0
    assert_same(g, o)


def test_empty_and_degenerate_inputs(gpu_face, oracle_face):
    tiny = np.zeros((10, 10), dtype=np.uint8)
    assert len(gpu_face.run_cascade_array(cp_of(tiny, 10, 10, 10, TEST_PARAMS), 0.0)) == 0   # no scale fits
    assert gpu_face.RunCascade(cp_of(tiny, 10, 10, 10, (100, 50, 0.2, 1.1)), 0.0) == []       # MinSize > MaxSize
    one = np.random.default_rng(0).integers(0, 256, size=(22, 22), dtype=np.uint8)           # exactly one window
    g = gpu_face.run_cascade_array(cp_of(one, 22, 22, 22, (20, 20, 0.2, 1.1)), 0.0)
    assert_same(g, oracle_face.run_cascade(one, 22, 22, 22, 20, 20, 0.2, 1.1, 0.0))
    assert pigo_b200.count_windows(22, 22, 20, 20, 0.2, 1.1) == 1
    assert pigo_b200.count_windows(21, 21, 20, 20, 0.2, 1.1) == 0
    # shift factor 0 -> step 1 (core/pigo.go:227 max(...,1))
    img = synth.frame_faces(None, 120, 100, shift=(-150, -100))
    g = gpu_face.run_cascade_array(cp_of(img, 120, 100, 100, (30, 60, 0.0, 1.5)), 0.0)
    assert_same(g, oracle_face.run_cascade(img, 120, 100, 100, 30, 60, 0.0, 1.5, 0.0))
    with pytest.raises(pigo_b200.PigoError):
        gpu_face.run_cascade_array(cp_of(img, 120, 100, 100, (-2, 60, 0.1, 1.5)), 0.0)         # negative MinSize: the reference would panic


@pytest.mark.parametrize("cls", ["U", "S", "F"])
def test_1080p_frame_each_content_class(gpu_face, oracle_face, cls):
    fr = synth.make_batch(2, 1080, 1920, cls * 2, seed0=3)[1]
    g = gpu_face.run_cascade_array(cp_of(fr, 1080, 1920, 1920, TEST_PARAMS), 0.0)
    assert_same(g, oracle_face.run_cascade(fr, 1080, 1920, 1920, *TEST_PARAMS, 0.0))


def test_1080p_golden_vector(gpu_face, golden, sample_gray):
    f1080 = synth.frame_faces(sample_gray, 1080, 1920)
    g = gpu_face.run_cascade_array(cp_of(f1080, 1080, 1920, 1920, TEST_PARAMS), 0.0)
    assert g.tobytes() == golden["f1080_test_dets"].tobytes()
    srt, cl = gpu_face.cluster_array(g, 0.2)
    assert cl.tobytes() == golden["f1080_test_clusters"].tobytes()


def test_batch_matches_per_frame_oracle(gpu_face, oracle_face):
    frames = synth.make_batch(6, 540, 960, "USF", seed0=10)
    cp = cp_of(None, 540, 960, 960, TEST_PARAMS)
    dets, cnt = gpu_face.RunCascadeBatch(frames, cp, 0.0, cap_per_frame=256)
    for f in range(6):
        o = oracle_face.run_cascade(frames[f], 540, 960, 960, *TEST_PARAMS, 0.0)
        assert cnt[f] == len(o)
        assert dets[f, :cnt[f]].tobytes() == o.tobytes()


def test_capacity_overflow_reports_required_count(gpu_face, oracle_face):
    fr = synth.frame_faces(None, 1080, 1920, noise_seed=9)
    o = oracle_face.run_cascade(fr, 1080, 1920, 1920, *TEST_PARAMS, 0.0)
    assert len(o) > 8
    import ctypes as C
    out = np.zeros(4, dtype=pigo_b200.DET_DTYPE)
    n = C.c_int()
    rc = pigo_b200.lib().pigo_run_cascade(gpu_face._h, fr.ctypes.data, 1080, 1920, 1920, 20, 1000, 0.2, 1.1, 0.0,
                                          out.ctypes.data, 4, C.byref(n))
    assert rc == pigo_b200.PIGO_E_CAP and n.value == len(o)
    assert_same(gpu_face.run_cascade_array(cp_of(fr, 1080, 1920, 1920, TEST_PARAMS), 0.0, cap=4), o)  # retry path


def test_4k_rotated_slot(gpu_face, oracle_face):
    """config 4 shape (3840x2160), one table slot; property: slot 32 == unrotated where no clamp bites is NOT
    true on wide frames (column clamp quirk), so compare with the oracle only."""
    fr = synth.frame_faces(None, 2160, 3840, shift=(5, 9), noise_seed=4)
    for a in (7 / 32.0,):
        g = gpu_face.run_cascade_array(cp_of(fr, 2160, 3840, 3840, TEST_PARAMS), a)
        assert_same(g, oracle_face.run_cascade(fr, 2160, 3840, 3840, *TEST_PARAMS, a))
    assert pigo_b200.count_windows(2160, 3840, *TEST_PARAMS) == 3669137


# ---- ClusterDetections --------------------------------------------------------------------------------------
@pytest.mark.parametrize("thr", [0.0, 0.1, 0.15, 0.2, 0.5, 1.0])
def test_cluster_matches_oracle(gpu_face, oracle_face, thr):
    fr = synth.frame_faces(None, 1080, 1920, noise_seed=2)
    d = oracle_face.run_cascade(fr, 1080, 1920, 1920, *DOC_PARAMS, 0.0)
    assert len(d) > 100
    srt_o, cl_o = O.cluster(d, thr)
    srt_g, cl_g = gpu_face.cluster_array(d.copy(), thr)
    assert srt_g.tobytes() == srt_o.tobytes()       # in-place sort by Q ascending (stable)
    assert cl_g.tobytes() == cl_o.tobytes()


def test_cluster_with_exact_score_ties(gpu_face, oracle_face, sample_gray):
    fr = synth.frame_faces(sample_gray, 1080, 1920)
    d = oracle_face.run_cascade(fr, 1080, 1920, 1920, *DOC_PARAMS, 0.0)
    d["q"] = np.round(d["q"])                         # force many exact score ties (tie order: stable, documented)
    qs = d["q"]
    assert len(np.unique(qs)) < len(qs) // 2
    for thr in (0.0, 0.2):
        srt_o, cl_o = O.cluster(d, thr)
        srt_g, cl_g = gpu_face.cluster_array(d.copy(), thr)
        assert srt_g.tobytes() == srt_o.tobytes() and cl_g.tobytes() == cl_o.tobytes()


def test_cluster_edge_cases(gpu_face):
    assert gpu_face.ClusterDetections([], 0.2) == []
    one = [pigo_b200.Detection(10, 10, 20, 3.5)]
    assert gpu_face.ClusterDetections(one, 0.2) == [pigo_b200.Detection(10, 10, 20, 3.5)]


# ---- RunDetector / GetLandmarkPoint -------------------------------------------------------------------------
def test_puploc_golden_cases(golden, sample_gray):
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
    img = ImageParams(sample_gray, 400, 320, 320)
    rnd = golden["puploc_randoms"]
    for row in golden["puploc_cases"]:
        r0, cc, sc, P, ang, fl, o0, o1, o2 = row
        p = plc.RunDetector(Puploc(int(r0), int(cc), float(np.float32(sc)), int(P)), img, float(ang), bool(fl), randoms=rnd)
        assert (p.Row, p.Col) == (int(o0), int(o1)) and np.float32(p.Scale) == np.float32(o2)
        assert p.Perturbs == 0


def test_puploc_batch_vs_oracle_random_seeds(sample_gray):
    pk = pigo_b200.load_cascade("puploc")
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pk)
    ora = O.OraclePuploc(pk)
    rng = np.random.default_rng(99)
    img = ImageParams(sample_gray, 400, 320, 320)
    for ang in (0.0, 0.33):
        seeds, flips, rnds = [], [], []
        for k in range(40):
            seeds.append(Puploc(int(rng.integers(-5, 405)), int(rng.integers(-5, 325)), float(np.float32(rng.uniform(5, 120))),
                                int(rng.integers(0, 64))))
            flips.append(bool(rng.integers(0, 2)))
            rnds.append(rng.random(189, dtype=np.float32))
        out = plc.run_detector_batch(seeds, img, ang, flips, np.stack(rnds))
        for s, f, r, o in zip(seeds, flips, rnds, out):
            e = ora.run_detector(s.Row, s.Col, s.Scale, s.Perturbs, r, sample_gray, 400, 320, 320, ang, f)
            assert (o.Row, o.Col) == (e[0], e[1]) and np.float32(o.Scale) == e[2]


def test_puploc_perturbs_above_63_is_rejected(sample_gray):
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
    with pytest.raises(pigo_b200.PigoError):   # the reference panics (index out of range on the 63-slot pool)
        plc.RunDetector(Puploc(100, 100, 30.0, 64), ImageParams(sample_gray, 400, 320, 320), 0.0, False)


def test_reference_landmark_assertion_through_the_mirror_api(gpu_face, sample_gray):
    """core/flploc_test.go:75-154 replayed on the GPU path (library RNG): 15 points with Row>0 && Col>0."""
    img = ImageParams(sample_gray, 400, 320, 320)
    dets = gpu_face.RunCascade(cp_of(sample_gray, 400, 320, 320, TEST_PARAMS), 0.0)
    dets = gpu_face.ClusterDetections(dets, 0.1)
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
    flpcs = plc.ReadCascadeDir(pigo_b200.CASCADE_DIR + "/lps")
    n = 0
    for det in dets:
        if det.Scale > 50:
            row = det.Row - int(np.float32(0.075) * np.float32(det.Scale))
            le = plc.RunDetector(Puploc(row, det.Col - int(np.float32(0.175) * np.float32(det.Scale)),
                                        float(np.float32(det.Scale) * np.float32(0.25)), 50), img, 0.0, False, rng_seed=1)
            re_ = plc.RunDetector(Puploc(row, det.Col + int(np.float32(0.185) * np.float32(det.Scale)),
                                         float(np.float32(det.Scale) * np.float32(0.25)), 50), img, 0.0, False, rng_seed=2)
            for eye in ("lp46", "lp44", "lp42", "lp38", "lp312"):
                for flpc in flpcs[eye]:
                    for fl in (False, True):
                        p = flpc.GetLandmarkPoint(le, re_, img, 63, fl, rng_seed=3)
                        n += 1 if (p.Row > 0 and p.Col > 0) else 0
            for mouth in ("lp93", "lp84", "lp82", "lp81"):
                for flpc in flpcs[mouth]:
                    p = flpc.GetLandmarkPoint(le, re_, img, 63, False, rng_seed=4)
                    n += 1 if (p.Row > 0 and p.Col > 0) else 0
            p = flpcs["lp84"][0].GetLandmarkPoint(le, re_, img, 63, True, rng_seed=5)
            n += 1 if (p.Row > 0 and p.Col > 0) else 0
    assert n == 2 * 5 + 4 + 1


def test_get_landmark_point_vs_oracle(sample_gray):
    pk = pigo_b200.load_cascade("lps/lp42")
    flp = pigo_b200.NewPuplocCascade().UnpackCascade(pk)
    ora = O.OraclePuploc(pk)
    img = ImageParams(sample_gray, 400, 320, 320)
    rnd = np.random.default_rng(5).random(189, dtype=np.float32)
    le, re_ = Puploc(186, 118, 0, 0), Puploc(188, 205, 0, 0)
    for fl in (False, True):
        p = flp.GetLandmarkPoint(le, re_, img, 63, fl, randoms=rnd)
        e = P.oracle_landmark(ora, (le.Row, le.Col), (re_.Row, re_.Col), rnd, (sample_gray, 400, 320, 320), fl)
        assert (p.Row, p.Col) == (e[0], e[1]) and np.float32(p.Scale) == e[2]


# ---- scan implementation variants (tiled shared-memory kernel vs gather kernel) ------------------------------
# Each variant names the kernels it runs on one 720p frame (TEST_PARAMS), and the test asserts them: a variant whose kernel
# falls back on this geometry fails rather than testing another path.  "universal": the standalone gather kernel alone;
# "classic" / "head" / "ptab": the fused kernel with that tile role (classic lane refill, dense head, per-scale offset
# tables); "gather": the gather-v2 kernel; "deep": the deep kernel.
VARIANTS = [
    ({"scan_mode": 1}, "universal"),
    ({"scan_mode": 0}, "classic deep"),                                  # default: fused kernel (tile + gather warps) + deep
    ({"scan_mode": 0, "tile_ni": 1, "tile_warps": 4, "tile_ks": 16, "tile_tail_min": 33}, "classic deep"),   # everything spills early
    ({"scan_mode": 0, "tile_ni": 4, "tile_warps": 12, "tile_ks": 128, "tile_tail_min": 0}, "classic deep"),  # nothing spills at tails
    ({"scan_mode": 0, "tile_ni": 3, "tile_warps": 16, "tile_ks": 200, "tile_band_ratio": 130}, "classic gather deep"),   # no room for gather warps
    ({"scan_mode": 0, "tile_max_scale": 30, "chunk": 64}, "classic deep"),
    ({"scan_mode": 0, "gather_warps": 0, "tile_warps": 8, "tile_ni": 2}, "classic gather deep"),   # tiles fused kernel + separate gather launch
    ({"scan_mode": 0, "gather_warps": 24, "tile_warps": 8, "tile_ni": 1, "tile_ks": 32}, "classic deep"),
    ({"scan_mode": 3, "gather_ks": 32, "gather_ni": 1, "sub_batch": 2, "lanes": 2}, "gather deep"),   # gather-v2 + deep kernel only
    ({"scan_mode": 0, "gather_ni": 3, "sub_batch": 1, "lanes": 3}, "classic deep"),
    ({"scan_mode": 0, "deep_group": 32, "tile_ks": 8, "gather_ks": 8}, "classic deep"),
    ({"scan_mode": 0, "tile_tail_min": 33, "tile_ks": 5, "gather_ks": 7}, "classic deep"),
    ({"scan_mode": 0, "gather_block": 8, "tile_prefetch": 1, "deep_group": 16}, "classic deep"),
    ({"scan_mode": 0, "fused_smem_kb": 160, "tile_warps": 14, "gather_warps": 18}, "classic deep"),
    ({"scan_mode": 0, "tile_warps": 4, "gather_warps": 28, "tile_max_scale": 24}, "classic deep"),
    ({"scan_mode": 3, "gather_block": 16, "gather_ni": 2}, "gather deep"),
    ({"scan_mode": 3, "gather_ks": 4}, "gather deep"),                                                  # nearly everything through the deep kernel
    # no room for tiles beside a 446-tree prefix: gather-v2 alone keeps 446 trees resident, the deep kernel walks the last 22
    ({"scan_mode": 0, "gather_ks": 468, "gather_limit": 468, "tile_ks": 468, "tile_warps": 4, "gather_warps": 0}, "gather deep"),
    ({"scan_mode": 0, "deep_flat": 1, "deep_group": 8, "tile_ks": 6}, "classic deep"),                   # flat deep loop, lots of Q2 traffic
    ({"scan_mode": 3, "deep_flat": 1, "deep_group": 16, "gather_ks": 3}, "gather deep"),
    ({"scan_mode": 0, "tile_head": 2, "tile_warps": 22}, "head deep"),                                   # dense head over trees 0..1, ring + generic tail
    ({"scan_mode": 0, "tile_head": 1, "tile_warps": 24, "head_back": 1}, "head deep"),
    ({"scan_mode": 0, "tile_ptab": 1}, "ptab deep"),                                                     # per-scale offset tables, scale-synchronous rounds
    ({"scan_mode": 0, "tile_ptab": 1, "ptab_kt": 4, "ptab_ks": 6, "tile_warps": 7, "gather_warps": 3}, "ptab deep"),
    ({"scan_mode": 0, "tile_ptab": 1, "ptab_kt": 468, "tile_tail_min": 33, "tile_warps": 12}, "ptab deep"),   # capped at 60 trees; every drained tile spills
    ({"scan_mode": 0, "tile_ptab": 1, "ptab_kt": 5, "tile_tail_min": 0, "gather_warps": 0, "tile_warps": 16}, "ptab gather deep"),
    ({"scan_mode": 0, "tile_ptab": 1, "ptab_kt": 1, "tile_max_scale": 30, "tile_band_ratio": 110}, "ptab deep"),   # many narrow bands
    ({"scan_mode": 0, "queue_cap": 40, "tile_ks": 4, "gather_ks": 6, "tile_tail_min": 33}, "classic deep"),   # both queues overflow: producers finish their windows in place
    ({"scan_mode": 0, "queue_cap": 7, "tile_ptab": 1, "ptab_kt": 3, "ptab_ks": 5, "tile_tail_min": 33}, "ptab deep"),
    ({"scan_mode": 3, "queue_cap": 16, "gather_ks": 2}, "gather deep"),
    ({"scan_mode": 0, "deep_smem": 1, "deep_smem_k": 468, "deep_smem_lo": 0}, "classic deep"),          # deep kernel, tree records in shared memory
    ({"scan_mode": 0, "deep_smem": 1, "deep_group": 4, "gather_limit": 4, "tile_ks": 6, "deep_smem_threads": 512, "deep_smem_k": 30, "deep_smem_lo": 11},
     "classic deep"),                                                                                    # + entries below its first resident tree
    ({"scan_mode": 3, "deep_smem": 1, "deep_group": 32, "gather_ks": 3, "deep_smem_threads": 256}, "gather deep"),
    # everything spills, tiny prefix (tile_max_scale keeps the tiled ladder within the head's 16 table slots)
    ({"scan_mode": 0, "tile_head": 3, "tile_warps": 6, "tile_ks": 5, "head_back": 16, "tile_tail_min": 33, "tile_max_scale": 60}, "head deep"),
    ({"scan_mode": 0, "tile_head": 4, "tile_warps": 12, "tile_ks": 63, "gather_warps": 0, "tile_tail_min": 0}, "head gather deep"),
    ({"scan_mode": 0, "tile_head": 2, "tile_ks": 2}, "classic deep"),                                   # prefix not longer than the head: classic kernel
]


def run_timed(fn):
    """fn() with per-kernel timing on; returns its result and the launch counts of the fused, gather and deep kernel slots."""
    with options(timing=1):
        out = fn()
        launches = {k: pigo_b200.get_option(k) for k in ("t_tiled_n", "t_gather_n", "t_deep_n")}
    return out, launches


def assert_kernels(expect: str, launches: dict, rows, cols, prm, nframes, groups=1):
    """The launches of one call (of `groups` pipeline groups) are the kernels `expect` names, and the fused kernel's tile role
    is the one the planner picks for the call (describe_plan with the call's frame count)."""
    k = expect.split()
    role = next((r for r in k if r in ("classic", "head", "ptab")), None)
    want = {"t_tiled_n": groups * (role is not None), "t_gather_n": groups * ("gather" in k or "universal" in k), "t_deep_n": groups * ("deep" in k)}
    assert launches == want, f"expected {expect}"
    if role is not None:
        p = pigo_b200.describe_plan(rows, cols, *prm, nframes=nframes)
        assert ("head" if p["head"] else "ptab" if p["ptab_kt"] else "classic") == role, p


@pytest.mark.parametrize("variant,expect", VARIANTS, ids=[f"variant{i}" for i in range(len(VARIANTS))])
def test_scan_variants_agree_with_oracle(gpu_face, oracle_face, sample_gray, variant, expect):
    frames = synth.make_batch(3, 720, 1280, "SFU", seed0=21)
    cases = [(frames[0], 720, 1280, 1280, TEST_PARAMS), (frames[1], 720, 1280, 1280, DOC_PARAMS),
             (frames[2], 720, 1280, 1280, CLI_PARAMS), (sample_gray, 400, 320, 320, (20, 1000, 0.05, 1.05))]
    with options(**variant):
        _, launches = run_timed(lambda: gpu_face.run_cascade_array(cp_of(frames[0], 720, 1280, 1280, TEST_PARAMS), 0.0))
        assert_kernels(expect, launches, 720, 1280, TEST_PARAMS, 1)
        for img, r, c, d, prm in cases:
            g = gpu_face.run_cascade_array(cp_of(img, r, c, d, prm), 0.0)
            assert_same(g, oracle_face.run_cascade(img, r, c, d, *prm, 0.0))
        # unaligned stride (Dim % 16 != 0) takes the byte-wise tile fill
        buf = np.zeros((301, 523), dtype=np.uint8)
        buf[:, :500] = synth.frame_faces(None, 301, 500, shift=(3, 1), noise_seed=8)
        g = gpu_face.run_cascade_array(cp_of(buf, 301, 500, 523, TEST_PARAMS), 0.0)
        assert_same(g, oracle_face.run_cascade(buf, 301, 500, 523, *TEST_PARAMS, 0.0))
        # batch with the deep queue shared by several frames
        dets, cnt = gpu_face.RunCascadeBatch(frames, cp_of(None, 720, 1280, 1280, TEST_PARAMS), 0.0, cap_per_frame=512)
    for f in range(3):
        o = oracle_face.run_cascade(frames[f], 720, 1280, 1280, *TEST_PARAMS, 0.0)
        assert cnt[f] == len(o) and dets[f, :cnt[f]].tobytes() == o.tobytes()
        assert not np.frombuffer(dets[f, cnt[f]:].tobytes(), dtype=np.uint8).any()   # padding past the count is zero, not stale


def test_cpp_mirror_replays_reference_test():
    """include/pigo_b200.hpp (C++ mirror of the Go API) -> C-ABI -> GPU: core/pigo_test.go:68-84 on the sample image."""
    assert "dets=4 clusters=1" in run_cpp_mirror("test_mirror", timeout=120)


def test_full_pipeline_batch_vs_oracle(gpu_face, oracle_face, sample_gray, cascades):
    """BASELINE.json configs[4] shape: face -> cluster -> 2 pupils -> 15 landmarks per face, per frame of a batch,
    replayed on the CPU oracle with the same injected randoms (sequencing of core/flploc_test.go:75-154)."""
    from pigo_b200 import pipeline
    frames = np.stack([synth.frame_faces(sample_gray, 540, 960, shift=(40 * i, 25 * i), noise_seed=30 + i) for i in range(3)])
    cp = cp_of(None, 540, 960, 960, TEST_PARAMS)
    plc, flp, _, _ = cascades

    def randoms_for(f, call):
        return np.random.default_rng(10_000 * f + call).random((63, 3), dtype=np.float32)

    got = pipeline.detect_batch(gpu_face, plc, flp, frames, cp, iou=0.1, randoms_for=randoms_for)
    images = [(frames[f], 540, 960, 960) for f in range(3)]
    cls = [P.oracle_clusters(oracle_face, im, TEST_PARAMS, 0.0) for im in images]

    def randoms(f, k, slot):   # calls are numbered in sequence within a frame, 2 + 15 per refined face
        return randoms_for(f, int((cls[f]["scale"][:k] > 50).sum()) * (2 + len(pipeline.landmark_calls())) + slot)

    nfaces, _ = P.replay(cascades[2:], [(f, images[f], cls[f], 0.0) for f in range(3)], randoms, 50, P.face_arrays(got))
    assert nfaces >= 3


def test_rgb_to_grayscale_matches_oracle():
    """core/grayscale.go:8-23 on NRGBA pixels (section 8f row N2): float64 luma of the 16-bit expanded, alpha-premultiplied
    channels, truncated to uint8 -- bit-exact against both CPU restatements, opaque and translucent pixels, ragged sizes."""
    rng = np.random.default_rng(4)
    for shape in [(1080, 1920), (37, 53), (1, 1), (3, 5)]:
        rgba = rng.integers(0, 256, size=shape + (4,), dtype=np.uint8)
        if shape[0] > 100:
            rgba[..., 3] = 255
        g = pigo_b200.RgbToGrayscale(rgba)
        assert g.shape == shape and g.dtype == np.uint8
        assert np.array_equal(g, O.rgba_to_gray(rgba))
    assert pigo_b200.RgbToGrayscale(np.zeros((0, 0, 4), np.uint8)).size == 0


def test_concurrent_calls_on_one_classifier(gpu_face, oracle_face):
    """The reference's methods are re-entrant on a shared classifier (read-only tables, pooled scratch); so is the C-ABI:
    several OS threads call RunCascade on the same handle at once (ctypes releases the GIL during the call)."""
    import threading
    frames = synth.make_batch(6, 480, 640, "SFU", seed0=77)
    expect = [oracle_face.run_cascade(frames[i], 480, 640, 640, *TEST_PARAMS, 0.0) for i in range(6)]
    errors = []

    def work(i):
        try:
            for _ in range(5):
                g = gpu_face.run_cascade_array(cp_of(frames[i], 480, 640, 640, TEST_PARAMS), 0.0)
                if g.tobytes() != expect[i].tobytes():
                    errors.append(i)
        except Exception as e:   # noqa: BLE001
            errors.append(repr(e))

    ts = [threading.Thread(target=work, args=(i,)) for i in range(6)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert errors == []


def test_device_resident_async_api_matches_host_api(gpu_face, oracle_face):
    """pigo_run_cascade_batch with PIGO_FRAMES_DEVICE|PIGO_OUT_DEVICE on a caller stream (what bench.py times)."""
    import torch
    frames = synth.make_batch(5, 540, 960, "FSU", seed0=5)
    d = torch.from_numpy(frames).cuda()
    cap = 256
    out = torch.zeros((5, cap, 4), dtype=torch.int32, device="cuda")
    cnt = torch.zeros(5, dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for _ in range(2):   # back-to-back asynchronous calls reuse the same workspace
            gpu_face.run_cascade_batch_device(d.data_ptr(), 5, 540 * 960, 540, 960, 960, *TEST_PARAMS, 0.0, out.data_ptr(), cap,
                                              cnt.data_ptr(), st.cuda_stream)
    st.synchronize()
    o = out.cpu().numpy().view(np.uint8).reshape(5, cap, 16)
    for f in range(5):
        e = oracle_face.run_cascade(frames[f], 540, 960, 960, *TEST_PARAMS, 0.0)
        assert int(cnt[f]) == len(e)
        assert o[f, :len(e)].tobytes() == e.tobytes()


@pytest.mark.parametrize("depth,ntrees", [(6, 3), (6, 70), (4, 9), (1, 2), (8, 5), (6, 1)])
def test_synthetic_cascades_other_depths_and_sizes(depth, ntrees):
    """Generic tree depth (universal gather kernel) and tiny / odd-sized depth-6 cascades (resident prefix larger than the
    cascade, Q2 never used, ...), unrotated and rotated."""
    pk = synthetic_cascade(depth, ntrees, seed=depth * 100 + ntrees)
    clf = pigo_b200.NewPigo().Unpack(pk)
    ora = O.OracleFace(pk)
    assert (clf.treeDepth, clf.treeNum) == (depth, ntrees) == (ora.depth, ora.ntrees)
    img = synth.frame_smooth(300, 420, seed=depth + ntrees, sigma=3.0)
    for ang in (0.0, 0.4):
        for prm in ((20, 200, 0.2, 1.2), (24, 60, 0.1, 1.1)):
            g = clf.run_cascade_array(cp_of(img, 300, 420, 420, prm), ang, cap=64)
            o = ora.run_cascade(img, 300, 420, 420, *prm, ang, cap=1 << 18)
            assert_same(g, o)


def test_rotated_very_wide_frame_uses_64bit_coordinates(gpu_face, oracle_face):
    """cols > 32767: 65536*col no longer fits 31 bits, the rotated kernel must fall back to 64-bit coordinates (Go's int)."""
    img = synth.frame_noise(48, 33000, seed=12)
    img[:, ::7] //= 3
    for a in (0.3, 0.8):
        g = gpu_face.run_cascade_array(cp_of(img, 48, 33000, 33000, (20, 40, 0.2, 1.2)), a)
        assert_same(g, oracle_face.run_cascade(img, 48, 33000, 33000, 20, 40, 0.2, 1.2, a))
    g = gpu_face.run_cascade_array(cp_of(img, 48, 33000, 33000, (20, 40, 0.2, 1.2)), 0.0)
    assert_same(g, oracle_face.run_cascade(img, 48, 33000, 33000, 20, 40, 0.2, 1.2, 0.0))


# ================================================================================================================
# round 2
# ================================================================================================================
@pytest.fixture(scope="module")
def frame_4k():
    return synth.frame_faces(None, 2160, 3840, shift=(5, 9), noise_seed=4)


@pytest.mark.parametrize("k", list(range(1, 33)))
def test_4k_rotated_every_table_slot(gpu_face, oracle_face, frame_4k, k):
    """BASELINE configs[3]: 3840x2160, a = k/32 for EVERY table slot (core/pigo.go:156-160); the table-driven block/deep
    kernels against the oracle, integer-exact and in emission order."""
    g = gpu_face.run_cascade_array(cp_of(frame_4k, 2160, 3840, 3840, TEST_PARAMS), k / 32.0)
    assert_same(g, oracle_face.run_cascade(frame_4k, 2160, 3840, 3840, *TEST_PARAMS, k / 32.0))


ROTATED_VARIANTS = [
    ({"rot_mode": 1}, "universal"),
    ({"rot_mode": 0, "gather_ks": 4, "deep_group": 8}, "gather deep"),
    ({"rot_mode": 0, "gather_ni": 2, "deep_group": 16}, "gather deep"),
    ({"rot_mode": 0, "gather_ks": 468, "gather_limit": 468, "deep_group": 32}, "gather deep"),   # 446 trees resident, the deep kernel walks the last 22
    ({"rot_mode": 0, "gather_block": 8, "sub_batch": 1}, "gather deep"),
]


@pytest.mark.parametrize("variant,expect", ROTATED_VARIANTS, ids=[f"variant{i}" for i in range(len(ROTATED_VARIANTS))])
def test_rotated_kernel_variants(gpu_face, oracle_face, sample_gray, variant, expect):
    """Universal gather kernel vs table-driven kernels (gather-v2 + deep), tiny / longest resident prefix."""
    wide = synth.frame_faces(sample_gray, 300, 900, noise_seed=1)       # cols > rows: the nrows-1 column clamp bites
    tall = synth.frame_faces(sample_gray, 700, 260, noise_seed=2)
    frames = synth.make_batch(3, 360, 640, "FSU", seed0=41)
    with options(**variant):
        _, launches = run_timed(lambda: gpu_face.run_cascade_array(cp_of(sample_gray, 400, 320, 320, TEST_PARAMS), 0.26))
        assert_kernels(expect, launches, 400, 320, TEST_PARAMS, 1)
        for img, r, c in ((sample_gray, 400, 320), (wide, 300, 900), (tall, 700, 260)):
            for a in (1 / 32.0, 0.26, 0.5, 0.77, 1.0):
                g = gpu_face.run_cascade_array(cp_of(img, r, c, c, TEST_PARAMS), a)
                assert_same(g, oracle_face.run_cascade(img, r, c, c, *TEST_PARAMS, a))
        dets, cnt = gpu_face.RunCascadeBatch(frames, cp_of(None, 360, 640, 640, DOC_PARAMS), 0.4, cap_per_frame=64)
    for f in range(3):
        o = oracle_face.run_cascade(frames[f], 360, 640, 640, *DOC_PARAMS, 0.4)
        assert cnt[f] == len(o) and dets[f, :cnt[f]].tobytes() == o.tobytes()


def test_min_size_zero_is_a_valid_ladder(gpu_face, oracle_face):
    """MinSize 0: scale 0 gives step 1, offset 1 and every node compares a pixel with itself (core/pigo.go:226-231); the
    reference handles it, so does the library (ADVICE round 1).  Negative sizes are rejected (the reference indexes out of bounds)."""
    img = np.random.default_rng(3).integers(0, 256, size=(40, 50), dtype=np.uint8)
    for prm in ((0, 30, 0.1, 1.3), (0, 0, 0.2, 1.1), (1, 9, 0.5, 1.5)):
        g = gpu_face.run_cascade_array(cp_of(img, 40, 50, 50, prm), 0.0, cap=16)
        assert_same(g, oracle_face.run_cascade(img, 40, 50, 50, *prm, 0.0))
        assert pigo_b200.count_windows(40, 50, *prm) == O.count_windows(40, 50, *prm)
    with pytest.raises(pigo_b200.PigoError):
        gpu_face.run_cascade_array(cp_of(img, 40, 50, 50, (-4, 30, 0.1, 1.3)), 0.0)


def test_host_frames_with_tight_stride_and_short_last_frame(gpu_face, oracle_face):
    """Dim > Cols with the frames packed (rows-1)*Dim + Cols bytes apart -- the smallest buffer the reference can index
    (ADVICE round 1: the host path must not read rows*dim bytes per frame, and the 2-D copy must accept the tight pitch)."""
    rows, cols, dim, nf = 120, 150, 160, 5
    tight = (rows - 1) * dim + cols
    buf = np.zeros(nf * tight, dtype=np.uint8)
    imgs = []
    for f in range(nf):
        full = np.zeros((rows, dim), dtype=np.uint8)
        full[:, :cols] = synth.frame_faces(None, rows, cols, shift=(7 * f, 3 * f), noise_seed=60 + f)
        flat = full.reshape(-1)[:tight]
        buf[f * tight:(f + 1) * tight] = flat
        imgs.append(flat.copy())
    import ctypes as C
    cap = 256
    out = np.zeros((nf, cap), dtype=pigo_b200.DET_DTYPE)
    cnt = np.zeros(nf, dtype=np.int32)
    prm = (20, 100, 0.1, 1.1)
    rc = pigo_b200.lib().pigo_run_cascade_batch(gpu_face._h, buf.ctypes.data, nf, tight, rows, cols, dim, prm[0], prm[1], prm[2], prm[3], 0.0,
                                                out.ctypes.data, cap, cnt.ctypes.data, 0, None)
    assert rc == 0, pigo_b200.lib().pigo_last_error()
    for f in range(nf):
        padded = np.zeros(rows * dim, dtype=np.uint8)
        padded[:tight] = imgs[f]
        o = oracle_face.run_cascade(padded, rows, cols, dim, *prm, 0.0)
        assert cnt[f] == len(o) and out[f, :cnt[f]].tobytes() == o.tobytes()


# (options, kernels of the unrotated 11-frame call, pipeline groups of that call)
HOST_STREAM_VARIANTS = [
    ({"host_stream": 0}, "classic deep", 1),
    ({"host_stream": 1, "copy_chunk": 1, "sub_batch": 4}, "classic deep", 3),
    ({"host_stream": 1, "copy_chunk": 3}, "classic deep", 1),
    ({"host_stream": 1, "copy_chunk": 100, "deep_flat": 1}, "classic deep", 1),
    ({"host_stream": 1, "scan_mode": 3}, "gather deep", 1),
    ({"host_stream": 1, "tile_warps": 0}, "gather deep", 1),    # no tile warps: the fused kernel does not run
]


@pytest.mark.parametrize("variant,expect,groups", HOST_STREAM_VARIANTS, ids=[f"variant{i}" for i in range(len(HOST_STREAM_VARIANTS))])
def test_host_frames_streamed_behind_the_copy(gpu_face, oracle_face, variant, expect, groups):
    """Host frames: the scan kernels start at once and wait in-kernel for each frame's copy chunk (ready counter); the result
    must not depend on the chunking, the grouping, or on whether the polling fused kernel runs at all for the geometry."""
    frames = synth.make_batch(11, 270, 480, "USF", seed0=77)
    tiny = synth.make_batch(3, 30, 40, "UUU", seed0=2)      # no tileable band: the fused kernel does not run
    with options(**variant):
        for ang in (0.0, 0.3):
            (dets, cnt), launches = run_timed(lambda: gpu_face.RunCascadeBatch(frames, cp_of(None, 270, 480, 480, TEST_PARAMS), ang, cap_per_frame=128))
            if ang == 0.0:
                assert_kernels(expect, launches, 270, 480, TEST_PARAMS, 11, groups)
            for f in range(11):
                o = oracle_face.run_cascade(frames[f], 270, 480, 480, *TEST_PARAMS, ang)
                assert cnt[f] == len(o) and dets[f, :cnt[f]].tobytes() == o.tobytes()
        dets, cnt = gpu_face.RunCascadeBatch(tiny, cp_of(None, 30, 40, 40, (20, 30, 0.1, 1.1)), 0.0, cap_per_frame=64)
    for f in range(3):
        o = oracle_face.run_cascade(tiny[f], 30, 40, 40, 20, 30, 0.1, 1.1, 0.0)
        assert cnt[f] == len(o) and dets[f, :cnt[f]].tobytes() == o.tobytes()


@pytest.mark.parametrize("mode,stage", [(0, 2), (0, 1), (0, 0), (1, 0)])
def test_puploc_kernels_agree_with_oracle(sample_gray, mode, stage):
    """Both RunDetector kernels ((perturbation, tree)-pair kernel and warp-per-perturbation kernel), rotated and not,
    flips, Perturbs 0..63, seeds near and beyond the image border, on a frame batch."""
    with options(puploc_mode=mode, puploc_stage=stage):
        _puploc_kernels_agree_with_oracle(sample_gray)


def _puploc_kernels_agree_with_oracle(sample_gray):
    rng = np.random.default_rng(123)
    frames = np.stack([sample_gray, np.roll(sample_gray, 13, axis=1), 255 - sample_gray])
    for pkname in ("puploc", "lps/lp93"):
        pk = pigo_b200.load_cascade(pkname)
        plc = pigo_b200.NewPuplocCascade().UnpackCascade(pk)
        ora = O.OraclePuploc(pk)
        for ang in (0.0, 0.2, 0.93):
            seeds, flips, rnds, sfr = [], [], [], []
            for k in range(30):
                seeds.append(Puploc(int(rng.integers(-20, 420)), int(rng.integers(-20, 340)), float(np.float32(rng.uniform(2, 300))),
                                    int(rng.integers(0, 64))))
                flips.append(bool(rng.integers(0, 2)))
                rnds.append(rng.random(189, dtype=np.float32))
                sfr.append(int(rng.integers(0, 3)))
            out = plc.run_detector_frames(seeds, sfr, frames, 3, 400 * 320, 400, 320, 320, ang, flips, np.stack(rnds))
            for s, f, r, fr, o in zip(seeds, flips, rnds, sfr, out):
                e = ora.run_detector(s.Row, s.Col, s.Scale, s.Perturbs, r, frames[fr], 400, 320, 320, ang, f)
                assert (o.Row, o.Col) == (e[0], e[1]) and np.float32(o.Scale) == e[2]


@pytest.mark.parametrize("angle,stage", [(0.0, 1), (0.03, 1), (0.0, 2), (0.03, 2)])
def test_device_pipeline_vs_oracle(gpu_face, oracle_face, sample_gray, cascades, angle, stage):
    """pigo_detect_batch (SURVEY.md 8f N1): the whole face -> cluster -> eye seeds -> RunDetector x2 -> landmark seeds ->
    15 x RunDetector sequence on the device in one call, replayed step by step on the CPU oracle with the same injected
    randoms (core/flploc_test.go:75-154; angle > 0 like cmd/pigo/main.go:422 passes det.angle to the eye RunDetector)."""
    from pigo_b200 import pipeline
    plc, flp, _, _ = cascades
    frames = np.stack([synth.frame_faces(sample_gray, 540, 960, shift=(40 * i, 25 * i), noise_seed=30 + i) for i in range(3)] +
                      [synth.frame_noise(540, 960, 5)])
    cp = cp_of(None, 540, 960, 960, TEST_PARAMS)
    face_cap = 24
    randoms = np.random.default_rng(8).random((4, face_cap, 17, 63, 3), dtype=np.float32)
    with options(puploc_stage=stage):
        got = pipeline.detect_batch_device(gpu_face, plc, flp, frames, cp, iou=0.1, face_cap=face_cap, randoms=randoms, angle=angle)
        # resident frames give the same answer
        df = pigo_b200.DeviceFrames(frames)
        try:
            got2 = pipeline.detect_batch_device(gpu_face, plc, flp, df, cp, iou=0.1, face_cap=face_cap, randoms=randoms, angle=angle)
        finally:
            df.free()
    images = [(frames[f], 540, 960, 960) for f in range(4)]
    cls = [P.oracle_clusters(oracle_face, im, TEST_PARAMS, angle) for im in images]
    assert all(len(cl) <= face_cap for cl in cls)
    n, _ = P.replay(cascades[2:], [(f, images[f], cls[f], angle) for f in range(4)], lambda f, k, slot: randoms[f, k, slot], 50, P.face_arrays(got))
    assert n >= 3 or angle > 0
    assert got[3] == [] or all(fc.left_eye is None or fc.det[2] > 50 for fc in got[3])
    assert got2 == got


def test_device_pipeline_capacity_and_rng_mode(gpu_face, sample_gray, cascades):
    """face_cap / det_cap too small -> PIGO_E_CAP (with the required count); library generator: deterministic, and
    independent of how the batch is split (keys are (seed, frame, cluster, call))."""
    from pigo_b200 import pipeline
    plc, flp, _, _ = cascades
    frames = np.stack([synth.frame_faces(sample_gray, 540, 960, shift=(11 * i, 7 * i), noise_seed=90 + i) for i in range(4)])
    cp = cp_of(None, 540, 960, 960, TEST_PARAMS)
    with pytest.raises(pigo_b200.PigoError) as e:
        pipeline.detect_batch_device(gpu_face, plc, flp, frames, cp, face_cap=1)
    assert e.value.status == pigo_b200.PIGO_E_CAP
    with pytest.raises(pigo_b200.PigoError) as e:
        pipeline.detect_batch_device(gpu_face, plc, flp, frames, cp, face_cap=16, det_cap=2)
    assert e.value.status == pigo_b200.PIGO_E_CAP
    a = pipeline.detect_batch_device(gpu_face, plc, flp, frames, cp, face_cap=16, rng_seed=5, raw=True)
    b = pipeline.detect_batch_device(gpu_face, plc, flp, frames, cp, face_cap=16, rng_seed=5, raw=True)
    c = pipeline.detect_batch_device(gpu_face, plc, flp, frames, cp, face_cap=16, rng_seed=6, raw=True)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    assert a[0].tobytes() == c[0].tobytes() and a[2].tobytes() != c[2].tobytes()
    assert (a[2]["row"][a[0]["scale"] > 50] > 0).all()
    # sharded entry point (one device selected: same code path as N devices, shard 0 only)
    pigo_b200.init_devices(1)
    s = pipeline.detect_batch_device(gpu_face, plc, flp, frames, cp, face_cap=16, rng_seed=5, raw=True, sharded=True)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, s))


def test_sharded_scan_matches_single_device(gpu_face, oracle_face):
    """pigo_run_cascade_batch_sharded over every visible device (1 on a single-GPU machine, 2+ on a multi-GPU one):
    frame shards, replicas built on first use, results in frame order == the per-frame oracle."""
    n = pigo_b200.device_count()
    pigo_b200.init_devices((1 << n) - 1)
    try:
        frames = synth.make_batch(7, 360, 640, "FUS", seed0=14)
        dets, cnt = gpu_face.RunCascadeBatchSharded(frames, cp_of(None, 360, 640, 640, TEST_PARAMS), 0.0, cap_per_frame=2)   # forces the retry
        for f in range(7):
            o = oracle_face.run_cascade(frames[f], 360, 640, 640, *TEST_PARAMS, 0.0)
            assert cnt[f] == len(o) and dets[f, :cnt[f]].tobytes() == o.tobytes()
    finally:
        pigo_b200.init(0)


@pytest.mark.parametrize("subsample", [0, 1, 2, 3, 4, 5])
def test_ycbcr_to_nrgba_matches_oracle(subsample):
    """ImgToNRGBA for *image.YCbCr (core/image.go:60-76, section 8f N3): bit-exact against the restated Go conversion for the six
    subsample ratios of core/image_test.go:21-57, non-zero rectangle origin, strides wider than the planes; fused gray =
    RgbToGrayscale of the converted image."""
    for (w, h, mx, my) in ((16, 16, 0, 0), (37, 21, 0, 0), (33, 18, 3, 5), (1920, 1080, 0, 0)):
        y, cb, cr = O.make_ycbcr_planes(100 * subsample + w, subsample, w, h, mx, my)
        got, gray = pigo_b200.YCbCrToNRGBA(y, cb, cr, subsample, w, h, mx, my, want_gray=True)
        exp = O.ycbcr_to_nrgba(y, cb, cr, subsample, w, h, mx, my)
        assert np.array_equal(got, exp)
        assert np.array_equal(gray, O.rgba_to_gray(exp))


def test_cpp_sharded_over_every_visible_device():
    """tests/cpp/test_sharded.cpp: one process drives every visible GPU through include/pigo_b200.h (pigo_init_devices,
    pigo_run_cascade_batch_sharded, pigo_detect_batch_sharded) and requires byte-identical results to the 1-GPU calls.
    With one GPU this exercises the same code with a single shard; on a machine with two GPUs it is the 2-device test."""
    import os
    out = run_cpp_mirror("test_sharded")
    assert "== single device" in out
    need = int(os.environ.get("PIGO_REQUIRE_DEVICES", "1"))
    assert int(out.split("devices=")[1].split()[0]) >= need


# ---------------------------------------------------------------------------------------------------------------
# Randomised geometry / parameter fuzz and full-size (BASELINE configs[2]) properties
# ---------------------------------------------------------------------------------------------------------------
def _fuzz_case(rng, sample_gray, case):
    """One random call.  Half of the cases are built to produce survivors: the reference's sample face (rotated by the call's
    angle, so that the rotated scan finds it) inside a frame large enough to hold it, MaxSize 1000."""
    from scipy import ndimage
    ang = float(rng.choice([0.0, 0.0, rng.uniform(0.01, 1.2)]))
    shift = float(rng.choice([0.03, 0.05, 0.1, 0.15, 0.2, 0.33, 1.0]))
    scale = float(rng.choice([1.03, 1.05, 1.1, 1.15, 1.3, 2.0]))
    kind = int(rng.choice([0, 1, 1, 1, 2]))
    if kind == 1:
        rows, cols = int(rng.integers(400, 520)), int(rng.integers(320, 560))
        mn, mx = int(rng.choice([20, 24, 50, 100])), 1000
        face = sample_gray if ang == 0.0 else ndimage.rotate(sample_gray, min(ang, 1.0) * 360.0, reshape=False, order=1, mode="nearest").astype(np.uint8)
        img = rng.integers(0, 256, (rows, cols), dtype=np.uint8)
        r0, c0 = int(rng.integers(0, rows - 400 + 1)), int(rng.integers(0, cols - 320 + 1))
        img[r0:r0 + 400, c0:c0 + 320] = face
        shift = min(shift, 0.2)
        scale = min(scale, 1.3)
    else:
        rows, cols = int(rng.integers(24, 420)), int(rng.integers(24, 520))
        mn = int(rng.choice([0, 1, 7, 20, 20, 24, 33]))
        mx = int(rng.choice([mn, mn + 5, 60, 150, 1000]))
        if kind == 0:
            img = rng.integers(0, 256, (rows, cols), dtype=np.uint8)
        else:
            img = np.full((rows, cols), int(rng.integers(0, 256)), dtype=np.uint8)   # flat: every comparison is a tie
    dim = cols + int(rng.choice([0, 0, 1, 3, 16, 37]))
    buf = np.zeros((rows, dim), dtype=np.uint8)
    buf[:, :cols] = img
    return buf, rows, cols, dim, (mn, mx, shift, scale), ang, kind


def test_random_geometry_and_parameter_fuzz(gpu_face, oracle_face, sample_gray):
    """40 random calls: frame size, stride, MinSize/MaxSize, ShiftFactor, ScaleFactor, angle and content drawn at random;
    every one bit-equal to the oracle (core/pigo.go:212-258 incl. the ladder's float64 truncations)."""
    rng = np.random.default_rng(20260923)
    total = 0
    for case in range(40):
        buf, rows, cols, dim, prm, ang, kind = _fuzz_case(rng, sample_gray, case)
        g = gpu_face.run_cascade_array(cp_of(buf, rows, cols, dim, prm), ang)
        o = oracle_face.run_cascade(buf, rows, cols, dim, *prm, ang)
        assert len(g) == len(o) and g.tobytes() == o.tobytes(), f"case {case}: {rows}x{cols} dim {dim} {prm} angle {ang} kind {kind}"
        total += len(o)
    assert total > 100   # the fuzz must exercise survivors (score bits), not only rejections


def test_full_size_batch_properties(gpu_face, oracle_face):
    """BASELINE configs[2] at full size (256 x 1080p, the bench workload): size-independent properties of the batch entry points.
    (i) sampled frames equal the oracle; (ii) host frames streamed behind the copy == the same frames resident on the device,
    byte for byte over all 256 frames; (iii) frames are independent: reversing the batch reverses the result; (iv) the README
    parameters (4.1 M windows per frame) on one frame equal the oracle."""
    import torch
    nf, R, C = 256, 1080, 1920
    base = synth.make_batch(12, R, C, "USF")
    frames = np.concatenate([base] * ((nf + 11) // 12))[:nf]
    cp = cp_of(None, R, C, C, TEST_PARAMS)
    cap = 256
    host_dets, host_cnt = gpu_face.RunCascadeBatch(frames, cp, 0.0, cap_per_frame=cap)      # host frames (streamed copy)
    assert int(host_cnt.max()) <= cap
    for f in (0, 1, 2, 100, 255):                                                           # (i)
        o = oracle_face.run_cascade(frames[f], R, C, C, *TEST_PARAMS, 0.0)
        assert host_cnt[f] == len(o) and host_dets[f, :host_cnt[f]].tobytes() == o.tobytes()
    d = torch.from_numpy(frames).cuda()
    d_out = torch.zeros((nf, cap, 4), dtype=torch.int32, device="cuda")
    d_cnt = torch.zeros(nf, dtype=torch.int32, device="cuda")
    gpu_face.run_cascade_batch_device(d.data_ptr(), nf, R * C, R, C, C, *TEST_PARAMS, 0.0, d_out.data_ptr(), cap, d_cnt.data_ptr())
    torch.cuda.synchronize()
    dev_cnt = d_cnt.cpu().numpy()
    dev_dets = d_out.cpu().numpy().view(np.uint8).reshape(nf, cap * 16)
    assert (dev_cnt == host_cnt[:nf]).all()                                                 # (ii)
    hb = np.ascontiguousarray(host_dets).view(np.uint8).reshape(nf, cap * 16)
    for f in range(nf):
        assert hb[f, :16 * host_cnt[f]].tobytes() == dev_dets[f, :16 * dev_cnt[f]].tobytes()
    d_rev = torch.flip(d, dims=[0]).contiguous()                                            # (iii)
    d_out.zero_(); d_cnt.zero_()
    gpu_face.run_cascade_batch_device(d_rev.data_ptr(), nf, R * C, R, C, C, *TEST_PARAMS, 0.0, d_out.data_ptr(), cap, d_cnt.data_ptr())
    torch.cuda.synchronize()
    rev_cnt = d_cnt.cpu().numpy()
    rev_dets = d_out.cpu().numpy().view(np.uint8).reshape(nf, cap * 16)
    assert (rev_cnt[::-1] == dev_cnt).all()
    for f in range(nf):
        assert rev_dets[nf - 1 - f, :16 * dev_cnt[f]].tobytes() == dev_dets[f, :16 * dev_cnt[f]].tobytes()
    # every frame of the batch is one of 12 distinct images: equal images must give equal results (a checksum of checksums)
    for f in range(12, nf):
        assert dev_cnt[f] == dev_cnt[f % 12] and dev_dets[f, :16 * dev_cnt[f]].tobytes() == dev_dets[f % 12, :16 * dev_cnt[f]].tobytes()
    del d, d_rev, d_out, d_cnt
    g = gpu_face.run_cascade_array(cp_of(frames[2], R, C, C, DOC_PARAMS), 0.0)               # (iv)
    assert_same(g, oracle_face.run_cascade(frames[2], R, C, C, *DOC_PARAMS, 0.0))


def test_full_turn_equals_unrotated_scan_where_the_clamp_is_idle(gpu_face, oracle_face):
    """SURVEY config 4: angle 32/32 has qcos = 256, qsin = 0, i.e. the unrotated sample points -- so on a frame that is at least as
    tall as wide (the rotated path clamps COLUMNS with nrows-1, core/pigo.go:168,171) RunCascade(angle 1.0) == RunCascade(angle 0),
    detection for detection and bit for bit; on a wide frame the clamp quirk makes them differ, and both agree with the oracle."""
    tall = synth.frame_faces(None, 2160, 1600, shift=(11, 5), noise_seed=4)
    a0 = gpu_face.run_cascade_array(cp_of(tall, 2160, 1600, 1600, TEST_PARAMS), 0.0)
    a1 = gpu_face.run_cascade_array(cp_of(tall, 2160, 1600, 1600, TEST_PARAMS), 1.0)
    assert len(a0) > 20 and a0.tobytes() == a1.tobytes()
    a2 = gpu_face.run_cascade_array(cp_of(tall, 2160, 1600, 1600, TEST_PARAMS), 7.5)     # angle > 1 is clamped to 1 (:233-235)
    assert a2.tobytes() == a1.tobytes()
    wide = synth.frame_faces(None, 600, 1900, shift=(3, 9), noise_seed=5)
    w0 = gpu_face.run_cascade_array(cp_of(wide, 600, 1900, 1900, TEST_PARAMS), 0.0)
    w1 = gpu_face.run_cascade_array(cp_of(wide, 600, 1900, 1900, TEST_PARAMS), 1.0)
    assert_same(w1, oracle_face.run_cascade(wide, 600, 1900, 1900, *TEST_PARAMS, 1.0))
    assert w0.tobytes() != w1.tobytes()
