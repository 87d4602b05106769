"""RunDetector's kernels against the C oracle over synthetic pupil / landmark cascades (tests/puploc_cases.py), geometries and
rotation slots.  Every output equals the oracle exactly: Row and Col as integers, Scale bit for bit.  Every standalone call
also reads which kernel ran ("t_puploc_warp_n" counts the calls of the 64-bit warp-per-perturbation kernel) and, under option
walk_stats, how many stages the pair kernel served from its shared pixel patch ("pup_patch_stages") and from global memory
("pup_global_stages"); both are compared with the host restatement of the launch plan."""
import numpy as np
import pytest

import oracle_lib as O
import pigo_b200
from mixed_images import TEST_PARAMS, cp_of
from option_guard import options, options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)
from pigo_b200 import CascadeParams, ImageParams, Puploc, pipeline, synth
from pipeline_oracle import oracle_clusters, replay
from puploc_cases import header, library_randoms, pair_launch, patch_stages, puploc_cascade, standalone_kernel

pytestmark = pytest.mark.gpu

# (name, depth, trees, stages, scales): depth 10 with 20 / 24 / 25 trees (patch fits / staged without a patch / unstaged under
# puploc_stage 2), 203 / 204 trees (pair kernel / warp kernel), depth 1, zero stages, zero trees, more than 32 trees
# (the warp kernel's second round of lanes), negative and growing scales
SHAPES = [("d10t20", 10, 20, 4, 0.8), ("d10t24", 10, 24, 3, 0.8), ("d10t25", 10, 25, 3, 0.8), ("t203", 4, 203, 2, 0.7),
          ("t204", 4, 204, 2, 0.7), ("d1", 1, 40, 5, 0.9), ("s0", 6, 20, 0, 0.8), ("t0", 6, 0, 3, 0.8), ("d2t33", 2, 33, 7, 1.3),
          ("d12", 12, 3, 2, -0.8), ("d7t70", 7, 70, 3, 0.75)]
ANGLES = [0.0, 0.01, 1.5] + [k / 32 for k in range(1, 33)]    # unrotated, slot 0 through (0, 1/32), clamped, every slot
PERTURBS = [0, 1, 2, 62, 63]
_PACKETS = {}


def packet(name):
    if name not in _PACKETS:
        _, d, t, s, sc = next(x for x in SHAPES if x[0] == name)
        _PACKETS[name] = puploc_cascade(d, t, s, sc, seed=len(_PACKETS) + 7)
    return _PACKETS[name]


def counted(fn):
    """Runs fn() with the timing and walk_stats counters fresh; returns (fn(), counters)."""
    pigo_b200.set_option("timing", 1)
    pigo_b200.set_option("walk_stats", 1)
    out = fn()
    keys = ("t_puploc_n", "t_puploc_warp_n", "pup_patch_stages", "pup_global_stages")
    return out, {k: pigo_b200.get_option(k) for k in keys}


def expect(oracle, seeds, images, seed_image, randoms, angle, flips):
    return [oracle.run_detector(s[0], s[1], s[2], min(s[3], 63), randoms[i].ravel(), *images[seed_image[i]][:4], angle, flips[i])
            for i, s in enumerate(seeds)]


def assert_points(got, want, what):
    for i, (g, w) in enumerate(zip(got, want)):
        assert (g.Row, g.Col) == (w[0], w[1]) and np.float32(g.Scale).tobytes() == np.float32(w[2]).tobytes(), (what, i, g, w)


def predicted(pk, seeds, images, seed_image, randoms, angle, flips, mode, stage):
    """(kernel, patch stages, global stages) of a standalone call from the host restatement."""
    kernel = standalone_kernel(pk, [s[2] for s in seeds], mode)
    if kernel == "warp":
        return kernel, 0, 0
    _, _, tr, dp = header(pk)
    _, cap = pair_launch([(tr, dp)], stage)
    patch = glob = 0
    for i, s in enumerate(seeds):
        im = images[seed_image[i]]
        p, g = patch_stages(pk, s, randoms[i], im[:4], angle, flips[i], cap, im[4])
        patch += p
        glob += g
    return kernel, patch, glob


def random_seeds(rng, n, rows, cols, nimages):
    """Seeds inside the image, on its border and far outside it (boxes that clamp to one row or column), scales 1..16384."""
    seeds = []
    for _ in range(n):
        kind = rng.integers(4)
        scale = float(np.float32(np.exp(rng.uniform(0, np.log(16384)))))
        if kind == 0:
            r, c = int(rng.integers(0, rows)), int(rng.integers(0, cols))
        elif kind == 1:
            r, c = int(rng.choice([0, rows - 1])), int(rng.integers(-3, cols + 3))
        elif kind == 2:
            r, c = int(rng.choice([-5000, rows + 5000])), int(rng.integers(0, cols))
            scale = float(rng.uniform(1, 8))
        else:
            r, c = int(rng.integers(0, rows)), int(rng.choice([-4000, cols + 4000]))
        seeds.append((r, c, scale, int(rng.choice(PERTURBS + [int(rng.integers(0, 64))]))))
    return seeds, [int(rng.integers(nimages)) for _ in range(n)]


def make_images(rng, how):
    """[(pixels, rows, cols, dim, aligned)] and the ImageParams of a call: host images (16-byte pitch or not) or device
    images, one of them at a base that is not 16-byte aligned."""
    geoms = [(int(rng.integers(1, 300)), int(rng.integers(1, 300))) for _ in range(3)] + [(1, 40), (33, 1)]
    out, params, keep = [], [], []
    for k, (r, c) in enumerate(geoms):
        dim = c + int(rng.choice([0, 1, 5, 16])) if how != "frames" else c
        if k % 2 == 0:
            dim = (dim + 15) & ~15
        pix = np.full((r, dim), 0x33, dtype=np.uint8)
        smooth = k % 2 == 0 and min(r, c) >= 16
        pix[:, :c] = synth.frame_smooth(r, c, int(rng.integers(1 << 20))) if smooth else synth.frame_noise(r, c, int(rng.integers(1 << 20)))
        aligned = True
        if how == "device":
            import torch
            off = 1 if k == 0 else 0
            buf = torch.zeros(r * dim + 32, dtype=torch.uint8, device="cuda")
            base = buf.data_ptr()
            buf[off:off + r * dim] = torch.from_numpy(pix.reshape(-1).copy()).cuda()
            keep.append(buf)
            params.append(ImageParams(base + off, r, c, dim))
            aligned = (base + off) % 16 == 0
        else:
            params.append(ImageParams(pix, r, c, dim))
        out.append((pix, r, c, dim, aligned))
    return out, params, keep


def run_call(casc, seeds, seed_image, params, angle, flips, randoms, frames=None):
    pts = [Puploc(*s) for s in seeds]
    if frames is not None:
        buf, n, stride, r, c, d = frames
        return casc.run_detector_frames(pts, seed_image, buf, n, stride, r, c, d, angle, flips, randoms)
    return casc.run_detector_images(pts, seed_image, params, angle, flips, randoms)


CALLS = [(name, mode, stage) for name, *_ in SHAPES for mode in (0, 1) for stage in (0, 1, 2)]


def test_standalone_fuzz_against_the_oracle_and_the_plan():
    """A seeded fuzz of standalone calls over every shape x puploc_mode x puploc_stage: uniform frames, host images (pitches
    that are not multiples of 16) and device images (one at an unaligned base), flips, every rotation slot, Perturbs
    0..63, seeds inside, on and far outside the image.  Each call's kernel and patch / global stage counts match the plan."""
    rng = np.random.default_rng(2024)
    seen = {"patch": 0, "warp_204": 0}
    for k, (name, mode, stage) in enumerate(CALLS):
        pk = packet(name)
        casc = pigo_b200.NewPuplocCascade().UnpackCascade(pk)
        oracle = O.OraclePuploc(pk)
        how = ["frames", "host", "device"][k % 3]
        angle = ANGLES[k % len(ANGLES)]
        if how == "frames":
            r, c = int(rng.integers(20, 260)), int(rng.integers(20, 260))
            dim = (c + 15) & ~15 if k % 2 else c + 3
            n = 3
            fr = np.zeros((n, r, dim), dtype=np.uint8)
            for f in range(n):
                fr[f, :, :c] = synth.frame_noise(r, c, 100 * k + f) if f % 2 else synth.frame_smooth(r, c, 100 * k + f)
            stride = r * dim
            images = [(fr[f], r, c, dim, (f * stride) % 16 == 0) for f in range(n)]
            frames, params = (fr, n, stride, r, c, dim), None
        else:
            images, params, keep = make_images(rng, how)
            frames = None
        nseeds = int(rng.integers(1, 9))
        rows0, cols0 = images[0][1], images[0][2]
        seeds, sidx = random_seeds(rng, nseeds, rows0, cols0, len(images))
        flips = [bool(rng.integers(2)) for _ in seeds]
        rnd = rng.random((nseeds, 63, 3), dtype=np.float32)
        with options(puploc_mode=mode, puploc_stage=stage):
            got, cnt = counted(lambda: run_call(casc, seeds, sidx, params, angle, flips, rnd, frames))
        what = (name, mode, stage, how, angle)
        assert_points(got, expect(oracle, seeds, images, sidx, rnd, angle, flips), what)
        kernel, patch, glob = predicted(pk, seeds, images, sidx, rnd, angle, flips, mode, stage)
        assert cnt["t_puploc_n"] == 1 and cnt["t_puploc_warp_n"] == (kernel == "warp"), (what, cnt)
        assert (cnt["pup_patch_stages"], cnt["pup_global_stages"]) == (patch, glob), (what, cnt, patch, glob)
        seen["patch"] += patch
        seen["warp_204"] += name == "t204" and cnt["t_puploc_warp_n"] == 1 and mode == 0
    assert seen["patch"] > 0 and seen["warp_204"] == 3, seen


def test_patch_box_radius_and_alignment_are_visible_in_the_counters():
    """Seeds whose sample box is one row short of the patch cap, or one row over it: the restatement with the kernel's radius
    says which, and the counters must agree (a radius one smaller would accept the boxes that are one row over).  The same
    seeds on an image at an unaligned device base, or with a pitch that is not a multiple of 16, never use the patch."""
    import torch
    pk = packet("d10t20")
    casc, oracle = pigo_b200.NewPuplocCascade().UnpackCascade(pk), O.OraclePuploc(pk)
    _, cap = pair_launch([(20, 10)], 2)
    rows, cols, dim = 300, 400, 400
    pix = synth.frame_smooth(rows, cols, 9)
    rnd = np.zeros((1, 63, 3), dtype=np.float32) + 0.5
    found = {}
    for scale in np.arange(60.0, 240.0, 0.5, dtype=np.float32):
        if len(found) == 2:
            break
        seed = (150, 200, float(scale), 1)
        exact = patch_stages(pk, seed, rnd[0], (pix, rows, cols, dim), 0.0, False, cap, True)
        short = patch_stages(pk, seed, rnd[0], (pix, rows, cols, dim), 0.0, False, cap, True, margin=1)
        if exact != short and "differ" not in found:
            found["differ"] = (seed, exact)
        if exact[0] > 0 and "patch" not in found:
            found["patch"] = (seed, exact)
    assert "differ" in found and "patch" in found, found
    with options(puploc_stage=2):
        for seed, (patch, glob) in found.values():
            got, cnt = counted(lambda: casc.run_detector_images([Puploc(*seed)], [0], [ImageParams(pix, rows, cols, dim)], 0.0, [False], rnd))
            assert_points(got, expect(oracle, [seed], [(pix, rows, cols, dim)], [0], rnd, 0.0, [False]), seed)
            assert (cnt["pup_patch_stages"], cnt["pup_global_stages"]) == (patch, glob), (seed, cnt)
            buf = torch.zeros(rows * dim + 16, dtype=torch.uint8, device="cuda")
            buf[1:1 + rows * dim] = torch.from_numpy(pix.reshape(-1).copy()).cuda()
            odd = np.full((rows, dim + 3), 7, dtype=np.uint8)
            odd[:, :cols] = pix
            for im in (ImageParams(buf.data_ptr() + 1, rows, cols, dim), ImageParams(odd, rows, cols, dim + 3)):
                got, cnt = counted(lambda: casc.run_detector_images([Puploc(*seed)], [0], [im], 0.0, [False], rnd))
                assert_points(got, expect(oracle, [seed], [(pix, rows, cols, dim)], [0], rnd, 0.0, [False]), seed)
                assert (cnt["pup_patch_stages"], cnt["pup_global_stages"]) == (0, patch + glob), (seed, cnt)
            torch.cuda.synchronize()


@pytest.mark.parametrize("mode", [0, 1])
def test_library_generator_matches_its_restatement(mode):
    """randoms=None: the draws of seed i are library_randoms(rng_seed, i) on both kernels."""
    pk = packet("d2t33")
    casc, oracle = pigo_b200.NewPuplocCascade().UnpackCascade(pk), O.OraclePuploc(pk)
    pix = synth.frame_smooth(200, 240, 3)
    seeds = [(100, 120, 30.0, 63), (50, 60, 12.5, 40), (150, 200, 60.0, 7), (10, 10, 5.0, 2), (199, 239, 80.0, 63), (90, 100, 20.0, 1)]
    rnd = np.stack([library_randoms(987654321, i) for i in range(len(seeds))])
    with options(puploc_mode=mode):
        got, cnt = counted(lambda: casc.run_detector_frames([Puploc(*s) for s in seeds], [0] * len(seeds), pix, 1, 200 * 240, 200, 240, 240,
                                                            0.2, [i % 2 == 0 for i in range(len(seeds))], None, rng_seed=987654321))
    assert cnt["t_puploc_warp_n"] == mode
    assert_points(got, expect(oracle, seeds, [(pix, 200, 240, 240)], [0] * len(seeds), rnd, 0.2, [i % 2 == 0 for i in range(len(seeds))]), mode)


def test_scale_growth_runs_on_the_64_bit_kernel():
    """scales = 2.0 over 20 stages: from a seed of Scale 100 the last stages sample with |s| > 2^24, where the pair kernel's
    32-bit offsets wrap.  The predictions shrink by 1/2 per stage so that the points stay in the image.  Such calls must run
    on puploc_kernel (t_puploc_warp_n) and equal the oracle; a seed inside the envelope still runs the pair kernel."""
    rng = np.random.default_rng(5)
    st, sc, tr, dp = 20, 2.0, 12, 6
    L = 1 << dp
    import struct
    body = bytearray(struct.pack("<IfII", st, sc, tr, dp))
    for s in range(st):
        for _ in range(tr):
            body += rng.integers(-128, 128, size=4 * L - 4).astype(np.int8).tobytes()
            body += (rng.uniform(-0.02, 0.02, size=2 * L) / 2.0 ** s).astype("<f4").tobytes()
    pk = bytes(body)
    casc, oracle = pigo_b200.NewPuplocCascade().UnpackCascade(pk), O.OraclePuploc(pk)
    pix = synth.frame_noise(240, 320, 8)
    seeds = [(120, 160, 100.0, 63), (60, 100, 150.0, 50), (200, 300, 80.0, 63)]
    rnd = rng.random((3, 63, 3), dtype=np.float32)
    for mode in (0, 1):
        with options(puploc_mode=mode):
            got, cnt = counted(lambda: casc.run_detector_frames([Puploc(*s) for s in seeds], [0, 0, 0], pix, 1, 240 * 320, 240, 320, 320, 0.0,
                                                                [False, True, False], rnd))
        assert_points(got, expect(oracle, seeds, [(pix, 240, 320, 320)], [0, 0, 0], rnd, 0.0, [False, True, False]), mode)
        assert cnt["t_puploc_warp_n"] == 1, cnt
    tiny = [(120, 160, 0.03, 63)]
    with options():
        got, cnt = counted(lambda: casc.run_detector_frames([Puploc(*tiny[0])], [0], pix, 1, 240 * 320, 240, 320, 320, 0.0, [False], rnd[:1]))
    assert cnt["t_puploc_warp_n"] == 0
    assert_points(got, expect(oracle, tiny, [(pix, 240, 320, 320)], [0], rnd[:1], 0.0, [False]), "tiny")


@pytest.mark.parametrize("mode", [0, 1])
def test_device_seeds_above_63_perturbs_write_every_field(mode):
    """Seeds on the device are not checked on the host (include/pigo_b200.h): Perturbs above 63 run as 63.  Every output
    field must be written over a sentinel, and equal the oracle's Perturbs-63 result."""
    import torch
    pk = packet("d10t20")
    oracle = O.OraclePuploc(pk)
    casc = pigo_b200.NewPuplocCascade().UnpackCascade(pk)
    pix = synth.frame_smooth(200, 256, 11)
    seeds = [(100, 128, 40.0, 64), (80, 90, 25.0, 100), (120, 200, 33.0, 127), (60, 60, 50.0, 500), (150, 150, 20.0, 63)]
    rnd = np.random.default_rng(3).random((len(seeds), 63, 3), dtype=np.float32)
    d_seeds = torch.from_numpy(np.array(seeds, dtype=pigo_b200.POINT_DTYPE).view(np.uint8)).cuda()
    d_rnd = torch.from_numpy(rnd.reshape(-1)).cuda()
    d_pix = torch.from_numpy(pix.reshape(-1).copy()).cuda()
    sentinel = np.array([(0x7EADBEEF, 0x7EADBEEF, 0.0, 0x5A5A5A5A)] * len(seeds), dtype=pigo_b200.POINT_DTYPE)
    sentinel["scale"] = np.frombuffer(np.uint32(0x7FBADBAD).tobytes(), np.float32)[0]
    d_out = torch.from_numpy(sentinel.view(np.uint8).copy()).cuda()
    with options(puploc_mode=mode):
        rc = pigo_b200.lib().pigo_puploc_run_frames(casc._h, d_seeds.data_ptr(), len(seeds), None, d_rnd.data_ptr(), 0, d_pix.data_ptr(), 1,
                                                    200 * 256, 200, 256, 256, 0.0, None, d_out.data_ptr(),
                                                    pigo_b200.FRAMES_DEVICE | pigo_b200.OUT_DEVICE, None)
        torch.cuda.synchronize()
    assert rc == 0
    out = d_out.cpu().numpy().view(pigo_b200.POINT_DTYPE)
    for i, s in enumerate(seeds):
        w = oracle.run_detector(s[0], s[1], s[2], 63, rnd[i].ravel(), pix, 200, 256, 256)
        assert (int(out[i]["row"]), int(out[i]["col"]), out[i]["scale"].tobytes(), int(out[i]["perturbs"])) == (w[0], w[1], w[2].tobytes(), 0), (i, out[i])


@pytest.mark.parametrize("mode", [0, 1])
def test_nan_leaves_give_one_answer_over_dirty_scratch(mode):
    """A cascade with NaN leaf predictions: NaN rows and columns fill part of the pool.  With the total order (NaN above every
    number, ties by slot) exactly one thread publishes each field, so two calls over differently dirtied scratch agree and
    equal the oracle (int(NaN) is 0)."""
    pk = puploc_cascade(6, 20, 3, 0.8, seed=77, nan_leaves=0.006)
    casc, oracle = pigo_b200.NewPuplocCascade().UnpackCascade(pk), O.OraclePuploc(pk)
    pix = synth.frame_smooth(200, 256, 13)
    rng = np.random.default_rng(9)
    seeds = [(100, 128, 40.0, 63), (80, 90, 25.0, 63), (120, 200, 33.0, 40), (60, 60, 50.0, 63), (150, 150, 20.0, 11), (30, 40, 60.0, 63)]
    rnd = rng.random((len(seeds), 63, 3), dtype=np.float32)
    want = expect(oracle, seeds, [(pix, 200, 256, 256)], [0] * len(seeds), rnd, 0.0, [False] * len(seeds))
    nans = [sum(np.isnan(oracle.classify(*_perturb(s, rnd[i], j), pix, 200, 256, 256)[0]) for j in range(s[3])) for i, s in enumerate(seeds)]
    assert any(0 < n < 63 for n in nans) and any(n >= 32 for n in nans), nans
    outs = []
    with options(puploc_mode=mode):
        for dirty in (20, 150):   # the call before leaves its outputs in the scratch the next call's outputs go to
            casc.run_detector_frames([Puploc(dirty + k, dirty + 2 * k, 30.0 + k, 63) for k in range(len(seeds))], [0] * len(seeds), pix, 1,
                                     200 * 256, 200, 256, 256, 0.0, None, rnd)
            outs.append(casc.run_detector_frames([Puploc(*s) for s in seeds], [0] * len(seeds), pix, 1, 200 * 256, 200, 256, 256, 0.0, None, rnd))
    assert outs[0] == outs[1]
    assert_points(outs[0], want, mode)


def _perturb(seed, r, j):
    f32 = np.float32
    t1 = f32(f32(seed[2]) * f32(0.15))
    return (f32(f32(seed[0]) + f32(t1 * f32(f32(0.5) - r[j, 0]))), f32(f32(seed[1]) + f32(t1 * f32(f32(0.5) - r[j, 1]))),
            f32(f32(seed[2]) * f32(f32(0.925) + f32(f32(0.15) * r[j, 2]))))


# ---- pipeline -------------------------------------------------------------------------------------------------------------
LANDMARK_SHAPES = {"A": (9, 20, 6, 0.7), "B": (5, 33, 4, 0.8), "C": (10, 12, 3, 0.75)}
NAME_SHAPE = {"lp46": "A", "lp44": "A", "lp42": "A", "lp38": "B", "lp312": "B", "lp93": "C", "lp84": "C", "lp82": "C", "lp81": "C"}


@pytest.fixture(scope="module")
def synthetic_pipeline():
    """A synthetic pupil cascade and landmark positions that use three synthetic cascades of different shapes, on the GPU
    and on the oracle."""
    pup = puploc_cascade(10, 20, 5, 0.8, seed=101, pred=0.01)
    lm = {k: puploc_cascade(*v, seed=200 + i, pred=0.01) for i, (k, v) in enumerate(LANDMARK_SHAPES.items())}
    g = {k: pigo_b200.NewPuplocCascade().UnpackCascade(v) for k, v in lm.items()}
    o = {k: O.OraclePuploc(v) for k, v in lm.items()}
    return (pigo_b200.NewPuplocCascade().UnpackCascade(pup), {n: g[s] for n, s in NAME_SHAPE.items()},
            (O.OraclePuploc(pup), {n: o[s] for n, s in NAME_SHAPE.items()}))


@pytest.mark.parametrize("stage", [1, 2])
def test_pipeline_with_synthetic_cascades(gpu_face, oracle_face, synthetic_pipeline, stage):
    """pigo_detect_batch with injected randoms, pigo_detect_images with the library generator and the sharded mixed-size
    call split in two on one card (its second shard's keys are offset by slot_base): each replayed on the oracle."""
    plc, flp, oracle = synthetic_pipeline
    frames = np.stack([synth.frame_faces(synth.sample_gray(), 360, 480, noise_seed=s) for s in (1, 2)])
    face_cap, stride = 8, 17
    rnd = np.random.default_rng(4).random((2, face_cap, stride, 63, 3), dtype=np.float32)
    cp = CascadeParams(ImageParams(None, 360, 480, 480), *TEST_PARAMS)
    cases = [(i, (frames[i], 360, 480, 480), oracle_clusters(oracle_face, (frames[i], 360, 480, 480), TEST_PARAMS, 0.0), 0.0) for i in range(2)]
    with options(puploc_stage=stage):
        got = pipeline.detect_batch_device(gpu_face, plc, flp, frames, cp, face_cap=face_cap, randoms=rnd, raw=True)
        refined, _ = replay(oracle, cases, lambda i, k, slot: rnd[i, k, slot].ravel(), 50, got)
        assert refined >= 2
        ims = [ImageParams(frames[i], 360, 480, 480) for i in range(2)]
        lib_rnd = lambda i, k, slot: library_randoms(31337, (i * face_cap + k) * stride + slot).ravel()   # noqa: E731
        got = pipeline.detect_images_device(gpu_face, plc, flp, ims, cp_of(), face_cap=face_cap, rng_seed=31337, raw=True)
        assert replay(oracle, cases, lib_rnd, 50, got)[0] == refined
        pigo_b200.set_option("shard_split", 2)
        got = pipeline.detect_images_sharded(gpu_face, plc, flp, ims, cp_of(), None, face_cap=face_cap, rng_seed=31337, raw=True)
        assert replay(oracle, cases, lib_rnd, 50, got)[0] == refined


def test_pipeline_refuses_cascades_it_cannot_run(gpu_face, synthetic_pipeline):
    """A pupil cascade of 204 trees per stage (its leaves do not fit the pair kernel) and one whose scale grows by more
    than 512 over its stages give PIGO_E_INVALID."""
    _, flp, _ = synthetic_pipeline
    frames = synth.frame_faces(synth.sample_gray(), 360, 480, noise_seed=1)[None]
    cp = CascadeParams(ImageParams(None, 360, 480, 480), *TEST_PARAMS)
    for pk in (puploc_cascade(2, 204, 1, 0.8, seed=1), puploc_cascade(2, 2, 11, 2.0, seed=1)):
        plc = pigo_b200.NewPuplocCascade().UnpackCascade(pk)
        with pytest.raises(pigo_b200.PigoError) as e:
            pipeline.detect_batch_device(gpu_face, plc, flp, frames, cp, face_cap=8, raw=True)
        assert e.value.status == pigo_b200.PIGO_E_INVALID
