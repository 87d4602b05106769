"""The fused kernel's region role against the C oracle over what the fixed cases of test_region_gpu.py leave out: random
geometries (Dim != Cols, thin and tall frames), frame strides, frame counts, scan parameters and region-plan options;
cascades whose trees all fit in shared memory; windows handed over between a CTA's two buffers; the capacity path; the fallbacks to per-warp tiles; the auto choice of the
tile role; and the face pipeline on a batch that runs the region role.  Every call is compared frame by frame, byte for
byte, with the oracle (or with the same call on per-warp tiles), and every call reads the "t_region_n" timing counter:
the number of fused launches that really ran the region role, which a silent fallback would leave at 0."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle_lib as O
import pigo_b200
import pipeline_oracle as P
from mixed_images import cascades   # noqa: F401 (fixture)
from option_guard import options, options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)
from pigo_b200 import pipeline, synth
from synthetic import synthetic_cascade
from test_gpu_parity import TEST_PARAMS

pytestmark = pytest.mark.gpu

NTHREADS = max(1, min(16, os.cpu_count() or 1))


def pack_frames(frames, dim, stride):
    """(nf, rows, cols) frames laid out Dim bytes per row and `stride` bytes apart; the buffer ends right after the last
    frame's last readable byte ((rows - 1) * Dim + Cols), the least a caller has to provide.  Bytes outside the frames are
    0x5a, so that a kernel reading them would see non-zero values."""
    nf, rows, cols = frames.shape
    buf = np.full((nf - 1) * stride + (rows - 1) * dim + cols, 0x5a, dtype=np.uint8)
    for f in range(nf):
        v = buf[f * stride:f * stride + (rows - 1) * dim + cols]
        for r in range(rows):
            v[r * dim:r * dim + cols] = frames[f, r]
    return buf


def oracle_frames(clf_oracle, frames, dim, prm):
    """The oracle's detections of every frame (frames on Dim-byte rows, columns past Cols zero)."""
    nf, rows, cols = frames.shape
    padded = np.zeros((nf, rows, dim), dtype=np.uint8)
    padded[:, :, :cols] = frames
    out, n = clf_oracle.run_cascade_batch(padded, rows, cols, dim, *prm, 0.0, cap_per_frame=1 << 12, nthreads=NTHREADS)
    if n.max(initial=0) > 1 << 12:
        out, n = clf_oracle.run_cascade_batch(padded, rows, cols, dim, *prm, 0.0, cap_per_frame=int(n.max()), nthreads=NTHREADS)
    return [out[f, :n[f]].copy() for f in range(nf)]


def run_batch(clf, buf, nf, stride, rows, cols, dim, prm, cap, device=False, offset=0):
    """pigo_run_cascade_batch on `buf` (host memory, or a device copy of it placed `offset` bytes past a 256-byte aligned
    address) with host outputs; the output slots start as 0xa5 bytes so that the zeroed padding is the library's.  Returns
    (rc, dets[nf, cap], counts, {"t_tiled_n", "t_region_n"})."""
    import torch
    keep = None
    if device:
        keep = torch.zeros(len(buf) + offset + 256, dtype=torch.uint8, device="cuda")
        base = (-keep.data_ptr()) % 256
        keep[base + offset:base + offset + len(buf)] = torch.from_numpy(buf).cuda()
        ptr = keep.data_ptr() + base + offset
    else:
        ptr = buf.ctypes.data
    out = np.full(nf * max(cap, 1) * 16, 0xa5, dtype=np.uint8).view(pigo_b200.DET_DTYPE).reshape(nf, max(cap, 1))
    cnt = np.full(nf, -7, dtype=np.int32)
    with options(timing=1):
        rc = pigo_b200.lib().pigo_run_cascade_batch(clf._h, C.c_void_p(ptr), nf, stride, rows, cols, dim, prm[0], prm[1], prm[2], prm[3], 0.0,
                                                    out.ctypes.data, cap, cnt.ctypes.data,
                                                    pigo_b200.FRAMES_DEVICE if device else pigo_b200.MEM_HOST, None)
        launches = {k: pigo_b200.get_option(k) for k in ("t_tiled_n", "t_region_n")}
    if device:
        torch.cuda.synchronize()
        del keep
    return rc, out, cnt, launches


def assert_frames_equal(out, cnt, want, what=""):
    """Every frame's detections equal the oracle's byte for byte.  The library copies each frame's slots up to the largest
    count of the call: those past the frame's own count must be zero, the slots past the largest count stay the caller's."""
    copied = min(int(cnt.max(initial=0)), out.shape[1])
    for f, o in enumerate(want):
        assert cnt[f] == len(o), f"{what} frame {f}: {cnt[f]} detections vs oracle {len(o)}"
        assert out[f, :cnt[f]].tobytes() == o.tobytes(), f"{what} frame {f}"
        assert not out[f, cnt[f]:copied].tobytes().strip(b"\0"), f"{what} frame {f}: padding past the count is not zero"
        assert not out[f, copied:].tobytes().strip(b"\xa5"), f"{what} frame {f}: slots past the largest count were written"


def run_checked(clf, buf, nf, stride, rows, cols, dim, prm, want, cap=256, device=False, offset=0, what=""):
    """run_batch, retried with the required capacity on PIGO_E_CAP, against the oracle's `want`; returns the launches."""
    rc, out, cnt, launches = run_batch(clf, buf, nf, stride, rows, cols, dim, prm, cap, device, offset)
    if rc == pigo_b200.PIGO_E_CAP:
        assert list(cnt) == [len(o) for o in want], f"{what}: required counts {list(cnt)}"
        rc, out, cnt, launches = run_batch(clf, buf, nf, stride, rows, cols, dim, prm, int(cnt.max()), device, offset)
    assert rc == 0, f"{what}: {pigo_b200.lib().pigo_last_error().decode()}"
    assert_frames_equal(out, cnt, want, what)
    return launches


def face_frames(sample_gray, nf, rows, cols, seed, zoom=1.0):
    """Frames tiled with the sample face, shifted per frame; zoom < 1 shrinks the face first (0.12 .. 0.25: faces found at
    scales 22 .. 50, the scales the region role scans, where the full-size face is found at about 180, a gather-role scale)."""
    patch = sample_gray
    if zoom != 1.0:
        from scipy import ndimage
        patch = ndimage.zoom(sample_gray.astype(np.float32), zoom, order=1).clip(0, 255).astype(np.uint8)
    return np.stack([synth.frame_faces(patch, rows, cols, shift=(37 * f + seed, 53 * f + 3 * seed), noise_seed=seed + f) for f in range(nf)])


# ---- seeded random fuzz of the region role ---------------------------------------------------------------------------
SHIFTS = [0.03, 0.05, 0.1, 0.15, 0.2, 0.33, 1.0]
SCALES = [1.03, 1.05, 1.1, 1.15, 1.3, 2.0]
CALL_WINDOWS = 6_000_000   # per case (all frames): keeps the oracle's share of the run short


def _region_case(rng, sample_gray):
    """One random call: geometry, stride, frames, content, scan parameters and region-plan options."""
    if rng.random() < 0.12:
        rows, cols = int(rng.integers(24, 48)), int(rng.choice([4000, 3008, 2640]))          # thin frames
    else:
        rows = int(rng.integers(24, 1201))
        cols = 16 * int(rng.integers(2, 129)) if rng.random() < 0.8 else int(rng.integers(24, 2049))
    u = rng.random()
    if cols % 16 and u < 0.5:
        dim = cols + (-cols) % 16 + 16 * int(rng.choice([0, 0, 1]))                           # Cols ragged, Dim aligned
    elif u < 0.85:
        dim = cols + 16 * int(rng.choice([0, 0, 0, 1, 3]))
    else:
        dim = cols + int(rng.choice([1, 3, 7, 21]))                                           # Dim % 16 != 0 (when Cols is aligned)
    nf = int(rng.choice([1, 2, 3, 7, 11]))
    mn = int(rng.choice([0, 1, 7, 12, 20, 20, 24, 33, 50]))
    mx = int(rng.choice([mn, mn + 5, 60, 150, 1000, 1000]))
    shift, scale = float(rng.choice(SHIFTS)), float(rng.choice(SCALES))
    kind = str(rng.choice(["noise", "flat", "face", "small faces", "small faces"]))
    if kind == "face" and rows >= 300 and cols >= 300:   # parameters that find the sample face (as in test_gpu_parity's fuzz)
        mn, mx = int(rng.choice([20, 24, 50])), 1000
        shift, scale = min(shift, 0.2), min(scale, 1.3)
    if kind == "small faces":
        mx = max(mx, 60)
        shift, scale = min(shift, 0.2), min(scale, 1.3)
    while pigo_b200.count_windows(rows, cols, mn, mx, shift, scale) * nf > CALL_WINDOWS:
        if nf > 1:
            nf = {2: 1, 3: 2, 7: 3, 11: 7}[nf]
        elif shift < 1.0:
            shift = SHIFTS[SHIFTS.index(shift) + 1]
        else:
            mn += 20
    seed = int(rng.integers(1 << 30))
    if kind == "noise":
        frames = np.stack([synth.frame_noise(rows, cols, seed + f) for f in range(nf)])
    elif kind == "flat":
        frames = np.stack([np.full((rows, cols), int(rng.integers(0, 256)), dtype=np.uint8) for _ in range(nf)])
    else:
        zoom = float(rng.choice([0.12, 0.16, 0.2, 0.25])) if kind == "small faces" else 1.0
        frames = face_frames(sample_gray, nf, rows, cols, seed % 1000, zoom)
    device = bool(rng.random() < 0.5)
    extra = int(rng.choice([0, 0, 1, 5]))
    stride = rows * dim + (16 * extra if dim % 16 == 0 else 3 * extra)
    opts = {"tile_region": 1,
            "tile_warps": int(rng.choice([1, 2, 3, 7, 24])), "gather_warps": int(rng.choice([0, 1, 8])),
            "tile_ks": int(rng.choice([1, 6, 48, 250])), "tile_band_ratio": int(rng.choice([0, 100, 110, 400])),
            "tile_max_scale": int(rng.choice([0, 24, 40, 80])), "tile_tail_min": int(rng.choice([6, 0, 33])),
            "queue_cap": int(rng.choice([0, 0, 7, 40, 3000])), "deep_group": int(rng.choice([0, 8, 16, 32]))}
    if device:
        opts["sub_batch"] = int(rng.choice([0, 1, 2, 4]))
    else:
        opts.update(host_stream=int(rng.choice([0, 1])), copy_chunk=int(rng.choice([1, 3, 8])), sub_batch=int(rng.choice([0, 1, 4])))
    return frames, rows, cols, dim, nf, stride, (mn, mx, shift, scale), kind, device, opts


def test_region_role_random_fuzz(gpu_face, oracle_face, sample_gray):
    """48 random calls with the region role forced, each bit-equal to the oracle, padding past each count zero.  With Dim
    % 16 != 0 the role must fall back (t_region_n == 0); where describe_plan describes the call (facefinder, Dim == Cols)
    the role runs exactly when it says so.  Floors: most calls ran the region role, the calls of face frames found many
    faces, and several calls overflowed the deep queue (more windows outlive the resident prefix and the gather limit than
    the queue holds)."""
    rng = np.random.default_rng(20261016)
    ran = faces = overflowed = 0
    ncases = 48
    for case in range(ncases):
        frames, rows, cols, dim, nf, stride, prm, kind, device, opts = _region_case(rng, sample_gray)
        what = (f"case {case}: {nf} x {rows}x{cols} dim {dim} stride {stride} {'device' if device else 'host'} {prm} {kind} "
                f"options {opts}")
        want = oracle_frames(oracle_face, frames, dim, prm)
        buf = pack_frames(frames, dim, stride)
        with options(**opts):
            launches = run_checked(gpu_face, buf, nf, stride, rows, cols, dim, prm, want, cap=int(rng.choice([1, 64, 1024])),
                                   device=device, what=what)
            plan = pigo_b200.describe_plan(rows, cols, *prm, nframes=nf)
        n = launches["t_region_n"]
        assert n <= launches["t_tiled_n"], what
        if dim % 16:
            assert n == 0, what
        elif dim == cols:
            assert n == (launches["t_tiled_n"] if plan["region"] else 0), f"{what}: plan region {plan['region']}, {launches}"
        ran += n > 0
        if "face" in kind:
            faces += sum(len(o) for o in want)
        if n > 0 and opts["queue_cap"] in (7, 40):
            hist = oracle_face.run_cascade(np.pad(frames[0], ((0, 0), (0, dim - cols))), rows, cols, dim, *prm, 0.0, with_hist=True)[1]
            overflowed += int(hist[max(opts["tile_ks"], 8) + 1:].sum()) > opts["queue_cap"]
    print(f"region fuzz: {ran} of {ncases} calls ran the region role, {faces} detections on face frames, {overflowed} overflowed the queue")
    assert ran >= ncases // 2, ran
    assert faces >= 10000, faces
    assert overflowed >= 5, overflowed


# ---- cascades whose trees all fit in shared memory ---------------------------------------------------------------------
@pytest.mark.parametrize("ntrees", [1, 3, 20, 47, 48, 49, 70])
def test_region_role_all_resident_synthetic_cascades(ntrees):
    """Depth-6 synthetic cascades with the resident prefix one tree short of the cascade, the whole cascade, and 48 trees;
    with and without a 7-item deep queue (windows then finish in the tile warps, overflow mode, down to the last tree).
    Five frames per call, so that the two buffers of a CTA hold regions of different frames when windows are handed over."""
    pk = synthetic_cascade(6, ntrees, seed=900 + ntrees)
    clf = pigo_b200.NewPigo().Unpack(pk)
    ora = O.OracleFace(pk)
    rows, cols, prm = 270, 480, (20, 200, 0.1, 1.1)
    frames = np.stack([synth.frame_smooth(rows, cols, seed=ntrees + f, sigma=3.0) for f in range(5)])
    want = oracle_frames(ora, frames, cols, prm)
    assert sum(len(o) for o in want) > 0
    buf = pack_frames(frames, cols, rows * cols)
    for ks in sorted({max(1, ntrees - 1), ntrees, 48}):
        for qcap in (0, 7):
            what = f"{ntrees} trees, tile_ks {ks}, queue_cap {qcap}"
            with options(tile_region=1, tile_ks=ks, queue_cap=qcap):
                launches = run_checked(clf, buf, 5, rows * cols, rows, cols, cols, prm, want, cap=64, what=what)
            assert launches["t_region_n"] == launches["t_tiled_n"] == 1, f"{what}: {launches}"


@pytest.mark.parametrize("opt", [{"tile_ks": 48}, {"tile_ks": 250, "tile_warps": 3}, {"tile_ks": 120, "gather_warps": 0, "tile_tail_min": 0}],
                         ids=["ks48", "ks250-3warps", "ks120-no-gather-warps"])
def test_region_role_hands_over_between_buffers(gpu_face, oracle_face, sample_gray, opt):
    """Small faces (found at scales 22 .. 50) over an 11 x 720p batch: several regions per CTA, and many windows that live
    long in the tile warps, so that warps still hold windows of the older buffer's region when they move on to the next and
    hand those to the deep queue with their partial sums."""
    rows, cols, nf, prm = 720, 1280, 11, (20, 1000, 0.1, 1.1)
    frames = face_frames(sample_gray, nf, rows, cols, 23, zoom=0.12 + 0.02 * (opt["tile_ks"] % 5))
    want = oracle_frames(oracle_face, frames, cols, prm)
    assert min(len(o) for o in want) > 1000
    buf = pack_frames(frames, cols, rows * cols)
    with options(tile_region=1, **opt):
        launches = run_checked(gpu_face, buf, nf, rows * cols, rows, cols, cols, prm, want, cap=1 << 15, device=True)
    assert launches == {"t_tiled_n": 1, "t_region_n": 1}, launches


# ---- capacity ------------------------------------------------------------------------------------------------------------
def test_region_role_capacity(gpu_face, oracle_face, sample_gray):
    """cap_per_frame below the detections: PIGO_E_CAP with every frame's required count equal to the oracle's, and the
    retry equal to the oracle; on host and on device frames."""
    rows, cols, nf = 540, 960, 4
    frames = face_frames(sample_gray, nf, rows, cols, 11)
    want = oracle_frames(oracle_face, frames, cols, TEST_PARAMS)
    assert min(len(o) for o in want) > 2
    buf = pack_frames(frames, cols, rows * cols)
    for device in (False, True):
        with options(tile_region=1):
            rc, out, cnt, launches = run_batch(gpu_face, buf, nf, rows * cols, rows, cols, cols, TEST_PARAMS, 2, device)
            assert rc == pigo_b200.PIGO_E_CAP and launches["t_region_n"] == 1
            assert list(cnt) == [len(o) for o in want]
            run_checked(gpu_face, buf, nf, rows * cols, rows, cols, cols, TEST_PARAMS, want, cap=int(cnt.max()), device=device)


# ---- fallbacks to the per-warp tiles -------------------------------------------------------------------------------------
FALLBACKS = [
    ("pointer offset by one byte", dict(device=True, offset=1), {}),
    ("frame stride not a multiple of 16", dict(device=True, stride_extra=8), {}),
    ("Dim % 16 != 0", dict(dim_extra=5), {}),
    ("no tensor maps", dict(), {"tile_tmap": 0}),
]


@pytest.mark.parametrize("how,call,opt", FALLBACKS, ids=[f[0].replace(" ", "_") for f in FALLBACKS])
def test_region_role_fallbacks_are_visible(gpu_face, oracle_face, sample_gray, how, call, opt):
    """Frames the region role cannot fill by TMA tensor copies: the fused kernel runs the per-warp tiles instead, the
    counter shows it (t_region_n == 0 with the region role forced), and the result still equals the oracle."""
    rows, cols, nf = 360, 640, 3
    dim = cols + call.get("dim_extra", 0)
    stride = rows * dim + call.get("stride_extra", 0)
    frames = face_frames(sample_gray, nf, rows, cols, 5)
    want = oracle_frames(oracle_face, frames, dim, TEST_PARAMS)
    buf = pack_frames(frames, dim, stride)
    with options(tile_region=1, **opt):
        launches = run_checked(gpu_face, buf, nf, stride, rows, cols, dim, TEST_PARAMS, want, device=call.get("device", False),
                               offset=call.get("offset", 0), what=how)
    assert launches == {"t_tiled_n": 1, "t_region_n": 0}, launches
    # the same frames aligned: the region role runs
    buf = pack_frames(frames, cols + 16 * (dim != cols), rows * (cols + 16 * (dim != cols)))
    with options(tile_region=1):
        d = cols + 16 * (dim != cols)
        launches = run_checked(gpu_face, buf, nf, rows * d, rows, cols, d, TEST_PARAMS, oracle_frames(oracle_face, frames, d, TEST_PARAMS),
                               device=call.get("device", False), what=how + " (aligned)")
    assert launches == {"t_tiled_n": 1, "t_region_n": 1}, launches


def test_region_role_tight_aligned_device_stride(gpu_face, oracle_face, sample_gray):
    """1904-wide frames on 1920-byte rows, packed (rows - 1) * Dim + Cols bytes apart on the device: a 16-byte multiple, so
    the tensor maps are encoded (their column extent is Cols: the last frame's last row ends at its Cols-th byte) and the
    region role runs, equal to the oracle."""
    rows, cols, dim, nf = 300, 1904, 1920, 4
    stride = (rows - 1) * dim + cols
    assert stride % 16 == 0
    frames = face_frames(sample_gray, nf, rows, cols, 9)
    want = oracle_frames(oracle_face, frames, dim, TEST_PARAMS)
    assert sum(len(o) for o in want) > 0
    buf = pack_frames(frames, dim, stride)
    with options(tile_region=1):
        launches = run_checked(gpu_face, buf, nf, stride, rows, cols, dim, TEST_PARAMS, want, device=True)
    assert launches == {"t_tiled_n": 1, "t_region_n": 1}, launches


# ---- the planner's choice on real calls --------------------------------------------------------------------------------
@pytest.mark.parametrize("nf,prm,region", [(2, TEST_PARAMS, 0), (3, TEST_PARAMS, 1), (3, (20, 1000, 0.1, 1.1), 0)])
def test_auto_tile_role_on_real_calls(gpu_face, nf, prm, region):
    """Auto: the region role runs on calls of more than 2 M windows at most one window per pixel (3 x 1080p at the test
    parameters), not on 2 x 1080p nor at ShiftFactor 0.1; each call byte-equal to the per-warp tiles (tile_region=2)."""
    rows, cols = 1080, 1920
    frames = synth.make_batch(nf, rows, cols, "FSU", seed0=31)
    buf = pack_frames(frames, cols, rows * cols)
    rc, out, cnt, launches = run_batch(gpu_face, buf, nf, rows * cols, rows, cols, cols, prm, 1024)
    assert rc == 0 and launches == {"t_tiled_n": 1, "t_region_n": region}, launches
    assert pigo_b200.describe_plan(rows, cols, *prm, nframes=nf)["region"] == region
    with options(tile_region=2):
        rc2, out2, cnt2, launches2 = run_batch(gpu_face, buf, nf, rows * cols, rows, cols, cols, prm, 1024)
    assert rc2 == 0 and launches2 == {"t_tiled_n": 1, "t_region_n": 0}, launches2
    assert cnt.tobytes() == cnt2.tobytes() and out.tobytes() == out2.tobytes()
    assert cnt.sum() > 0


def test_pipeline_on_the_region_role(gpu_face, oracle_face, sample_gray, cascades):
    """pigo_detect_batch on 3 x 1080p face frames (auto: the region role) equals the same call on per-warp tiles, faces and
    points byte for byte; frame 0 replayed on the oracle."""
    rows, cols, nf = 1080, 1920, 3
    frames = face_frames(sample_gray, nf, rows, cols, 17)
    plc, flp, _, _ = cascades
    face_cap = 64
    randoms = np.random.default_rng(12).random((nf, face_cap, 17, 63, 3), dtype=np.float32)
    cp = pigo_b200.CascadeParams(pigo_b200.ImageParams(None, rows, cols, cols), *TEST_PARAMS)
    with options(timing=1):
        got = pipeline.detect_batch_device(gpu_face, plc, flp, frames, cp, iou=0.1, face_cap=face_cap, randoms=randoms, raw=True)
        assert pigo_b200.get_option("t_region_n") == 1
    with options(tile_region=2, timing=1):
        per_warp = pipeline.detect_batch_device(gpu_face, plc, flp, frames, cp, iou=0.1, face_cap=face_cap, randoms=randoms, raw=True)
        assert pigo_b200.get_option("t_region_n") == 0
    assert all(a.tobytes() == b.tobytes() for a, b in zip(got, per_warp))
    image = (frames[0], rows, cols, cols)
    cls = P.oracle_clusters(oracle_face, image, TEST_PARAMS, 0.0)
    assert 0 < len(cls) <= face_cap
    refined, _ = P.replay(cascades[2:], [(0, image, cls, 0.0)], lambda f, k, slot: randoms[f, k, slot], 50, got)
    assert refined >= 3
