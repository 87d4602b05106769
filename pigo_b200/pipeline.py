"""Face -> cluster -> pupils -> 15 landmark points for a batch of frames (BASELINE.json configs[4]).

The sequencing (which seeds, which cascades, which flips) is the CALLER's logic in the reference --
core/flploc_test.go:75-154 and cmd/pigo/main.go:416-563 -- so it lives here on the host side above the C-ABI and uses
only mirrored API calls: RunCascadeBatch, ClusterDetections, RunDetector (batched over seeds), GetLandmarkPoint.
`randoms_for(frame, call_index)` (optional) injects the [63][3] perturbation randoms of each RunDetector call so that a
CPU oracle can replay the exact same pipeline; without it the library's counter-based generator is used."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional

import numpy as np

from . import CascadeParams, ImageParams, Pigo, Puploc, PuplocCascade

EYE_CASCADES = ["lp46", "lp44", "lp42", "lp38", "lp312"]      # core/flploc_test.go:77
MOUTH_CASCADES = ["lp93", "lp84", "lp82", "lp81"]             # core/flploc_test.go:78


@dataclass
class Face:
    det: tuple                   # clustered (row, col, scale, q)
    left_eye: Optional[Puploc] = None
    right_eye: Optional[Puploc] = None
    landmarks: List[Puploc] = field(default_factory=list)   # 15 points in the reference test's call order


def eye_seeds(row: int, col: int, scale: int, perturbs: int):
    """core/flploc_test.go:103-118 (float32 arithmetic, int() truncation)."""
    f32 = np.float32
    r = row - int(f32(0.075) * f32(scale))
    sc = float(f32(scale) * f32(0.25))
    left = Puploc(r, col - int(f32(0.175) * f32(scale)), sc, perturbs)
    right = Puploc(r, col + int(f32(0.185) * f32(scale)), sc, perturbs)
    return left, right


def landmark_calls():
    calls = [(e, f) for e in EYE_CASCADES for f in (False, True)]
    calls += [(m, False) for m in MOUTH_CASCADES] + [("lp84", True)]
    return calls


def detect_batch(clf: Pigo, plc: PuplocCascade, flpcs: Dict[str, PuplocCascade], frames: np.ndarray, cp: CascadeParams,
                 iou: float = 0.1, min_face: int = 50, eye_perturbs: int = 50, flp_perturbs: int = 63,
                 randoms_for: Optional[Callable[[int, int], np.ndarray]] = None) -> List[List[Face]]:
    """The frames are uploaded ONCE (DeviceFrames) and stay resident; then: one batched RunCascade, one batched
    ClusterDetections, ONE RunDetector launch for the eye seeds of all faces of all frames, and one launch per landmark
    cascade for all faces, both flips, all frames.  Per-call results are identical to calling RunDetector /
    GetLandmarkPoint face by face as the reference's test does (each seed carries its own randoms / RNG key)."""
    from . import DeviceFrames, landmark_seed_host
    frames = np.ascontiguousarray(frames, dtype=np.uint8)
    nf = frames.shape[0]
    rows, cols, dim = cp.ImageParams.Rows, cp.ImageParams.Cols, cp.ImageParams.Dim
    df = DeviceFrames(frames)
    try:
        dets, cnt = clf.RunCascadeBatch(df, cp, 0.0)
        clusters, ncl = clf.cluster_batch_array(dets, cnt, iou)
        calls = landmark_calls()
        out: List[List[Face]] = []
        big = []            # (frame, face index, call-index base)
        for f in range(nf):
            faces = [Face((int(c["row"]), int(c["col"]), int(c["scale"]), float(c["q"]))) for c in clusters[f, :ncl[f]]]
            out.append(faces)
            # call indices follow the reference's sequential order inside a frame: per face 2 eye calls, then 15 landmark calls
            nb = 0
            for k, fc in enumerate(faces):
                if fc.det[2] > min_face:
                    big.append((f, k, nb * (2 + len(calls))))
                    nb += 1
        if not big:
            return out

        def run(casc, seeds, seed_frames, flips, rnds, key):
            return casc.run_detector_frames(seeds, seed_frames, df.ptr, nf, df.stride, rows, cols, dim, 0.0, flips,
                                            np.stack(rnds) if randoms_for else None, rng_seed=key, frames_on_device=True)

        seeds, sfr, rnds = [], [], []
        for f, k, base in big:
            r, c, sc, _ = out[f][k].det
            ls, rs = eye_seeds(r, c, sc, eye_perturbs)
            seeds += [ls, rs]; sfr += [f, f]
            if randoms_for:
                rnds += [randoms_for(f, base), randoms_for(f, base + 1)]
        eyes = run(plc, seeds, sfr, [False] * len(seeds), rnds, 1)
        for i, (f, k, base) in enumerate(big):
            out[f][k].left_eye, out[f][k].right_eye = eyes[2 * i], eyes[2 * i + 1]
            out[f][k].landmarks = [None] * len(calls)
        for name in sorted(set(n for n, _ in calls)):
            seeds, sfr, flips, rnds, where = [], [], [], [], []
            for f, k, base in big:
                fc = out[f][k]
                for ci, (n, flip) in enumerate(calls):
                    if n != name:
                        continue
                    seeds.append(landmark_seed_host(fc.left_eye, fc.right_eye, flp_perturbs))
                    sfr.append(f); flips.append(flip); where.append((f, k, ci))
                    if randoms_for:
                        rnds.append(randoms_for(f, base + 2 + ci))
            pts = run(flpcs[name], seeds, sfr, flips, rnds, 7)
            for (f, k, ci), p in zip(where, pts):
                out[f][k].landmarks[ci] = p
        return out
    finally:
        df.free()


# ---- the same sequence on the device: ONE library call, no host round trips (pigo_detect_batch) --------------------------
def landmark_call_arrays(flpcs: Dict[str, PuplocCascade]):
    """(handles[ncalls], flips[ncalls]) of the reference's 15-call landmark sequence (core/flploc_test.go:122-146)."""
    import ctypes as C
    calls = landmark_calls()
    hs = (C.c_void_p * len(calls))(*[flpcs[n]._h.value if isinstance(flpcs[n]._h, C.c_void_p) else flpcs[n]._h for n, _ in calls])
    fl = np.array([1 if f else 0 for _, f in calls], dtype=np.uint8)
    return hs, fl


def detect_batch_device(clf: Pigo, plc: PuplocCascade, flpcs: Dict[str, PuplocCascade], frames, cp: CascadeParams, iou: float = 0.1,
                        min_face: int = 50, eye_perturbs: int = 50, flp_perturbs: int = 63, face_cap: int = 32, angle: float = 0.0,
                        randoms: Optional[np.ndarray] = None, rng_seed: int = 0, sharded: bool = False, det_cap: int = 0,
                        raw: bool = False):
    """face -> cluster -> pupils -> 15 landmarks for a frame batch with the sequencing on the device.
    frames: (N, Rows, Dim) uint8 host array, or a DeviceFrames.  randoms: optional [N][face_cap][17][63][3] float32.
    Returns List[List[Face]] like detect_batch (raw=True: the (faces, n_faces, points) arrays)."""
    import ctypes as C
    from . import DET_DTYPE, POINT_DTYPE, FRAMES_DEVICE, MEM_HOST, PIGO_E_CAP, DeviceFrames, PipelineParams, _check, lib
    hs, fl = landmark_call_arrays(flpcs)
    ncalls = len(fl)
    on_dev = isinstance(frames, DeviceFrames)
    if on_dev:
        nf, stride, fptr = frames.nframes, frames.stride, frames.ptr
    else:
        frames = np.ascontiguousarray(frames, dtype=np.uint8)
        nf, stride, fptr = frames.shape[0], frames.strides[0], frames.ctypes.data
    img = cp.ImageParams
    prm = PipelineParams(cp.MinSize, cp.MaxSize, cp.ShiftFactor, cp.ScaleFactor, angle, iou, min_face, eye_perturbs, flp_perturbs, det_cap)
    rnd = None
    if randoms is not None:
        rnd = np.ascontiguousarray(randoms, dtype=np.float32)
        assert rnd.size == nf * face_cap * (2 + ncalls) * 189, "randoms must be [N][face_cap][2+ncalls][63][3]"
    faces = np.zeros((nf, face_cap), dtype=DET_DTYPE)
    nfaces = np.zeros(max(nf, 1), dtype=np.int32)
    points = np.zeros((nf, face_cap, 2 + ncalls), dtype=POINT_DTYPE)
    L = lib()
    if sharded:
        rc = L.pigo_detect_batch_sharded(clf._h, plc._h, hs, fl.ctypes.data, ncalls, fptr, nf, stride, img.Rows, img.Cols, img.Dim, C.byref(prm),
                                         rnd.ctypes.data if rnd is not None else None, rng_seed, faces.ctypes.data, face_cap,
                                         nfaces.ctypes.data, points.ctypes.data)
    else:
        rc = L.pigo_detect_batch(clf._h, plc._h, hs, fl.ctypes.data, ncalls, fptr, nf, stride, img.Rows, img.Cols, img.Dim, C.byref(prm),
                                 rnd.ctypes.data if rnd is not None else None, rng_seed, faces.ctypes.data, face_cap, nfaces.ctypes.data,
                                 points.ctypes.data, FRAMES_DEVICE if on_dev else MEM_HOST, None)
    _check(rc)
    if raw:
        return faces, nfaces[:nf], points
    return _faces_of(faces, nfaces, points, min_face)


def _faces_of(faces, nfaces, points, min_face) -> List[List[Face]]:
    out: List[List[Face]] = []
    for f in range(len(faces)):
        fl_ = []
        for k in range(int(nfaces[f])):
            d = faces[f, k]
            fc = Face((int(d["row"]), int(d["col"]), int(d["scale"]), float(d["q"])))
            if d["scale"] > min_face:
                pts = [Puploc(int(p["row"]), int(p["col"]), float(np.float32(p["scale"])), int(p["perturbs"])) for p in points[f, k]]
                fc.left_eye, fc.right_eye, fc.landmarks = pts[0], pts[1], pts[2:]
            fl_.append(fc)
        out.append(fl_)
    return out


def detect_images_device(clf: Pigo, plc: PuplocCascade, flpcs: Dict[str, PuplocCascade], images, cp: CascadeParams, iou: float = 0.1,
                         min_face: int = 50, eye_perturbs: int = 50, flp_perturbs: int = 63, face_cap: int = 32, angle: float = 0.0,
                         randoms: Optional[np.ndarray] = None, rng_seed: int = 0, det_cap: int = 0, raw: bool = False):
    """detect_batch_device for images of different sizes in one call (pigo_detect_images).  images: ImageParams with host
    arrays, or for every image alike device pointers (int) holding Rows*Dim bytes; cp's MinSize / MaxSize / ShiftFactor /
    ScaleFactor are shared (cp.ImageParams is not used).  randoms: optional [N][face_cap][17][63][3] float32.
    Returns List[List[Face]] (raw=True: the (faces, n_faces, points) arrays)."""
    return _detect_images(clf, plc, flpcs, images, cp, iou, min_face, eye_perturbs, flp_perturbs, face_cap, angle, None, randoms, rng_seed,
                          det_cap, raw)


def detect_images_angles_device(clf: Pigo, plc: PuplocCascade, flpcs: Dict[str, PuplocCascade], images, cp: CascadeParams, angles,
                                iou: float = 0.1, min_face: int = 50, eye_perturbs: int = 50, flp_perturbs: int = 63, face_cap: int = 32,
                                randoms: Optional[np.ndarray] = None, rng_seed: int = 0, det_cap: int = 0, raw: bool = False):
    """detect_images_device with image i scanned and its eyes refined at angles[i] (pigo_detect_images_angles); the landmark
    calls stay at angle 0.  An angle sweep is one call: list an image once per angle (its host pixels are copied once)."""
    if len(angles) != len(images):
        raise ValueError("angles must have one entry per image")
    return _detect_images(clf, plc, flpcs, images, cp, iou, min_face, eye_perturbs, flp_perturbs, face_cap, 0.0, angles, randoms, rng_seed,
                          det_cap, raw)


def detect_images_sweep_device(clf: Pigo, plc: PuplocCascade, flpcs: Dict[str, PuplocCascade], images, cp: CascadeParams, angles,
                               iou: float = 0.1, min_face: int = 50, eye_perturbs: int = 50, flp_perturbs: int = 63, face_cap: int = 32,
                               randoms: Optional[np.ndarray] = None, rng_seed: int = 0, det_cap: int = 0, raw: bool = False):
    """Every image scanned at every angle of `angles`, one merged face list per image (pigo_detect_images_sweep): each face is
    refined with its eyes at the angle it was found at (the landmark calls stay at angle 0).  images as detect_images_device;
    randoms: optional [N][face_cap][17][63][3] float32.  Returns List[List[(Face, angle)]] with `angle` the listed value
    (raw=True: the (faces, n_faces, points, face_angle) arrays, face_angle indexing `angles`)."""
    import ctypes as C
    from . import DET_DTYPE, POINT_DTYPE, PipelineParams, _check, _image_table, lib
    hs, fl = landmark_call_arrays(flpcs)
    ncalls = len(fl)
    n = len(images)
    desc, flags, keep = _image_table(images)
    ang = np.ascontiguousarray(angles, dtype=np.float64)
    prm = PipelineParams(cp.MinSize, cp.MaxSize, cp.ShiftFactor, cp.ScaleFactor, 0.0, iou, min_face, eye_perturbs, flp_perturbs, det_cap)
    rnd = None
    if randoms is not None:
        rnd = np.ascontiguousarray(randoms, dtype=np.float32)
        assert rnd.size == n * face_cap * (2 + ncalls) * 189, "randoms must be [N][face_cap][2+ncalls][63][3]"
    faces = np.zeros((n, face_cap), dtype=DET_DTYPE)
    nfaces = np.zeros(max(n, 1), dtype=np.int32)
    points = np.zeros((n, face_cap, 2 + ncalls), dtype=POINT_DTYPE)
    face_angle = np.full((n, face_cap), -1, dtype=np.int32)
    _check(lib().pigo_detect_images_sweep(clf._h, plc._h, hs, fl.ctypes.data, ncalls, desc, n, ang.ctypes.data, len(ang), C.byref(prm),
                                          rnd.ctypes.data if rnd is not None else None, rng_seed, faces.ctypes.data, face_angle.ctypes.data,
                                          face_cap, nfaces.ctypes.data, points.ctypes.data, flags, None))
    if raw:
        return faces, nfaces[:n], points, face_angle
    return [[(fc, float(ang[face_angle[i, k]])) for k, fc in enumerate(row)] for i, row in enumerate(_faces_of(faces, nfaces, points, min_face))]


def detect_images_sweep_device_ptrs(clf: Pigo, plc: PuplocCascade, flpcs: Dict[str, PuplocCascade], images, angles, prm, faces_ptr: int,
                                    face_angle_ptr: int, face_cap: int, nfaces_ptr: int, points_ptr: int, randoms_ptr: int = 0,
                                    rng_seed: int = 0, stream: int = 0):
    """Fully device-resident, asynchronous pigo_detect_images_sweep: images = [(device pointer, rows, cols, dim)], prm a
    PipelineParams, every output a device pointer (face_angle_ptr 0 = not wanted); no host sync."""
    from . import FRAMES_DEVICE, OUT_DEVICE, _check, image_descs, lib
    import ctypes as C
    hs, fl = landmark_call_arrays(flpcs)
    ang = np.ascontiguousarray(angles, dtype=np.float64)
    _check(lib().pigo_detect_images_sweep(clf._h, plc._h, hs, fl.ctypes.data, len(fl), image_descs(images), len(images), ang.ctypes.data, len(ang),
                                          C.byref(prm), randoms_ptr or None, rng_seed, faces_ptr, face_angle_ptr or None, face_cap, nfaces_ptr,
                                          points_ptr, FRAMES_DEVICE | OUT_DEVICE, stream or None))


def detect_images_sharded(clf: Pigo, plc: PuplocCascade, flpcs: Dict[str, PuplocCascade], images, cp: CascadeParams, angles=None,
                          iou: float = 0.1, min_face: int = 50, eye_perturbs: int = 50, flp_perturbs: int = 63, face_cap: int = 32,
                          angle: float = 0.0, randoms: Optional[np.ndarray] = None, rng_seed: int = 0, det_cap: int = 0, raw: bool = False):
    """detect_images_angles_device over the devices of init_devices (pigo_detect_images_sharded): host images cut into
    contiguous shards of about equal modelled cost; angles None = every image at `angle`.  Results, generator keys and
    injected randoms are those of the single-device call, byte for byte."""
    if angles is not None and len(angles) != len(images):
        raise ValueError("angles must have one entry per image")
    return _detect_images(clf, plc, flpcs, images, cp, iou, min_face, eye_perturbs, flp_perturbs, face_cap, angle, angles, randoms, rng_seed,
                          det_cap, raw, sharded=True)


def _detect_images(clf, plc, flpcs, images, cp, iou, min_face, eye_perturbs, flp_perturbs, face_cap, angle, angles, randoms, rng_seed, det_cap,
                   raw, sharded=False, sources=None):
    import ctypes as C
    from . import DET_DTYPE, POINT_DTYPE, FRAMES_DEVICE, MEM_HOST, PipelineParams, _check, _image_table, lib
    from . import decoded_descs
    hs, fl = landmark_call_arrays(flpcs)
    ncalls = len(fl)
    if sources is not None:   # decoded sources (host planes): converted on the devices by the call
        n = len(sources)
        desc = decoded_descs(sources)
        flags = MEM_HOST
    else:
        n = len(images)
        desc, flags, keep = _image_table(images)
    prm = PipelineParams(cp.MinSize, cp.MaxSize, cp.ShiftFactor, cp.ScaleFactor, angle, iou, min_face, eye_perturbs, flp_perturbs, det_cap)
    rnd = None
    if randoms is not None:
        rnd = np.ascontiguousarray(randoms, dtype=np.float32)
        assert rnd.size == n * face_cap * (2 + ncalls) * 189, "randoms must be [N][face_cap][2+ncalls][63][3]"
    faces = np.zeros((n, face_cap), dtype=DET_DTYPE)
    nfaces = np.zeros(max(n, 1), dtype=np.int32)
    points = np.zeros((n, face_cap, 2 + ncalls), dtype=POINT_DTYPE)
    rptr = rnd.ctypes.data if rnd is not None else None
    if sharded:
        if flags == FRAMES_DEVICE:
            raise ValueError("the sharded calls take host images")
        ang = np.ascontiguousarray(angles, dtype=np.float64) if angles is not None else None
        fn = lib().pigo_detect_decoded_sharded if sources is not None else lib().pigo_detect_images_sharded
        _check(fn(clf._h, plc._h, hs, fl.ctypes.data, ncalls, desc, n, ang.ctypes.data if ang is not None else None, C.byref(prm), rptr, rng_seed,
                  faces.ctypes.data, face_cap, nfaces.ctypes.data, points.ctypes.data))
    elif angles is None:
        _check(lib().pigo_detect_images(clf._h, plc._h, hs, fl.ctypes.data, ncalls, desc, n, C.byref(prm), rptr, rng_seed, faces.ctypes.data,
                                        face_cap, nfaces.ctypes.data, points.ctypes.data, flags, None))
    else:
        ang = np.ascontiguousarray(angles, dtype=np.float64)
        _check(lib().pigo_detect_images_angles(clf._h, plc._h, hs, fl.ctypes.data, ncalls, desc, n, ang.ctypes.data, C.byref(prm), rptr,
                                               rng_seed, faces.ctypes.data, face_cap, nfaces.ctypes.data, points.ctypes.data, flags, None))
    if raw:
        return faces, nfaces[:n], points
    return _faces_of(faces, nfaces, points, min_face)


def detect_decoded(clf: Pigo, plc: PuplocCascade, flpcs: Dict[str, PuplocCascade], sources, cp: CascadeParams, angles=None, iou: float = 0.1,
                   min_face: int = 50, eye_perturbs: int = 50, flp_perturbs: int = 63, face_cap: int = 32, randoms: Optional[np.ndarray] = None,
                   rng_seed: int = 0, det_cap: int = 0, raw: bool = False, device_sources: bool = False, sharded: bool = False):
    """Go's DetectDecoded: RgbToGrayscale(ImgToNRGBA(img)) of every DecodedImage in one pigo_gray_images call, then
    detect_images_angles_device on the device arena (angles None = every image at 0).  Returns what
    detect_images_angles_device returns for the oracle-made gray images with Dim = Cols.  sharded=True: the same result
    from pigo_detect_decoded_sharded, every device of init_devices converting and detecting its own shard of the (host)
    sources."""
    if sharded:
        if device_sources:
            raise ValueError("the sharded call takes host sources")
        if angles is not None and len(angles) != len(sources):
            raise ValueError("angles must have one entry per image")
        angles = [0.0] * len(sources) if angles is None else angles
        return _detect_images(clf, plc, flpcs, None, cp, iou, min_face, eye_perturbs, flp_perturbs, face_cap, 0.0, angles, randoms, rng_seed,
                              det_cap, raw, sharded=True, sources=sources)
    from . import gray_images
    arena, images = gray_images(sources, device_sources=device_sources)
    angles = [0.0] * len(images) if angles is None else angles
    out = detect_images_angles_device(clf, plc, flpcs, images, cp, angles, iou, min_face, eye_perturbs, flp_perturbs, face_cap, randoms,
                                      rng_seed, det_cap, raw)
    del arena   # the call above returns after its results are on the host
    return out

