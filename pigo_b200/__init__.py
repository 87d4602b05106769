"""pigo_b200 -- host-side mirror (Python/ctypes) of the pigo Go API over libpigo_b200.so.

The product is the C-ABI library (include/pigo_b200.h, hand-written sm_90a CUDA).  The reference's
host language is Go, so the Go shim lives in go/pigo/ (see INTEGRATION.md) and THIS module is the mirror the tests and bench.py drive.
Names follow the reference (core/pigo.go, core/puploc.go, core/flploc.go):

    Pigo / NewPigo().Unpack(bytes)            core/pigo.go:46-110
    Pigo.RunCascade(CascadeParams, angle)     core/pigo.go:212-258
    Pigo.ClusterDetections(dets, iou)         core/pigo.go:262-308
    PuplocCascade.UnpackCascade / RunDetector core/puploc.go:38-103, :239-277
    PuplocCascade.UnpackFlp / GetLandmarkPoint / ReadCascadeDir   core/flploc.go:27-81
    CascadeParams, ImageParams, Detection, Puploc, FlpCascade     same exported fields

There is NO CPU fallback: importing works anywhere (so that CPU-only checks can verify the exported
symbols), but every compute call needs the CUDA library and an sm_90 (H100) device and raises otherwise.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libpigo_b200.so")
DATA_DIR = os.path.join(_HERE, "data")
CASCADE_DIR = os.path.join(DATA_DIR, "cascade")

PIGO_OK, PIGO_E_INVALID, PIGO_E_CUDA, PIGO_E_CAP, PIGO_E_NOMEM, PIGO_E_NODEVICE = 0, -1, -2, -3, -4, -5
MEM_HOST, FRAMES_DEVICE, OUT_DEVICE = 0, 1, 2

DET_DTYPE = np.dtype([("row", "<i4"), ("col", "<i4"), ("scale", "<i4"), ("q", "<f4")])
POINT_DTYPE = np.dtype([("row", "<i4"), ("col", "<i4"), ("scale", "<f4"), ("perturbs", "<i4")])

# every symbol include/pigo_b200.h declares (checked by tests/test_abi.py)
ABI_SYMBOLS = [
    "pigo_last_error", "pigo_version", "pigo_init", "pigo_shutdown", "pigo_launch_count", "pigo_alloc_pinned",
    "pigo_free_pinned", "pigo_cascade_create", "pigo_cascade_destroy", "pigo_cascade_info", "pigo_scale_ladder",
    "pigo_count_windows", "pigo_run_cascade", "pigo_run_cascade_batch", "pigo_cluster", "pigo_cluster_batch",
    "pigo_puploc_create", "pigo_puploc_destroy", "pigo_puploc_info", "pigo_puploc_run", "pigo_get_landmark_point",
    "pigo_set_option", "pigo_get_option", "pigo_rgba_to_gray", "pigo_puploc_run_frames", "pigo_device_alloc",
    "pigo_device_free", "pigo_device_upload", "pigo_describe_plan", "pigo_init_devices", "pigo_device_count",
    "pigo_device_download", "pigo_run_cascade_batch_sharded", "pigo_detect_batch", "pigo_detect_batch_sharded",
    "pigo_ycbcr_to_nrgba",
]


class PigoError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"libpigo_b200 status {status}: {msg}")
        self.status = status


_lib = None


def lib() -> C.CDLL:
    """Loads libpigo_b200.so (built by pigo_b200/build.py or __graft_entry__.build()); raises if absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            # not built yet (fresh checkout): compile it in-tree with nvcc; there is no CPU or PyTorch fallback, so a
            # missing toolchain is a hard error
            try:
                from . import build as _build
                _build.build()
            except Exception as e:
                raise ImportError(f"{LIB_PATH} is missing and could not be built with nvcc ({e}); "
                                  "there is no CPU or PyTorch fallback for the detection path") from e
        L = C.CDLL(LIB_PATH)
        vp, i, d, u64, sz = C.c_void_p, C.c_int, C.c_double, C.c_uint64, C.c_size_t
        L.pigo_last_error.restype = C.c_char_p
        L.pigo_launch_count.restype = C.c_int64
        L.pigo_init.argtypes = [i]
        L.pigo_alloc_pinned.argtypes = [C.POINTER(vp), sz]
        L.pigo_free_pinned.argtypes = [vp]
        L.pigo_cascade_create.argtypes = [C.c_char_p, sz, C.POINTER(vp)]
        L.pigo_cascade_destroy.argtypes = [vp]
        L.pigo_cascade_destroy.restype = None
        L.pigo_cascade_info.argtypes = [vp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.pigo_scale_ladder.argtypes = [i, i, d, vp, i, C.POINTER(i)]
        L.pigo_count_windows.argtypes = [i, i, i, i, d, d]
        L.pigo_count_windows.restype = C.c_int64
        L.pigo_run_cascade.argtypes = [vp, vp, i, i, i, i, i, d, d, d, vp, i, C.POINTER(i)]
        L.pigo_run_cascade_batch.argtypes = [vp, vp, i, sz, i, i, i, i, i, d, d, d, vp, i, vp, C.c_uint, vp]
        L.pigo_cluster.argtypes = [vp, i, d, vp, i, C.POINTER(i)]
        L.pigo_cluster_batch.argtypes = [vp, vp, i, i, d, vp, i, vp, C.c_uint, vp]
        L.pigo_puploc_create.argtypes = [C.c_char_p, sz, C.POINTER(vp)]
        L.pigo_puploc_destroy.argtypes = [vp]
        L.pigo_puploc_destroy.restype = None
        L.pigo_puploc_info.argtypes = [vp, C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.pigo_puploc_run.argtypes = [vp, vp, i, vp, u64, vp, i, i, i, d, vp, vp, C.c_uint, vp]
        L.pigo_get_landmark_point.argtypes = [vp, vp, vp, vp, i, i, i, i, i, vp, u64, vp]
        L.pigo_rgba_to_gray.argtypes = [vp, sz, vp, C.c_uint, vp]
        L.pigo_puploc_run_frames.argtypes = [vp, vp, i, vp, vp, u64, vp, i, sz, i, i, i, d, vp, vp, C.c_uint, vp]
        L.pigo_device_alloc.argtypes = [C.POINTER(vp), sz]
        L.pigo_device_free.argtypes = [vp]
        L.pigo_device_upload.argtypes = [vp, vp, sz]
        L.pigo_describe_plan.argtypes = [i, i, i, i, d, d, C.c_char_p, sz]
        L.pigo_init_devices.argtypes = [C.c_uint]
        L.pigo_device_download.argtypes = [vp, vp, sz]
        L.pigo_run_cascade_batch_sharded.argtypes = [vp, vp, i, sz, i, i, i, i, i, d, d, d, vp, i, vp]
        L.pigo_detect_batch.argtypes = [vp, vp, vp, vp, i, vp, i, sz, i, i, i, vp, vp, u64, vp, i, vp, vp, C.c_uint, vp]
        L.pigo_detect_batch_sharded.argtypes = [vp, vp, vp, vp, i, vp, i, sz, i, i, i, vp, vp, u64, vp, i, vp, vp]
        L.pigo_ycbcr_to_nrgba.argtypes = [vp, vp, vp, i, i, i, i, i, i, i, vp, vp, C.c_uint, vp]
        L.pigo_set_option.argtypes = [C.c_char_p, C.c_int64]
        L.pigo_get_option.argtypes = [C.c_char_p]
        L.pigo_get_option.restype = C.c_int64
        _lib = L
    return _lib


def _check(rc: int):
    if rc != PIGO_OK:
        raise PigoError(rc, lib().pigo_last_error().decode("utf-8", "replace"))


def init(device: int = 0):
    _check(lib().pigo_init(device))


def init_devices(mask: int):
    """Selects the devices of the *_sharded entry points (bit d = device d); SURVEY.md section 8e."""
    _check(lib().pigo_init_devices(mask))


def device_count() -> int:
    return int(lib().pigo_device_count())


def set_option(name: str, value: int):
    _check(lib().pigo_set_option(name.encode(), int(value)))


def get_option(name: str) -> int:
    return int(lib().pigo_get_option(name.encode()))


def launch_count() -> int:
    return int(lib().pigo_launch_count())


def describe_plan(rows, cols, min_size, max_size, shift_factor, scale_factor) -> dict:
    """Host-only view of the scan schedule (tile bands, tile geometry, gather scales) for this geometry."""
    import json
    buf = C.create_string_buffer(1 << 20)
    _check(lib().pigo_describe_plan(rows, cols, min_size, max_size, shift_factor, scale_factor, buf, len(buf)))
    return json.loads(buf.value.decode())


def count_windows(rows, cols, min_size, max_size, shift_factor, scale_factor) -> int:
    return int(lib().pigo_count_windows(rows, cols, min_size, max_size, shift_factor, scale_factor))


def scale_ladder(min_size, max_size, scale_factor) -> List[int]:
    n = C.c_int()
    _check(lib().pigo_scale_ladder(min_size, max_size, scale_factor, None, 0, C.byref(n)))
    buf = np.zeros(max(n.value, 1), dtype=np.int32)
    _check(lib().pigo_scale_ladder(min_size, max_size, scale_factor, buf.ctypes.data, n.value, C.byref(n)))
    return buf[:n.value].tolist()


# ---- the reference's exported types (core/pigo.go:16-34, :195-200; core/puploc.go:14-19) -------------------
@dataclass
class ImageParams:
    Pixels: np.ndarray = None   # []uint8, row-major, stride Dim
    Rows: int = 0
    Cols: int = 0
    Dim: int = 0


@dataclass
class CascadeParams:
    ImageParams: ImageParams = field(default_factory=ImageParams)
    MinSize: int = 0
    MaxSize: int = 0
    ShiftFactor: float = 0.0
    ScaleFactor: float = 0.0


@dataclass
class Detection:
    Row: int = 0
    Col: int = 0
    Scale: int = 0
    Q: float = 0.0


@dataclass
class Puploc:
    Row: int = 0
    Col: int = 0
    Scale: float = 0.0
    Perturbs: int = 0


def _dets_to_array(dets) -> np.ndarray:
    if isinstance(dets, np.ndarray) and dets.dtype == DET_DTYPE:
        return np.ascontiguousarray(dets)
    a = np.zeros(len(dets), dtype=DET_DTYPE)
    for k, dd in enumerate(dets):
        a[k] = (dd.Row, dd.Col, dd.Scale, dd.Q)
    return a


def _array_to_dets(a: np.ndarray) -> List[Detection]:
    return [Detection(int(x["row"]), int(x["col"]), int(x["scale"]), float(np.float32(x["q"]))) for x in a]


def _pixels(img: ImageParams) -> np.ndarray:
    p = np.ascontiguousarray(img.Pixels, dtype=np.uint8).reshape(-1)
    if p.size < (img.Rows - 1) * img.Dim + img.Cols and img.Rows > 0:
        raise ValueError("Pixels shorter than Rows*Dim")   # the reference would panic with index out of range
    return p


class Pigo:
    """pigo.Pigo (core/pigo.go:37-43): the face classifier; tables live on the device."""

    def __init__(self):
        self._h = None

    def Unpack(self, packet: bytes) -> "Pigo":
        """(*Pigo).Unpack, core/pigo.go:51-110.  Returns a new classifier like the reference does."""
        h = C.c_void_p()
        _check(lib().pigo_cascade_create(bytes(packet), len(packet), C.byref(h)))
        p = Pigo()
        p._h = h
        d, n = C.c_uint32(), C.c_uint32()
        lib().pigo_cascade_info(h, C.byref(d), C.byref(n))
        p.treeDepth, p.treeNum = d.value, n.value
        return p

    def __del__(self):
        if getattr(self, "_h", None) is not None and _lib is not None:
            _lib.pigo_cascade_destroy(self._h)
            self._h = None

    def _need(self):
        if self._h is None:
            raise PigoError(PIGO_E_INVALID, "classifier not unpacked")

    # -- RunCascade --------------------------------------------------------------------------------------
    def run_cascade_array(self, cp: CascadeParams, angle: float, cap: int = 1024) -> np.ndarray:
        """RunCascade returning a DET_DTYPE array (retries on PIGO_E_CAP)."""
        self._need()
        img = cp.ImageParams
        pix = _pixels(img)
        while True:
            out = np.zeros(max(cap, 1), dtype=DET_DTYPE)
            n = C.c_int()
            rc = lib().pigo_run_cascade(self._h, pix.ctypes.data, img.Rows, img.Cols, img.Dim, cp.MinSize, cp.MaxSize,
                                        cp.ShiftFactor, cp.ScaleFactor, angle, out.ctypes.data, cap, C.byref(n))
            if rc == PIGO_E_CAP:
                cap = int(n.value)
                continue
            _check(rc)
            return out[:n.value].copy()

    def RunCascade(self, cp: CascadeParams, angle: float) -> List[Detection]:
        """(*Pigo).RunCascade, core/pigo.go:212-258."""
        return _array_to_dets(self.run_cascade_array(cp, angle))

    def RunCascadeBatch(self, frames, cp: CascadeParams, angle: float = 0.0, cap_per_frame: int = 1024):
        """Additive batch entry point: frames is (N, Rows, Dim) uint8 on the host, or a DeviceFrames.
        Returns (dets[N, cap] DET_DTYPE, counts[N])."""
        self._need()
        img = cp.ImageParams
        on_dev = isinstance(frames, DeviceFrames)
        if on_dev:
            nf, stride, fptr = frames.nframes, frames.stride, frames.ptr
        else:
            frames = np.ascontiguousarray(frames, dtype=np.uint8)
            nf = frames.shape[0]
            stride = frames.strides[0] if nf > 0 else 0
            fptr = frames.ctypes.data
        while True:
            out = np.zeros((nf, max(cap_per_frame, 1)), dtype=DET_DTYPE)
            cnt = np.zeros(max(nf, 1), dtype=np.int32)
            rc = lib().pigo_run_cascade_batch(self._h, fptr, nf, stride, img.Rows, img.Cols, img.Dim,
                                              cp.MinSize, cp.MaxSize, cp.ShiftFactor, cp.ScaleFactor, angle,
                                              out.ctypes.data, cap_per_frame, cnt.ctypes.data,
                                              FRAMES_DEVICE if on_dev else MEM_HOST, None)
            if rc == PIGO_E_CAP:
                cap_per_frame = int(cnt.max())
                continue
            _check(rc)
            return out, cnt[:nf]

    def RunCascadeBatchSharded(self, frames: np.ndarray, cp: CascadeParams, angle: float = 0.0, cap_per_frame: int = 1024):
        """RunCascadeBatch over the devices of init_devices (host frames; identical result)."""
        self._need()
        img = cp.ImageParams
        frames = np.ascontiguousarray(frames, dtype=np.uint8)
        nf = frames.shape[0]
        while True:
            out = np.zeros((nf, max(cap_per_frame, 1)), dtype=DET_DTYPE)
            cnt = np.zeros(max(nf, 1), dtype=np.int32)
            rc = lib().pigo_run_cascade_batch_sharded(self._h, frames.ctypes.data, nf, frames.strides[0] if nf else 0, img.Rows, img.Cols,
                                                      img.Dim, cp.MinSize, cp.MaxSize, cp.ShiftFactor, cp.ScaleFactor, angle,
                                                      out.ctypes.data, cap_per_frame, cnt.ctypes.data)
            if rc == PIGO_E_CAP:
                cap_per_frame = int(cnt.max())
                continue
            _check(rc)
            return out, cnt[:nf]

    def run_cascade_batch_device(self, frames_ptr: int, nframes: int, frame_stride: int, rows: int, cols: int, dim: int,
                                 min_size: int, max_size: int, shift: float, scale: float, angle: float, out_ptr: int,
                                 cap_per_frame: int, counts_ptr: int, stream: int = 0):
        """Fully device-resident, asynchronous form (frames, out, counts are device pointers; no host sync)."""
        self._need()
        _check(lib().pigo_run_cascade_batch(self._h, frames_ptr, nframes, frame_stride, rows, cols, dim, min_size, max_size,
                                            shift, scale, angle, out_ptr, cap_per_frame, counts_ptr,
                                            FRAMES_DEVICE | OUT_DEVICE, stream or None))

    # -- ClusterDetections -----------------------------------------------------------------------------------
    def cluster_array(self, dets: np.ndarray, iou: float):
        """Returns (dets sorted in place by Q, clusters) as DET_DTYPE arrays."""
        d = np.ascontiguousarray(dets, dtype=DET_DTYPE)
        n = len(d)
        cap = max(n, 1)
        out = np.zeros(cap, dtype=DET_DTYPE)
        k = C.c_int()
        _check(lib().pigo_cluster(d.ctypes.data, n, iou, out.ctypes.data, cap, C.byref(k)))
        return d, out[:k.value].copy()

    def cluster_batch_array(self, dets: np.ndarray, counts: np.ndarray, iou: float):
        """ClusterDetections for every frame of a RunCascadeBatch result in one launch.
        dets: [N, cap] DET_DTYPE (sorted in place per frame), counts: [N].  Returns (clusters[N, cap], nclusters[N])."""
        d = np.ascontiguousarray(dets, dtype=DET_DTYPE)
        nf, cap = d.shape
        n = np.ascontiguousarray(np.minimum(counts, cap), dtype=np.int32)
        out = np.zeros((nf, max(cap, 1)), dtype=DET_DTYPE)
        k = np.zeros(max(nf, 1), dtype=np.int32)
        _check(lib().pigo_cluster_batch(d.ctypes.data, n.ctypes.data, nf, cap, iou, out.ctypes.data, cap, k.ctypes.data, MEM_HOST, None))
        if d is not dets and isinstance(dets, np.ndarray) and dets.shape == d.shape:
            dets[...] = d
        return out, k[:nf]

    def ClusterDetections(self, detections: List[Detection], iouThreshold: float) -> List[Detection]:
        """(*Pigo).ClusterDetections, core/pigo.go:262-308; sorts `detections` in place like the reference."""
        arr = _dets_to_array(detections)
        srt, cl = self.cluster_array(arr, iouThreshold)
        if isinstance(detections, list):
            detections[:] = _array_to_dets(srt)
        return _array_to_dets(cl)


def NewPigo() -> Pigo:
    """core/pigo.go:46."""
    return Pigo()


class PuplocCascade:
    """pigo.PuplocCascade (core/puploc.go:23-30)."""

    def __init__(self):
        self._h = None

    def UnpackCascade(self, packet: bytes) -> "PuplocCascade":
        """core/puploc.go:38-103."""
        h = C.c_void_p()
        _check(lib().pigo_puploc_create(bytes(packet), len(packet), C.byref(h)))
        p = PuplocCascade()
        p._h = h
        st, sc, tr, dp = C.c_uint32(), C.c_float(), C.c_uint32(), C.c_uint32()
        lib().pigo_puploc_info(h, C.byref(st), C.byref(sc), C.byref(tr), C.byref(dp))
        p.stages, p.scales, p.trees, p.treeDepth = st.value, sc.value, tr.value, dp.value
        return p

    def UnpackFlp(self, cf: str) -> "PuplocCascade":
        """core/flploc.go:27-33."""
        with open(cf, "rb") as f:
            return self.UnpackCascade(f.read())

    def ReadCascadeDir(self, path: str):
        """core/flploc.go:60-81: map name -> [FlpCascade]."""
        names = sorted(os.listdir(path))
        if not names:
            raise FileNotFoundError("the provided directory is empty")
        out = {}
        for nm in names:
            try:
                c, err = self.UnpackFlp(os.path.abspath(os.path.join(path, nm))), None
            except Exception as e:  # the reference stores the error next to the cascade
                c, err = None, e
            out.setdefault(nm, []).append(FlpCascade(c, err))
        return out

    def __del__(self):
        if getattr(self, "_h", None) is not None and _lib is not None:
            _lib.pigo_puploc_destroy(self._h)
            self._h = None

    def run_detector_batch(self, seeds: Sequence[Puploc], img: ImageParams, angle: float = 0.0,
                           flipv: Optional[Sequence[bool]] = None, randoms: Optional[np.ndarray] = None,
                           rng_seed: int = 0) -> List[Puploc]:
        if self._h is None:
            raise PigoError(PIGO_E_INVALID, "cascade not unpacked")
        n = len(seeds)
        s = np.zeros(max(n, 1), dtype=POINT_DTYPE)
        for k, p in enumerate(seeds):
            s[k] = (p.Row, p.Col, p.Scale, p.Perturbs)
        out = np.zeros(max(n, 1), dtype=POINT_DTYPE)
        pix = _pixels(img)
        rnd = None
        if randoms is not None:
            rnd = np.ascontiguousarray(randoms, dtype=np.float32)
            assert rnd.size == n * 63 * 3, "randoms must be [nseeds][63][3]"
        fl = None
        if flipv is not None:
            fl = np.ascontiguousarray(np.asarray(flipv, dtype=np.uint8))
        _check(lib().pigo_puploc_run(self._h, s.ctypes.data, n, rnd.ctypes.data if rnd is not None else None, rng_seed,
                                     pix.ctypes.data, img.Rows, img.Cols, img.Dim, angle,
                                     fl.ctypes.data if fl is not None else None, out.ctypes.data, MEM_HOST, None))
        return [Puploc(int(o["row"]), int(o["col"]), float(np.float32(o["scale"])), int(o["perturbs"])) for o in out[:n]]

    def run_detector_frames(self, seeds: Sequence[Puploc], seed_frame: Sequence[int], frames, nframes: int, frame_stride: int,
                            rows: int, cols: int, dim: int, angle: float = 0.0, flipv: Optional[Sequence[bool]] = None,
                            randoms: Optional[np.ndarray] = None, rng_seed: int = 0, frames_on_device: bool = False) -> List[Puploc]:
        """Batch over several frames: seed i refines on frame seed_frame[i].  `frames` is a host uint8 array, or a device
        pointer (int) when frames_on_device."""
        if self._h is None:
            raise PigoError(PIGO_E_INVALID, "cascade not unpacked")
        n = len(seeds)
        if n == 0:
            return []
        s = np.zeros(n, dtype=POINT_DTYPE)
        for k, p in enumerate(seeds):
            s[k] = (p.Row, p.Col, p.Scale, p.Perturbs)
        sf = np.ascontiguousarray(np.asarray(seed_frame, dtype=np.int32))
        out = np.zeros(n, dtype=POINT_DTYPE)
        rnd = np.ascontiguousarray(randoms, dtype=np.float32) if randoms is not None else None
        fl = np.ascontiguousarray(np.asarray(flipv, dtype=np.uint8)) if flipv is not None else None
        if frames_on_device:
            fptr = int(frames)
        else:
            fr = np.ascontiguousarray(frames, dtype=np.uint8)
            fptr = fr.ctypes.data
        _check(lib().pigo_puploc_run_frames(self._h, s.ctypes.data, n, sf.ctypes.data, rnd.ctypes.data if rnd is not None else None,
                                            rng_seed, fptr, nframes, frame_stride, rows, cols, dim, angle,
                                            fl.ctypes.data if fl is not None else None, out.ctypes.data,
                                            FRAMES_DEVICE if frames_on_device else MEM_HOST, None))
        return [Puploc(int(o["row"]), int(o["col"]), float(np.float32(o["scale"])), int(o["perturbs"])) for o in out]

    def RunDetector(self, pl: Puploc, img: ImageParams, angle: float, flipV: bool, randoms: Optional[np.ndarray] = None,
                    rng_seed: int = 0) -> Puploc:
        """(*PuplocCascade).RunDetector, core/puploc.go:239-277 (randoms: optional [63][3] float32 injection)."""
        return self.run_detector_batch([pl], img, angle, [flipV], randoms, rng_seed)[0]

    def GetLandmarkPoint(self, leftEye: Puploc, rightEye: Puploc, img: ImageParams, perturb: int, flipV: bool,
                         randoms: Optional[np.ndarray] = None, rng_seed: int = 0) -> Puploc:
        """core/flploc.go:36-57."""
        if self._h is None:
            raise PigoError(PIGO_E_INVALID, "cascade not unpacked")
        le = np.array([(leftEye.Row, leftEye.Col, leftEye.Scale, leftEye.Perturbs)], dtype=POINT_DTYPE)
        re_ = np.array([(rightEye.Row, rightEye.Col, rightEye.Scale, rightEye.Perturbs)], dtype=POINT_DTYPE)
        out = np.zeros(1, dtype=POINT_DTYPE)
        pix = _pixels(img)
        rnd = np.ascontiguousarray(randoms, dtype=np.float32) if randoms is not None else None
        _check(lib().pigo_get_landmark_point(self._h, le.ctypes.data, re_.ctypes.data, pix.ctypes.data, img.Rows, img.Cols,
                                             img.Dim, perturb, int(bool(flipV)), rnd.ctypes.data if rnd is not None else None,
                                             rng_seed, out.ctypes.data))
        o = out[0]
        return Puploc(int(o["row"]), int(o["col"]), float(np.float32(o["scale"])), int(o["perturbs"]))


def NewPuplocCascade() -> PuplocCascade:
    """core/puploc.go:33."""
    return PuplocCascade()


@dataclass
class FlpCascade:
    """core/flploc.go:12-15: embeds *PuplocCascade and an error."""
    PuplocCascade: Optional[PuplocCascade] = None
    error: Optional[Exception] = None

    def GetLandmarkPoint(self, *a, **k):
        return self.PuplocCascade.GetLandmarkPoint(*a, **k)


def landmark_seed_host(leftEye: Puploc, rightEye: Puploc, perturb: int) -> Puploc:
    """The float64 seed arithmetic of GetLandmarkPoint (core/flploc.go:37-50), for batching several calls into one launch."""
    import math
    dx = (leftEye.Row - rightEye.Row) ** 2
    dy = (leftEye.Col - rightEye.Col) ** 2
    dist = math.sqrt(float(dx + dy))
    row = float(leftEye.Row + rightEye.Row) / 2.0 + 0.25 * dist
    col = float(leftEye.Col + rightEye.Col) / 2.0 + 0.15 * dist
    return Puploc(int(row), int(col), float(np.float32(3.0 * dist)), perturb)


def RgbToGrayscale(rgba: np.ndarray) -> np.ndarray:
    """pigo.RgbToGrayscale, core/grayscale.go:8-23, for an NRGBA pixel array [..., 4] (R, G, B, A); returns uint8 [...]."""
    a = np.ascontiguousarray(rgba, dtype=np.uint8)
    if a.shape[-1] != 4:
        raise ValueError("expected [..., 4] NRGBA pixels")
    n = a.size // 4
    out = np.zeros(a.shape[:-1], dtype=np.uint8)
    _check(lib().pigo_rgba_to_gray(a.ctypes.data if n else None, n, out.ctypes.data if n else None, MEM_HOST, None))
    return out


class PipelineParams(C.Structure):
    """pigo_pipeline_params (include/pigo_b200.h)."""
    _fields_ = [("min_size", C.c_int32), ("max_size", C.c_int32), ("shift_factor", C.c_double), ("scale_factor", C.c_double),
                ("angle", C.c_double), ("iou_threshold", C.c_double), ("min_face_scale", C.c_int32), ("eye_perturbs", C.c_int32),
                ("flp_perturbs", C.c_int32), ("det_cap", C.c_int32)]


def YCbCrToNRGBA(y: np.ndarray, cb: np.ndarray, cr: np.ndarray, subsample: int, width: int, height: int, min_x: int = 0, min_y: int = 0,
                 want_gray: bool = False):
    """ImgToNRGBA for an *image.YCbCr (core/image.go:60-76): y is [height][YStride], cb/cr are [chroma rows][CStride] uint8 planes laid
    out like image.YCbCr for Rect (min_x, min_y)-(min_x+width, min_y+height); subsample = image.YCbCrSubsampleRatio (0..5).
    Returns nrgba [height][width][4] (and gray [height][width] = RgbToGrayscale of it when want_gray)."""
    y = np.ascontiguousarray(y, dtype=np.uint8); cb = np.ascontiguousarray(cb, dtype=np.uint8); cr = np.ascontiguousarray(cr, dtype=np.uint8)
    out = np.zeros((height, width, 4), dtype=np.uint8)
    gray = np.zeros((height, width), dtype=np.uint8) if want_gray else None
    _check(lib().pigo_ycbcr_to_nrgba(y.ctypes.data, cb.ctypes.data, cr.ctypes.data, y.shape[1] if y.ndim == 2 else width,
                                     cb.shape[1] if cb.ndim == 2 else 0, subsample, min_x, min_y, width, height,
                                     out.ctypes.data if out.size else None, gray.ctypes.data if want_gray and gray.size else None, MEM_HOST, None))
    return (out, gray) if want_gray else out


class DeviceFrames:
    """A frame batch kept resident on the device across calls (pigo_device_alloc/_upload/_free)."""

    def __init__(self, frames: np.ndarray):
        fr = np.ascontiguousarray(frames, dtype=np.uint8)
        self.nframes = fr.shape[0]
        self.stride = fr.strides[0] if fr.ndim == 3 else fr.size
        self.nbytes = fr.nbytes
        p = C.c_void_p()
        _check(lib().pigo_device_alloc(C.byref(p), self.nbytes))
        self.ptr = p.value
        _check(lib().pigo_device_upload(self.ptr, fr.ctypes.data, self.nbytes))

    def free(self):
        if getattr(self, "ptr", None):
            lib().pigo_device_free(self.ptr)
            self.ptr = None

    def __del__(self):
        if _lib is not None:
            self.free()


def load_cascade(name: str = "facefinder") -> bytes:
    """Reads one of the model files shipped under pigo_b200/data/cascade (copies of the reference's cascade/ data)."""
    with open(os.path.join(CASCADE_DIR, name), "rb") as f:
        return f.read()
