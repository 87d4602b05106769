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
MEM_HOST, FRAMES_DEVICE, OUT_DEVICE, FACES_DEVICE = 0, 1, 2, 4
DECODED_YCBCR, DECODED_NRGBA, DECODED_RGBA, DECODED_GRAY = 0, 1, 2, 3
DECODED_GRAY16, DECODED_RGBA64, DECODED_NRGBA64, DECODED_CMYK, DECODED_PALETTED = 5, 6, 7, 8, 9

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
    "pigo_ycbcr_to_nrgba", "pigo_run_cascade_images", "pigo_detect_images", "pigo_puploc_run_images",
    "pigo_run_cascade_images_angles", "pigo_detect_images_angles", "pigo_gray_images", "pigo_cascade_block_table",
    "pigo_run_cascade_images_sharded", "pigo_detect_images_sharded", "pigo_run_cascade_decoded_sharded", "pigo_detect_decoded_sharded",
    "pigo_shard_plan", "pigo_describe_plan_frames", "pigo_run_cascade_images_sweep", "pigo_detect_images_sweep",
    "pigo_run_cascade_images_params", "pigo_detect_images_params", "pigo_blur_faces", "pigo_blur_decoded",
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
        L.pigo_describe_plan_frames.argtypes = [i, i, i, i, d, d, i, C.c_char_p, sz]
        L.pigo_init_devices.argtypes = [C.c_uint]
        L.pigo_device_download.argtypes = [vp, vp, sz]
        L.pigo_run_cascade_batch_sharded.argtypes = [vp, vp, i, sz, i, i, i, i, i, d, d, d, vp, i, vp]
        L.pigo_run_cascade_images.argtypes = [vp, vp, i, i, i, d, d, d, vp, i, vp, C.c_uint, vp]
        L.pigo_detect_batch.argtypes = [vp, vp, vp, vp, i, vp, i, sz, i, i, i, vp, vp, u64, vp, i, vp, vp, C.c_uint, vp]
        L.pigo_detect_batch_sharded.argtypes = [vp, vp, vp, vp, i, vp, i, sz, i, i, i, vp, vp, u64, vp, i, vp, vp]
        L.pigo_detect_images.argtypes = [vp, vp, vp, vp, i, vp, i, vp, vp, u64, vp, i, vp, vp, C.c_uint, vp]
        L.pigo_puploc_run_images.argtypes = [vp, vp, i, vp, vp, u64, vp, i, d, vp, vp, C.c_uint, vp]
        L.pigo_run_cascade_images_angles.argtypes = [vp, vp, i, vp, i, i, d, d, vp, i, vp, C.c_uint, vp]
        L.pigo_detect_images_angles.argtypes = [vp, vp, vp, vp, i, vp, i, vp, vp, vp, u64, vp, i, vp, vp, C.c_uint, vp]
        L.pigo_ycbcr_to_nrgba.argtypes = [vp, vp, vp, i, i, i, i, i, i, i, vp, vp, C.c_uint, vp]
        L.pigo_gray_images.argtypes = [vp, i, vp, C.POINTER(sz), vp, C.c_uint, vp]
        L.pigo_set_option.argtypes = [C.c_char_p, C.c_int64]
        L.pigo_get_option.argtypes = [C.c_char_p]
        L.pigo_get_option.restype = C.c_int64
        L.pigo_cascade_block_table.argtypes = [vp, vp, C.POINTER(sz)]
        L.pigo_run_cascade_images_sharded.argtypes = [vp, vp, i, vp, i, i, d, d, vp, i, vp]
        L.pigo_detect_images_sharded.argtypes = [vp, vp, vp, vp, i, vp, i, vp, vp, vp, u64, vp, i, vp, vp]
        L.pigo_run_cascade_decoded_sharded.argtypes = [vp, vp, i, vp, i, i, d, d, vp, i, vp]
        L.pigo_detect_decoded_sharded.argtypes = [vp, vp, vp, vp, i, vp, i, vp, vp, vp, u64, vp, i, vp, vp]
        L.pigo_shard_plan.argtypes = [vp, i, vp, i, i, d, d, i, vp, C.POINTER(i)]
        L.pigo_run_cascade_images_sweep.argtypes = [vp, vp, i, vp, i, i, i, d, d, d, i, vp, vp, i, vp, C.c_uint, vp]
        L.pigo_detect_images_sweep.argtypes = [vp, vp, vp, vp, i, vp, i, vp, i, vp, vp, u64, vp, vp, i, vp, vp, C.c_uint, vp]
        L.pigo_run_cascade_images_params.argtypes = [vp, vp, i, vp, vp, vp, i, vp, C.c_uint, vp]
        L.pigo_detect_images_params.argtypes = [vp, vp, vp, vp, i, vp, i, vp, vp, vp, vp, u64, vp, i, vp, vp, C.c_uint, vp]
        L.pigo_blur_faces.argtypes = [vp, i, vp, i, vp, vp, C.c_uint, vp]
        L.pigo_blur_decoded.argtypes = [vp, vp, i, vp, vp, d, i, vp, vp, i, vp, C.c_uint, vp]
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


def describe_plan(rows, cols, min_size, max_size, shift_factor, scale_factor, nframes: Optional[int] = None) -> dict:
    """Host-only view of the scan schedule (tile bands, tile geometry, gather scales, tile role, band ratio) for this
    geometry, in a call of `nframes` frames (None: a call of many frames)."""
    import json
    buf = C.create_string_buffer(1 << 20)
    if nframes is None:
        _check(lib().pigo_describe_plan(rows, cols, min_size, max_size, shift_factor, scale_factor, buf, len(buf)))
    else:
        _check(lib().pigo_describe_plan_frames(rows, cols, min_size, max_size, shift_factor, scale_factor, nframes, buf, len(buf)))
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


class PigoImage(C.Structure):
    """pigo_image (include/pigo_b200.h): one image of a pigo_run_cascade_images call."""
    _fields_ = [("pixels", C.c_void_p), ("rows", C.c_int32), ("cols", C.c_int32), ("dim", C.c_int32)]


def image_descs(items) -> C.Array:
    """[(pixels pointer, rows, cols, dim)] -> the descriptor array pigo_run_cascade_images takes."""
    arr = (PigoImage * max(len(items), 1))()
    for k, (p, r, c, d) in enumerate(items):
        arr[k] = PigoImage(p, r, c, d)
    return arr


class PigoCascadeParams(C.Structure):
    """pigo_cascade_params (include/pigo_b200.h): pigo.CascadeParams without its ImageParams."""
    _fields_ = [("min_size", C.c_int32), ("max_size", C.c_int32), ("shift_factor", C.c_double), ("scale_factor", C.c_double)]


def cascade_params_array(items) -> C.Array:
    """[CascadeParams or (MinSize, MaxSize, ShiftFactor, ScaleFactor)] -> the pigo_cascade_params array of a per-image-parameter
    call (the CascadeParams' ImageParams are not read here)."""
    arr = (PigoCascadeParams * max(len(items), 1))()
    for k, cp in enumerate(items):
        arr[k] = PigoCascadeParams(cp.MinSize, cp.MaxSize, cp.ShiftFactor, cp.ScaleFactor) if isinstance(cp, CascadeParams) else PigoCascadeParams(*cp)
    return arr


def _angles_array(angles, n: int) -> Optional[np.ndarray]:
    """float64 array of one angle per entry, or None."""
    if angles is None:
        return None
    if len(angles) != n:
        raise ValueError("angles must have one entry per image")
    return np.ascontiguousarray(angles, dtype=np.float64)


def shard_plan(images, min_size: int, max_size: int, shift_factor: float, scale_factor: float, angles: Optional[Sequence[float]] = None,
               nshards: int = 0) -> List[int]:
    """The split the sharded mixed-size calls make (pigo_shard_plan; no device needed): the first entry of every shard, then
    len(images).  images: ImageParams or (pixels, rows, cols, dim) tuples (pixels are not read); nshards 0 = the count the
    calls use (option shard_split, else one per selected device)."""
    items = [(0, im.Rows, im.Cols, im.Dim) if isinstance(im, ImageParams) else (0, im[1], im[2], im[3]) for im in images]
    n = len(items)
    desc = image_descs(items)
    ang = _angles_array(angles, n)
    first = np.zeros(n + 1, dtype=np.int32)
    used = C.c_int()
    _check(lib().pigo_shard_plan(desc, n, ang.ctypes.data if ang is not None else None, min_size, max_size, shift_factor, scale_factor, nshards,
                                 first.ctypes.data, C.byref(used)))
    return first[:used.value + 1].tolist()


def _pixels(img: ImageParams) -> np.ndarray:
    p = np.ascontiguousarray(img.Pixels, dtype=np.uint8).reshape(-1)
    if p.size < (img.Rows - 1) * img.Dim + img.Cols and img.Rows > 0:
        raise ValueError("Pixels shorter than Rows*Dim")   # the reference would panic with index out of range
    return p


def _image_table(images):
    """(descriptor array, pixel flag, keep) of a mixed-size call's images: FRAMES_DEVICE when every image's Pixels is a device
    pointer (int), else MEM_HOST with host arrays, which `keep` holds alive for the call."""
    on_dev = len(images) > 0 and all(isinstance(im.Pixels, int) for im in images)
    keep = [None if on_dev else _pixels(im) for im in images]
    desc = image_descs([(im.Pixels if on_dev else p.ctypes.data, im.Rows, im.Cols, im.Dim) for im, p in zip(images, keep)])
    return desc, (FRAMES_DEVICE if on_dev else MEM_HOST), keep


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

    def RunCascadeImages(self, images: Sequence[ImageParams], cp: CascadeParams, angle: float = 0.0, cap_per_image: int = 1024):
        """Additive mixed-size entry point: RunCascade for every image of `images` (each with its own Rows, Cols, Dim) in one
        call, with cp's MinSize / MaxSize / ShiftFactor / ScaleFactor (cp.ImageParams is not used).  Pixels are host arrays,
        or for every image alike device pointers (int) holding Rows*Dim bytes.  Returns (dets[N, cap] DET_DTYPE, counts[N])."""
        self._need()
        n = len(images)
        desc, flags, keep = _image_table(images)
        return self._retry_cap(n, cap_per_image, lambda out, cap, cnt: lib().pigo_run_cascade_images(
            self._h, desc, n, cp.MinSize, cp.MaxSize, cp.ShiftFactor, cp.ScaleFactor, angle, out, cap, cnt, flags, None))

    def run_cascade_images_device(self, images, min_size: int, max_size: int, shift: float, scale: float, angle: float, out_ptr: int,
                                  cap_per_image: int, counts_ptr: int, stream: int = 0):
        """Fully device-resident, asynchronous mixed-size form: images = [(device pointer, rows, cols, dim)], out [N][cap] and
        counts [N] are device pointers; no host sync."""
        self._need()
        _check(lib().pigo_run_cascade_images(self._h, image_descs(images), len(images), min_size, max_size, shift, scale, angle, out_ptr,
                                             cap_per_image, counts_ptr, FRAMES_DEVICE | OUT_DEVICE, stream or None))

    def RunCascadeImagesAngles(self, images: Sequence[ImageParams], cp: CascadeParams, angles: Sequence[float], cap_per_image: int = 1024):
        """RunCascadeImages with image i scanned at angles[i] (one angle per image).  An angle sweep is one call: list an
        image once per angle; repeated host pixels are copied to the device once.  Returns (dets[N, cap] DET_DTYPE, counts[N])."""
        self._need()
        n = len(images)
        if len(angles) != n:
            raise ValueError("angles must have one entry per image")
        desc, flags, keep = _image_table(images)
        ang = np.ascontiguousarray(angles, dtype=np.float64)
        return self._retry_cap(n, cap_per_image, lambda out, cap, cnt: lib().pigo_run_cascade_images_angles(
            self._h, desc, n, ang.ctypes.data, cp.MinSize, cp.MaxSize, cp.ShiftFactor, cp.ScaleFactor, out, cap, cnt, flags, None))

    def run_cascade_images_angles_device(self, images, angles: Sequence[float], min_size: int, max_size: int, shift: float, scale: float,
                                         out_ptr: int, cap_per_image: int, counts_ptr: int, stream: int = 0):
        """Device-resident, asynchronous form of RunCascadeImagesAngles: images = [(device pointer, rows, cols, dim)], angles a
        host sequence with one entry per image, out [N][cap] and counts [N] device pointers; no host sync."""
        self._need()
        if len(angles) != len(images):
            raise ValueError("angles must have one entry per image")
        ang = np.ascontiguousarray(angles, dtype=np.float64)
        _check(lib().pigo_run_cascade_images_angles(self._h, image_descs(images), len(images), ang.ctypes.data, min_size, max_size, shift, scale,
                                                    out_ptr, cap_per_image, counts_ptr, FRAMES_DEVICE | OUT_DEVICE, stream or None))

    def RunCascadeImagesParams(self, cps: Sequence[CascadeParams], angles: Optional[Sequence[float]] = None, cap_per_image: int = 1024):
        """A list of RunCascade(cps[i], angles[i]) calls as one call (pigo_run_cascade_images_params): every CascadeParams carries
        its own ImageParams, MinSize, MaxSize, ShiftFactor and ScaleFactor; angles None = every image unrotated.  Pixels as
        RunCascadeImages.  Returns (dets[N, cap] DET_DTYPE, counts[N])."""
        self._need()
        n = len(cps)
        desc, flags, keep = _image_table([cp.ImageParams for cp in cps])
        prm = cascade_params_array(cps)
        ang = _angles_array(angles, n)
        return self._retry_cap(n, cap_per_image, lambda out, cap, cnt: lib().pigo_run_cascade_images_params(
            self._h, desc, n, prm, ang.ctypes.data if ang is not None else None, out, cap, cnt, flags, None))

    def run_cascade_images_params_device(self, images, params, angles: Optional[Sequence[float]], out_ptr: int, cap_per_image: int,
                                         counts_ptr: int, stream: int = 0):
        """Device-resident, asynchronous form of RunCascadeImagesParams: images = [(device pointer, rows, cols, dim)], params one
        (MinSize, MaxSize, ShiftFactor, ScaleFactor) or CascadeParams per image, angles a host sequence or None, out [N][cap] and
        counts [N] device pointers; no host sync."""
        self._need()
        if len(params) != len(images):
            raise ValueError("params must have one entry per image")
        ang = _angles_array(angles, len(images))
        _check(lib().pigo_run_cascade_images_params(self._h, image_descs(images), len(images), cascade_params_array(params),
                                                    ang.ctypes.data if ang is not None else None, out_ptr, cap_per_image, counts_ptr,
                                                    FRAMES_DEVICE | OUT_DEVICE, stream or None))

    def RunCascadeImagesSweep(self, images: Sequence[ImageParams], cp: CascadeParams, angles: Sequence[float], iou: float, det_cap: int = 0,
                              cap_per_image: int = 256):
        """Every image scanned at every angle of `angles`, merged per image (pigo_run_cascade_images_sweep): image i's clusters
        of the concatenation of its RunCascade lists over the angles, with the index into `angles` of each cluster's largest-Q
        member.  Pixels as RunCascadeImages.  PIGO_E_CAP is retried (a larger det_cap for raw lists, else the reported counts).
        Returns (clusters[N, cap] DET_DTYPE, angle_index[N, cap] int32, counts[N])."""
        self._need()
        n = len(images)
        desc, flags, keep = _image_table(images)
        ang = np.ascontiguousarray(angles, dtype=np.float64)
        while True:
            out = np.zeros((n, max(cap_per_image, 1)), dtype=DET_DTYPE)
            tag = np.full((n, max(cap_per_image, 1)), -1, dtype=np.int32)
            cnt = np.zeros(max(n, 1), dtype=np.int32)
            rc = lib().pigo_run_cascade_images_sweep(self._h, desc, n, ang.ctypes.data, len(ang), cp.MinSize, cp.MaxSize, cp.ShiftFactor,
                                                     cp.ScaleFactor, iou, det_cap, out.ctypes.data, tag.ctypes.data, cap_per_image,
                                                     cnt.ctypes.data, flags, None)
            if rc == PIGO_E_CAP:
                if "raw detections" in lib().pigo_last_error().decode():
                    det_cap = 4 * (det_cap or 2048)
                else:
                    cap_per_image = int(cnt.max())
                continue
            _check(rc)
            return out, tag, cnt[:n]

    def run_cascade_images_sweep_device(self, images, angles: Sequence[float], min_size: int, max_size: int, shift: float, scale: float,
                                        iou: float, det_cap: int, out_ptr: int, angle_index_ptr: int, cap_per_image: int, counts_ptr: int,
                                        stream: int = 0):
        """Device-resident, asynchronous form of RunCascadeImagesSweep: images = [(device pointer, rows, cols, dim)], angles a host
        sequence, out [N][cap], angle_index [N][cap] (0 = not wanted) and counts [N] device pointers; no host sync."""
        self._need()
        ang = np.ascontiguousarray(angles, dtype=np.float64)
        _check(lib().pigo_run_cascade_images_sweep(self._h, image_descs(images), len(images), ang.ctypes.data, len(ang), min_size, max_size, shift,
                                                   scale, iou, det_cap, out_ptr, angle_index_ptr or None, cap_per_image, counts_ptr,
                                                   FRAMES_DEVICE | OUT_DEVICE, stream or None))

    def run_cascade_images_sharded(self, images: Sequence[ImageParams], cp: CascadeParams, angles: Optional[Sequence[float]] = None,
                                   cap_per_image: int = 1024):
        """RunCascadeImagesAngles over the devices of init_devices (pigo_run_cascade_images_sharded): host images, cut into
        contiguous shards of about equal modelled cost; angles None = every image at 0.  The result equals the single-device
        call byte for byte.  Returns (dets[N, cap] DET_DTYPE, counts[N])."""
        self._need()
        n = len(images)
        keep = [_pixels(im) for im in images]   # host pixels stay alive for the call
        desc = image_descs([(p.ctypes.data, im.Rows, im.Cols, im.Dim) for im, p in zip(images, keep)])
        ang = _angles_array(angles, n)
        return self._retry_cap(n, cap_per_image, lambda out, cap, cnt: lib().pigo_run_cascade_images_sharded(
            self._h, desc, n, ang.ctypes.data if ang is not None else None, cp.MinSize, cp.MaxSize, cp.ShiftFactor, cp.ScaleFactor, out, cap, cnt))

    def run_cascade_decoded_sharded(self, sources: Sequence["DecodedImage"], cp: CascadeParams, angles: Optional[Sequence[float]] = None,
                                    cap_per_image: int = 1024):
        """gray_images of host DecodedImage sources, then RunCascadeImagesAngles, over the devices of init_devices
        (pigo_run_cascade_decoded_sharded): each device converts its own shard.  Returns (dets[N, cap] DET_DTYPE, counts[N])."""
        self._need()
        n = len(sources)
        desc = decoded_descs(sources)
        ang = _angles_array(angles, n)
        return self._retry_cap(n, cap_per_image, lambda out, cap, cnt: lib().pigo_run_cascade_decoded_sharded(
            self._h, desc, n, ang.ctypes.data if ang is not None else None, cp.MinSize, cp.MaxSize, cp.ShiftFactor, cp.ScaleFactor, out, cap, cnt))

    def BlurDecoded(self, sources: Sequence["DecodedImage"], cps: Sequence[CascadeParams], angles: Optional[Sequence[float]], iou: float,
                    params: "BlurParams", det_cap: int = 0, face_cap: Optional[int] = None, device_sources: bool = False, stream=None):
        """Blurs the faces of decoded images in place, in one call (pigo_blur_decoded): gray_images of `sources`, RunCascade of
        image i with cps[i]'s MinSize / MaxSize / ShiftFactor / ScaleFactor at angles[i] (None = unrotated), ClusterDetections(iou),
        then blur_faces on every cluster.  Returns the face lists, list i as ClusterDetections returns it for image i.  An entry
        past det_cap raw detections (0 = 2048) leaves the planes alone and is retried with a larger det_cap; face_cap None
        returns every cluster, a smaller face_cap that an image exceeds raises PIGO_E_CAP after the blur."""
        self._need()
        n = len(sources)
        desc = decoded_descs(sources)
        prm = cascade_params_array(cps)
        if len(cps) != n:
            raise ValueError("cps must have one entry per source")
        ang = _angles_array(angles, n)
        flags = FRAMES_DEVICE if device_sources else MEM_HOST
        sptr = (stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream)) if stream is not None else None
        while True:
            cap = face_cap if face_cap is not None else (det_cap or 2048)
            faces = np.zeros((n, max(cap, 1)), dtype=DET_DTYPE)
            cnt = np.zeros(max(n, 1), dtype=np.int32)
            rc = lib().pigo_blur_decoded(self._h, desc, n, prm, ang.ctypes.data if ang is not None else None, iou, det_cap, C.byref(params),
                                         faces.ctypes.data, cap, cnt.ctypes.data, flags, sptr)
            if rc == PIGO_E_CAP and "raw detections" in lib().pigo_last_error().decode():
                det_cap = 4 * (det_cap or 2048)
                continue
            _check(rc)
            return [_array_to_dets(faces[i, :cnt[i]]) for i in range(n)]

    @staticmethod
    def _retry_cap(n: int, cap: int, fn):
        """Calls fn(out, cap, counts) until the output capacity is enough (PIGO_E_CAP retries with the reported count)."""
        while True:
            out = np.zeros((n, max(cap, 1)), dtype=DET_DTYPE)
            cnt = np.zeros(max(n, 1), dtype=np.int32)
            rc = fn(out.ctypes.data, cap, cnt.ctypes.data)
            if rc == PIGO_E_CAP:
                cap = int(cnt.max())
                continue
            _check(rc)
            return out, cnt[:n]

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

    def run_detector_images(self, seeds: Sequence[Puploc], seed_image: Sequence[int], images: Sequence[ImageParams], angle: float = 0.0,
                            flipv: Optional[Sequence[bool]] = None, randoms: Optional[np.ndarray] = None, rng_seed: int = 0) -> List[Puploc]:
        """Batch over images of different sizes: seed i refines on images[seed_image[i]].  Pixels are host arrays, or for
        every image alike device pointers (int) holding Rows*Dim bytes, as in Pigo.RunCascadeImages."""
        if self._h is None:
            raise PigoError(PIGO_E_INVALID, "cascade not unpacked")
        n = len(seeds)
        if n == 0:
            return []
        s = np.zeros(n, dtype=POINT_DTYPE)
        for k, p in enumerate(seeds):
            s[k] = (p.Row, p.Col, p.Scale, p.Perturbs)
        si = np.ascontiguousarray(np.asarray(seed_image, dtype=np.int32))
        out = np.zeros(n, dtype=POINT_DTYPE)
        rnd = np.ascontiguousarray(randoms, dtype=np.float32) if randoms is not None else None
        fl = np.ascontiguousarray(np.asarray(flipv, dtype=np.uint8)) if flipv is not None else None
        desc, flags, keep = _image_table(images)
        _check(lib().pigo_puploc_run_images(self._h, s.ctypes.data, n, si.ctypes.data, rnd.ctypes.data if rnd is not None else None, rng_seed,
                                            desc, len(images), angle, fl.ctypes.data if fl is not None else None, out.ctypes.data,
                                            flags, None))
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


class PigoDecoded(C.Structure):
    """pigo_decoded (include/pigo_b200.h): one decoded image of a pigo_gray_images call."""
    _fields_ = [("format", C.c_int32), ("subsample", C.c_int32), ("min_x", C.c_int32), ("min_y", C.c_int32), ("width", C.c_int32),
                ("height", C.c_int32), ("plane", C.c_void_p * 3), ("stride", C.c_int32 * 2)]


def _row_bytes(a, default: int) -> int:
    """Row pitch in bytes of a uint8 plane given as a numpy array or torch tensor of two or more dimensions, else `default`."""
    if isinstance(a, np.ndarray) and a.ndim >= 2:
        return int(a.strides[0])
    if hasattr(a, "stride") and hasattr(a, "dim") and a.dim() >= 2:
        return int(a.stride(0))
    return int(default)


def _plane_ptr(a) -> Optional[int]:
    """Address of a plane: a device pointer (int), a torch tensor, or a host numpy uint8 array."""
    if a is None:
        return None
    if isinstance(a, int):
        return a
    if hasattr(a, "data_ptr"):
        return int(a.data_ptr())
    if not isinstance(a, np.ndarray) or a.dtype != np.uint8:
        raise TypeError("a plane is a uint8 numpy array, a torch tensor or a device pointer (int)")
    return int(a.ctypes.data)


@dataclass
class DecodedImage:
    """One decoded Go image as pigo_gray_images takes it (pigo_decoded): `planes` start at the rectangle's origin and are
    host numpy uint8 arrays, or (device_sources) device pointers / torch CUDA tensors.  Build it with one constructor per
    Go image type; strides default to the arrays' row pitch."""
    format: int
    width: int
    height: int
    planes: tuple
    strides: tuple = (0, 0)
    subsample: int = 0
    min_x: int = 0
    min_y: int = 0

    @classmethod
    def ycbcr(cls, y, cb, cr, subsample: int, width: int, height: int, min_x: int = 0, min_y: int = 0, y_stride: Optional[int] = None,
              c_stride: Optional[int] = None) -> "DecodedImage":
        """*image.YCbCr: Y[YOffset(Rect.Min):], Cb / Cr[COffset(Rect.Min):], SubsampleRatio (0..5), Rect.Min (>= 0)."""
        return cls(DECODED_YCBCR, width, height, (y, cb, cr), (y_stride if y_stride is not None else _row_bytes(y, width),
                                                               c_stride if c_stride is not None else _row_bytes(cb, 0)), subsample, min_x, min_y)

    @classmethod
    def nrgba(cls, pix, width: int, height: int, stride: Optional[int] = None) -> "DecodedImage":
        """*image.NRGBA: Pix[PixOffset(Rect.Min):] and Stride."""
        return cls(DECODED_NRGBA, width, height, (pix,), (stride if stride is not None else _row_bytes(pix, 4 * width), 0))

    @classmethod
    def rgba(cls, pix, width: int, height: int, stride: Optional[int] = None) -> "DecodedImage":
        """*image.RGBA (alpha-premultiplied): Pix[PixOffset(Rect.Min):] and Stride."""
        return cls(DECODED_RGBA, width, height, (pix,), (stride if stride is not None else _row_bytes(pix, 4 * width), 0))

    @classmethod
    def gray(cls, pix, width: int, height: int, stride: Optional[int] = None) -> "DecodedImage":
        """*image.Gray: Pix[PixOffset(Rect.Min):] and Stride."""
        return cls(DECODED_GRAY, width, height, (pix,), (stride if stride is not None else _row_bytes(pix, width), 0))

    @classmethod
    def gray16(cls, pix, width: int, height: int, stride: Optional[int] = None) -> "DecodedImage":
        """*image.Gray16: Pix[PixOffset(Rect.Min):] (2 bytes per pixel, big-endian) and Stride."""
        return cls(DECODED_GRAY16, width, height, (pix,), (stride if stride is not None else _row_bytes(pix, 2 * width), 0))

    @classmethod
    def rgba64(cls, pix, width: int, height: int, stride: Optional[int] = None) -> "DecodedImage":
        """*image.RGBA64 (alpha-premultiplied): Pix[PixOffset(Rect.Min):] (R, G, B, A big-endian uint16) and Stride."""
        return cls(DECODED_RGBA64, width, height, (pix,), (stride if stride is not None else _row_bytes(pix, 8 * width), 0))

    @classmethod
    def nrgba64(cls, pix, width: int, height: int, stride: Optional[int] = None) -> "DecodedImage":
        """*image.NRGBA64: Pix[PixOffset(Rect.Min):] (R, G, B, A big-endian uint16) and Stride."""
        return cls(DECODED_NRGBA64, width, height, (pix,), (stride if stride is not None else _row_bytes(pix, 8 * width), 0))

    @classmethod
    def cmyk(cls, pix, width: int, height: int, stride: Optional[int] = None) -> "DecodedImage":
        """*image.CMYK: Pix[PixOffset(Rect.Min):] (C, M, Y, K bytes) and Stride."""
        return cls(DECODED_CMYK, width, height, (pix,), (stride if stride is not None else _row_bytes(pix, 4 * width), 0))

    @classmethod
    def paletted(cls, pix, palette, width: int, height: int, stride: Optional[int] = None) -> "DecodedImage":
        """*image.Paletted: Pix[PixOffset(Rect.Min):] (palette indices) and Stride; `palette` is [k][4] uint8 NRGBA entries,
        entry i = color.NRGBAModel.Convert(Palette[i]), k in 1..256 (host array, or a CUDA tensor with device_sources)."""
        if isinstance(palette, np.ndarray):
            palette = np.ascontiguousarray(palette, dtype=np.uint8).reshape(-1, 4)
        return cls(DECODED_PALETTED, width, height, (pix, palette), (stride if stride is not None else _row_bytes(pix, width), len(palette)))

    def desc(self) -> PigoDecoded:
        d = PigoDecoded()
        d.format, d.subsample, d.min_x, d.min_y, d.width, d.height = self.format, self.subsample, self.min_x, self.min_y, self.width, self.height
        for k in range(3):
            d.plane[k] = _plane_ptr(self.planes[k]) if k < len(self.planes) else None
        d.stride[0], d.stride[1] = int(self.strides[0]), int(self.strides[1])
        return d


class DeviceImage(tuple):
    """A device image of the gray arena: the (pixels, rows, cols, dim) tuple run_cascade_images[_angles]_device takes, with the
    ImageParams field names pipeline.detect_images[_angles]_device reads (Pixels is a device pointer)."""
    def __new__(cls, pixels: int, rows: int, cols: int, dim: int):
        return super().__new__(cls, (pixels, rows, cols, dim))

    Pixels = property(lambda self: self[0])
    Rows = property(lambda self: self[1])
    Cols = property(lambda self: self[2])
    Dim = property(lambda self: self[3])


def decoded_descs(sources: Sequence[DecodedImage]) -> C.Array:
    arr = (PigoDecoded * max(len(sources), 1))()
    for k, s in enumerate(sources):
        arr[k] = s.desc()
    return arr


def gray_images_bytes(sources: Sequence[DecodedImage]) -> int:
    """Device bytes pigo_gray_images needs for `sources` (no device needed): sum of round256(width*height) over distinct sources."""
    need = C.c_size_t(0)
    imgs = (PigoImage * max(len(sources), 1))()
    rc = lib().pigo_gray_images(decoded_descs(sources), len(sources), None, C.byref(need), imgs, MEM_HOST, None)
    if rc not in (PIGO_OK, PIGO_E_CAP):
        _check(rc)
    return int(need.value)


def gray_images(sources: Sequence[DecodedImage], stream=None, device_sources: bool = False):
    """RgbToGrayscale(ImgToNRGBA(img)) of every source in one call (pigo_gray_images).  Returns (arena, images): the arena is a
    torch uint8 CUDA tensor and images[i] a DeviceImage {slot, height, width, width} that Pigo.run_cascade_images_angles_device
    and pipeline.detect_images_angles_device take as it is.  Repeated sources share a slot.  `stream` (a torch.cuda.Stream or
    a cudaStream_t as int) orders the call on the caller's stream; without it the arena is complete on return.  Host planes
    are read only during the call; with device_sources every plane is a device pointer or CUDA tensor."""
    import torch
    n = len(sources)
    desc = decoded_descs(sources)
    imgs = (PigoImage * max(n, 1))()
    flags = FRAMES_DEVICE if device_sources else MEM_HOST
    sptr = (stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream)) if stream is not None else None
    need = C.c_size_t(0)
    rc = lib().pigo_gray_images(desc, n, None, C.byref(need), imgs, flags, sptr)
    if rc not in (PIGO_OK, PIGO_E_CAP):
        _check(rc)
    if hasattr(stream, "cuda_stream"):
        with torch.cuda.stream(stream):
            arena = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    else:
        arena = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    size = C.c_size_t(arena.numel())
    _check(lib().pigo_gray_images(desc, n, arena.data_ptr() if arena.numel() else None, C.byref(size), imgs, flags, sptr))
    return arena, [DeviceImage(imgs[k].pixels, imgs[k].rows, imgs[k].cols, imgs[k].dim) for k in range(n)]


class BlurParams(C.Structure):
    """pigo_blur_params (include/pigo_b200.h): faces with Q >= min_q are blurred over a disc of radius int(Scale*disc_ratio)
    with a box of radius min(1023, max(radius, int(Scale*radius_ratio))).  examples/facedet/faceblur.py's values are
    BlurParams(5.0, 0.5, 0.0, 15)."""
    _fields_ = [("min_q", C.c_double), ("disc_ratio", C.c_double), ("radius_ratio", C.c_double), ("radius", C.c_int32)]


def blur_faces(sources: Sequence[DecodedImage], faces, counts, params: BlurParams, stream=None, device_sources: bool = False,
               device_faces: bool = False):
    """Blurs the faces of every source in place (pigo_blur_faces).  faces is [N][face_cap] DET_DTYPE and counts [N] (what
    cluster_batch_array and the pipeline calls return), or with device_faces device pointers / CUDA tensors of that layout
    (faces then a tensor of shape [N, face_cap, 4] int32, or (pointer, face_cap)).  Planes are host numpy arrays, written
    back before return, or (device_sources) device pointers / CUDA tensors; `stream` (a torch.cuda.Stream or a cudaStream_t as
    int) orders the call on the caller's stream, and with device planes the call then returns without synchronising."""
    n = len(sources)
    desc = decoded_descs(sources)
    if device_faces:
        fptr, face_cap = (int(faces.data_ptr()), int(faces.shape[1])) if hasattr(faces, "data_ptr") else (int(faces[0]), int(faces[1]))
        cptr = int(counts.data_ptr()) if hasattr(counts, "data_ptr") else int(counts)
    else:
        f = np.ascontiguousarray(faces, dtype=DET_DTYPE).reshape(n, -1) if n else np.zeros((0, 0), dtype=DET_DTYPE)
        face_cap = f.shape[1] if n else 0
        c = np.ascontiguousarray(counts, dtype=np.int32).reshape(-1)
        if len(c) != n:
            raise ValueError("counts must have one entry per source")
        fptr, cptr = (f.ctypes.data if f.size else None), (c.ctypes.data if n else None)
    flags = (FRAMES_DEVICE if device_sources else MEM_HOST) | (FACES_DEVICE if device_faces else 0)
    sptr = (stream.cuda_stream if hasattr(stream, "cuda_stream") else int(stream)) if stream is not None else None
    _check(lib().pigo_blur_faces(desc, n, fptr, face_cap, cptr, C.byref(params), flags, sptr))


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
