"""CPU-side checks of the mixed-size pipeline (pigo_detect_images) and mixed-size RunDetector (pigo_puploc_run_images):
every invalid argument is rejected with PIGO_E_INVALID and a message that names it before any device work, and the Go shim
binds the pipeline call."""
import ctypes as C
import glob
import os
import re

import numpy as np
import pytest

import pigo_b200
from test_abi import _calls

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PIX = np.zeros(64 * 64, dtype=np.uint8)
FAKE = C.c_void_p(16)   # a non-NULL handle that validation never dereferences (it fails on an earlier argument)


def _descs(*geoms, pixels=PIX.ctypes.data):
    return pigo_b200.image_descs([(pixels, r, c, d) for r, c, d in geoms])


def _detect(images, nimages, face=None, puploc=None, flp="default", ncalls=2, face_cap=4, prm_kw=None, faces=True, n_faces=True,
            points=True, params=True):
    """pigo_detect_images with NULL cascades unless given: the handles are validated last."""
    L = pigo_b200.lib()
    kw = dict(min_size=20, max_size=1000, shift_factor=0.2, scale_factor=1.1, angle=0.0, iou_threshold=0.1, min_face_scale=50,
              eye_perturbs=50, flp_perturbs=63, det_cap=0)
    kw.update(prm_kw or {})
    prm = pigo_b200.PipelineParams(**kw)
    hs = (C.c_void_p * 2)(None, None) if flp == "default" else flp
    fl = np.zeros(2, dtype=np.uint8)
    out_f = np.zeros(8 * 64, dtype=pigo_b200.DET_DTYPE)
    out_n = np.zeros(8, dtype=np.int32)
    out_p = np.zeros(8 * 64 * 32, dtype=pigo_b200.POINT_DTYPE)
    rc = L.pigo_detect_images(face, puploc, hs, fl.ctypes.data, ncalls, images, nimages, C.byref(prm) if params else None, None, 0,
                              out_f.ctypes.data if faces else None, face_cap, out_n.ctypes.data if n_faces else None,
                              out_p.ctypes.data if points else None, pigo_b200.MEM_HOST, None)
    return rc, L.pigo_last_error().decode()


@pytest.mark.parametrize("case,images,nimages,kw,msg", [
    ("too many images", _descs((8, 8, 8)), 65536, {}, "nimages"),
    ("negative count", _descs((8, 8, 8)), -1, {}, "nimages"),
    ("null images", None, 2, {}, "null images"),
    ("null params", _descs((8, 8, 8)), 1, {"params": False}, "null params"),
    ("null faces", _descs((8, 8, 8)), 1, {"faces": False}, "null faces"),
    ("null n_faces", _descs((8, 8, 8)), 1, {"n_faces": False}, "null n_faces"),
    ("null points", _descs((8, 8, 8)), 1, {"points": False}, "null points"),
    ("ncalls > 30", _descs((8, 8, 8)), 1, {"ncalls": 31}, "ncalls"),
    ("negative ncalls", _descs((8, 8, 8)), 1, {"ncalls": -1}, "ncalls"),
    ("null flp", _descs((8, 8, 8)), 1, {"flp": None}, "null flp"),
    ("face_cap 0", _descs((8, 8, 8)), 1, {"face_cap": 0}, "face_cap"),
    ("face_cap 4097", _descs((8, 8, 8)), 1, {"face_cap": 4097}, "face_cap"),
    ("eye perturbs", _descs((8, 8, 8)), 1, {"prm_kw": {"eye_perturbs": 64}}, "Perturbs"),
    ("flp perturbs", _descs((8, 8, 8)), 1, {"prm_kw": {"flp_perturbs": -1}}, "Perturbs"),
    ("pupil work > 2^31-1", _descs((8, 8, 8)), 65535, {"face_cap": 4096, "ncalls": 30}, "exceeds 2^31-1"),
    ("zero rows", _descs((8, 8, 8), (0, 8, 8)), 2, {}, "image 1: bad geometry"),
    ("zero cols", _descs((8, 0, 8)), 1, {}, "image 0: bad geometry"),
    ("dim < cols", _descs((8, 9, 8)), 1, {}, "image 0: bad geometry"),
    ("rows*dim >= 2^31", _descs((65536, 32768, 32768)), 1, {}, "image 0: larger than 2^31"),
    ("null pixels", _descs((8, 8, 8), pixels=None), 1, {}, "image 0: null pixels"),
    ("null pupil cascade", _descs((8, 8, 8)), 1, {"face": FAKE}, "null pupil cascade"),
    ("null landmark cascade", _descs((8, 8, 8)), 1, {"face": FAKE, "puploc": FAKE, "flp": (C.c_void_p * 2)(FAKE, None)}, "null landmark cascade 1"),
])
def test_detect_images_rejects_invalid_arguments_before_the_device(case, images, nimages, kw, msg):
    rc, err = _detect(images, nimages, **kw)
    assert rc == pigo_b200.PIGO_E_INVALID, case
    assert msg in err, (case, err)


def test_detect_images_valid_arguments_reach_the_cascade_check():
    """Control for the cases above: valid images (odd pitches, one pixel, no windows) fail only on the NULL cascade."""
    rc, err = _detect(_descs((64, 64, 64), (1, 1, 1), (10, 10, 16), (40, 30, 31)), 4)
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err


def _run_images(seeds, nseeds, seed_image, images, nimages, p=None, out=True):
    L = pigo_b200.lib()
    o = np.zeros(max(nseeds, 1), dtype=pigo_b200.POINT_DTYPE)
    si = None if seed_image is None else np.ascontiguousarray(seed_image, dtype=np.int32)
    rc = L.pigo_puploc_run_images(p, seeds.ctypes.data if seeds is not None else None, nseeds, si.ctypes.data if si is not None else None,
                                  None, 0, images, nimages, 0.0, None, o.ctypes.data if out else None, pigo_b200.MEM_HOST, None)
    return rc, L.pigo_last_error().decode()


def _seeds(*perturbs):
    s = np.zeros(len(perturbs), dtype=pigo_b200.POINT_DTYPE)
    for k, pt in enumerate(perturbs):
        s[k] = (5, 5, 10.0, pt)
    return s


@pytest.mark.parametrize("case,args,msg", [
    ("negative nseeds", (_seeds(1), -1, None, _descs((8, 8, 8)), 1), "negative nseeds"),
    ("null seeds", (None, 1, None, _descs((8, 8, 8)), 1), "null seeds"),
    ("no images", (_seeds(1), 1, None, _descs((8, 8, 8)), 0), "nimages"),
    ("too many images", (_seeds(1), 1, [0], _descs((8, 8, 8)), 65536), "nimages"),
    ("null images", (_seeds(1), 1, None, None, 1), "null images"),
    ("seed_image missing", (_seeds(1), 1, None, _descs((8, 8, 8), (9, 9, 9)), 2), "seed_image is required"),
    ("zero rows", (_seeds(1), 1, [0], _descs((8, 8, 8), (0, 9, 9)), 2), "image 1: bad geometry"),
    ("dim < cols", (_seeds(1), 1, None, _descs((8, 9, 8)), 1), "image 0: bad geometry"),
    ("rows*dim >= 2^31", (_seeds(1), 1, None, _descs((65536, 32768, 32768)), 1), "image 0: larger than 2^31"),
    ("null pixels", (_seeds(1), 1, None, _descs((8, 8, 8), pixels=None), 1), "image 0: null pixels"),
    ("perturbs > 63", (_seeds(3, 64), 2, None, _descs((8, 8, 8)), 1), "seed 1: Perturbs=64"),
    ("negative perturbs", (_seeds(-1), 1, None, _descs((8, 8, 8)), 1), "seed 0: Perturbs=-1"),
    ("image index past the end", (_seeds(1, 1), 2, [1, 2], _descs((8, 8, 8), (9, 9, 9)), 2), "seed 1: image index out of range"),
    ("negative image index", (_seeds(1), 1, [-1], _descs((8, 8, 8), (9, 9, 9)), 2), "seed 0: image index out of range"),
])
def test_puploc_run_images_rejects_invalid_arguments_before_the_device(case, args, msg):
    rc, err = _run_images(*args)
    assert rc == pigo_b200.PIGO_E_INVALID, case
    assert msg in err, (case, err)


def test_puploc_run_images_null_out_and_valid_arguments():
    rc, err = _run_images(_seeds(1), 1, None, _descs((8, 8, 8)), 1, out=False)
    assert rc == pigo_b200.PIGO_E_INVALID and "null out" in err
    rc, err = _run_images(_seeds(0, 63, 7), 3, [0, 2, 1], _descs((8, 8, 8), (1, 1, 1), (30, 40, 41)), 3)
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err


def test_go_shim_binds_detect_images():
    header = open(os.path.join(ROOT, "include", "pigo_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    protos = dict(_calls(header, ""))
    assert protos["pigo_detect_images"] == 16 and protos["pigo_puploc_run_images"] == 13
    go = "\n".join(open(f).read() for f in sorted(glob.glob(os.path.join(ROOT, "go", "pigo", "*.go"))))
    go = re.sub(r"//[^\n]*", "", go)
    calls = [n for name, n in _calls(go, "C.") if name == "pigo_detect_images"]
    assert calls and all(n == protos["pigo_detect_images"] for n in calls)
    assert re.search(r"^func \(pg \*Pigo\) DetectImages\(plc \*PuplocCascade, calls \[\]LandmarkCall, images \[\]ImageParams, "
                     r"cp CascadeParams, pp PipelineParams\) \[\]\[\]FaceResult \{", go, flags=re.M)
    body = go[go.index("func (pg *Pigo) DetectImages("):]
    body = body[:body.index("\n}\n")]
    assert "pp.Sharded" in body and "panic(" in body and "C.PIGO_E_CAP" in body
    assert "C.pigo_alloc_pinned" in body and "C.malloc" in body
