"""CPU-side checks of the angle sweep (pigo_run_cascade_images_sweep, pigo_detect_images_sweep): every invalid argument is
rejected with PIGO_E_INVALID before any device work, valid ones reach the cascade check, the Go shim binds both calls, and
the oracle restatement of the merge (tests/sweep_oracle.py) recovers the tilt of the rotated sample within one slot."""
import ctypes as C
import glob
import os
import re

import numpy as np
import pytest

import oracle_lib as O
import pigo_b200
import sweep_oracle as S
from test_abi import _calls

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PIX = np.zeros(64 * 64, dtype=np.uint8)
ANG = np.array([0.0, 0.25, float("nan"), 1.3], dtype=np.float64)
FAKE = C.c_void_p(16)   # a non-NULL handle that validation never dereferences (it fails on an earlier argument)


def _descs(*geoms, pixels=PIX.ctypes.data):
    return pigo_b200.image_descs([(pixels, r, c, d) for r, c, d in geoms])


def _scan(images, nimages, angles=True, nangles=4, cap=4, with_n_out=True, det_cap=0):
    """pigo_run_cascade_images_sweep with a NULL cascade: the cascade is validated last."""
    L = pigo_b200.lib()
    out = np.zeros((4, max(cap, 1)), dtype=pigo_b200.DET_DTYPE)
    tag = np.zeros((4, max(cap, 1)), dtype=np.int32)
    cnt = np.zeros(4, dtype=np.int32)
    rc = L.pigo_run_cascade_images_sweep(None, images, nimages, ANG.ctypes.data if angles else None, nangles, 20, 1000, 0.2, 1.1, 0.1, det_cap,
                                         out.ctypes.data, tag.ctypes.data, cap, cnt.ctypes.data if with_n_out else None, pigo_b200.MEM_HOST, None)
    return rc, L.pigo_last_error().decode()


@pytest.mark.parametrize("case,images,nimages,kw,msg", [
    ("null angles", _descs((8, 8, 8)), 1, {"angles": False}, "null angles"),
    ("no angles", _descs((8, 8, 8)), 1, {"nangles": 0}, "nangles"),
    ("negative nangles", _descs((8, 8, 8)), 1, {"nangles": -1}, "nangles"),
    ("entries > 65535", _descs((8, 8, 8)), 16384, {"nangles": 4}, "exceeds 65535"),
    ("negative det_cap", _descs((8, 8, 8)), 1, {"det_cap": -1}, "det_cap"),
    ("merged > 2^31-1", _descs((8, 8, 8)), 16383, {"det_cap": 1 << 16}, "exceeds 2^31-1"),
    ("null images", None, 2, {}, "null images"),
    ("negative count", _descs((8, 8, 8)), -1, {}, "nimages"),
    ("negative rows", _descs((8, 8, 8), (-1, 8, 8)), 2, {}, "image 1: bad geometry"),
    ("dim < cols", _descs((8, 9, 8)), 1, {}, "image 0: bad geometry"),
    ("rows*dim >= 2^31", _descs((65536, 32768, 32768)), 1, {}, "image 0: larger than 2^31"),
    ("negative capacity", _descs((8, 8, 8)), 1, {"cap": -1}, "negative capacity"),
    ("null n_out", _descs((8, 8, 8)), 1, {"with_n_out": False}, "null n_out"),
    ("null pixels", _descs((8, 8, 8), pixels=None), 1, {}, "image 0: null pixels"),
])
def test_run_cascade_images_sweep_rejects_invalid_arguments_before_the_device(case, images, nimages, kw, msg):
    rc, err = _scan(images, nimages, **kw)
    assert rc == pigo_b200.PIGO_E_INVALID, case
    assert msg in err, (case, err)


def test_run_cascade_images_sweep_valid_arguments_reach_the_cascade_check():
    rc, err = _scan(_descs((64, 64, 64), (64, 64, 64), (1, 1, 1), (0, 0, 0)), 4)
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err
    rc, err = _scan(_descs((8, 8, 8)), 0, nangles=1)
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err


def _detect(images, nimages, angles=True, nangles=4, face=None, puploc=None, flp="default", ncalls=2, face_cap=4, prm_kw=None, faces=True,
            n_faces=True, points=True, params=True):
    """pigo_detect_images_sweep with NULL cascades unless given: the handles are validated last."""
    L = pigo_b200.lib()
    kw = dict(min_size=20, max_size=1000, shift_factor=0.2, scale_factor=1.1, angle=0.0, iou_threshold=0.1, min_face_scale=50,
              eye_perturbs=50, flp_perturbs=63, det_cap=0)
    kw.update(prm_kw or {})
    prm = pigo_b200.PipelineParams(**kw)
    hs = (C.c_void_p * 2)(None, None) if flp == "default" else flp
    fl = np.zeros(2, dtype=np.uint8)
    out_f = np.zeros(8 * 64, dtype=pigo_b200.DET_DTYPE)
    out_a = np.zeros(8 * 64, dtype=np.int32)
    out_n = np.zeros(8, dtype=np.int32)
    out_p = np.zeros(8 * 64 * 32, dtype=pigo_b200.POINT_DTYPE)
    rc = L.pigo_detect_images_sweep(face, puploc, hs, fl.ctypes.data, ncalls, images, nimages, ANG.ctypes.data if angles else None, nangles,
                                    C.byref(prm) if params else None, None, 0, out_f.ctypes.data if faces else None, out_a.ctypes.data, face_cap,
                                    out_n.ctypes.data if n_faces else None, out_p.ctypes.data if points else None, pigo_b200.MEM_HOST, None)
    return rc, L.pigo_last_error().decode()


@pytest.mark.parametrize("case,images,nimages,kw,msg", [
    ("null angles", _descs((8, 8, 8)), 1, {"angles": False}, "null angles"),
    ("no angles", _descs((8, 8, 8)), 1, {"nangles": 0}, "nangles"),
    ("entries > 65535", _descs((8, 8, 8)), 32768, {"nangles": 2}, "exceeds 65535"),
    ("merged > 2^31-1", _descs((8, 8, 8)), 16000, {"prm_kw": {"det_cap": 1 << 16}}, "exceeds 2^31-1"),
    ("too many images", _descs((8, 8, 8)), 65536, {"nangles": 1}, "nimages"),
    ("negative count", _descs((8, 8, 8)), -1, {}, "nimages"),
    ("null images", None, 2, {}, "null images"),
    ("null params", _descs((8, 8, 8)), 1, {"params": False}, "null params"),
    ("null faces", _descs((8, 8, 8)), 1, {"faces": False}, "null faces"),
    ("null n_faces", _descs((8, 8, 8)), 1, {"n_faces": False}, "null n_faces"),
    ("null points", _descs((8, 8, 8)), 1, {"points": False}, "null points"),
    ("ncalls > 30", _descs((8, 8, 8)), 1, {"ncalls": 31}, "ncalls"),
    ("null flp", _descs((8, 8, 8)), 1, {"flp": None}, "null flp"),
    ("face_cap 0", _descs((8, 8, 8)), 1, {"face_cap": 0}, "face_cap"),
    ("eye perturbs", _descs((8, 8, 8)), 1, {"prm_kw": {"eye_perturbs": 64}}, "Perturbs"),
    ("pupil work > 2^31-1", _descs((8, 8, 8)), 65535, {"nangles": 1, "face_cap": 4096, "ncalls": 30}, "exceeds 2^31-1 pupil"),
    ("zero rows", _descs((8, 8, 8), (0, 8, 8)), 2, {}, "image 1: bad geometry"),
    ("null pixels", _descs((8, 8, 8), pixels=None), 1, {}, "image 0: null pixels"),
    ("null pupil cascade", _descs((8, 8, 8)), 1, {"face": FAKE}, "null pupil cascade"),
    ("null landmark cascade", _descs((8, 8, 8)), 1, {"face": FAKE, "puploc": FAKE, "flp": (C.c_void_p * 2)(FAKE, None)}, "null landmark cascade 1"),
])
def test_detect_images_sweep_rejects_invalid_arguments_before_the_device(case, images, nimages, kw, msg):
    rc, err = _detect(images, nimages, **kw)
    assert rc == pigo_b200.PIGO_E_INVALID, case
    assert msg in err, (case, err)


def test_detect_images_sweep_valid_arguments_reach_the_cascade_check():
    rc, err = _detect(_descs((64, 64, 64), (1, 1, 1), (64, 64, 64), (40, 30, 31)), 4)
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err
    rc, err = _detect(_descs((64, 64, 64)), 1, nangles=1)
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err


def test_go_shim_binds_the_sweep_calls():
    header = open(os.path.join(ROOT, "include", "pigo_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    protos = dict(_calls(header, ""))
    assert protos["pigo_run_cascade_images_sweep"] == 17 and protos["pigo_detect_images_sweep"] == 19
    go = "\n".join(open(f).read() for f in sorted(glob.glob(os.path.join(ROOT, "go", "pigo", "*.go"))))
    go = re.sub(r"//[^\n]*", "", go)
    for name in ("pigo_run_cascade_images_sweep", "pigo_detect_images_sweep"):
        calls = [n for nm, n in _calls(go, "C.") if nm == name]
        assert calls and all(n == protos[name] for n in calls), name
    assert re.search(r"^func \(pg \*Pigo\) RunCascadeImagesSweep\(images \[\]ImageParams, cp CascadeParams, angles \[\]float64, iou float64\) "
                     r"\[\]\[\]SweepDetection \{", go, flags=re.M)
    assert re.search(r"^func \(pg \*Pigo\) DetectImagesSweep\(plc \*PuplocCascade, calls \[\]LandmarkCall, images \[\]ImageParams, "
                     r"cp CascadeParams, pp PipelineParams, angles \[\]float64\) \[\]\[\]SweepFace \{", go, flags=re.M)
    assert re.search(r"type SweepDetection struct \{\s*Detection\s*Angle float64\s*\}", go)
    assert re.search(r"type SweepFace struct \{\s*FaceResult\s*Angle float64\s*\}", go)


def test_merge_rule_on_a_hand_made_list():
    """Two angles whose lists overlap at one place: one cluster, tagged with the angle of its largest-Q member; a Q tie
    goes to the angle listed first."""
    a0 = np.array([(100, 100, 40, 5.0), (300, 300, 40, 2.0)], dtype=O.DET_DTYPE)
    a1 = np.array([(102, 101, 40, 7.0), (301, 300, 40, 2.0)], dtype=O.DET_DTYPE)
    cl, idx = S.merge([a0, a1], 0.2)
    assert len(cl) == 2
    by_row = {int(c["row"]) // 100: int(i) for c, i in zip(cl, idx)}
    assert by_row == {1: 1, 3: 0}


@pytest.fixture(scope="module")
def oracle():
    return O.OracleFace(pigo_b200.load_cascade("facefinder"))


@pytest.mark.parametrize("tilt", [0, 30, -45, 100])
def test_oracle_sweep_recovers_the_tilt_of_the_rotated_sample(oracle, tilt):
    """The sample, edge-padded to 520x520 and rotated by `tilt` degrees, swept at k/32: the strongest merged face lies within
    one slot (11.25 degrees) of the tilt, at the DOC parameters with IoU 0.2 and at the TEST parameters with IoU 0.1."""
    img = S.rotate(S.padded_sample(), tilt)
    angles = S.sweep_angles()
    for params, iou in (((20, 1000, 0.1, 1.1), 0.2), ((20, 1000, 0.2, 1.1), 0.1)):
        cl, idx = S.sweep_oracle(oracle, (img, 520, 520, 520), angles, params, iou)
        assert len(cl) > 0
        got = S.strongest_slot(cl, idx, angles)
        assert S.slot_distance(got, S.expected_slot(tilt)) <= 1, (tilt, params, got)
