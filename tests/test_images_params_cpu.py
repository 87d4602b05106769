"""CPU-side checks of pigo_run_cascade_images_params / pigo_detect_images_params (every image of a mixed-size call with its own
CascadeParams): invalid arguments, including one image's parameters that pigo_run_cascade rejects, fail with PIGO_E_INVALID
before any device work and name the image; pigo_cascade_params has the header's layout; the Go shim binds both calls."""
import ctypes as C
import re

import numpy as np
import pytest

import pigo_b200
from abi_cases import FAKE, IMAGE_CASES, LATER_PIPELINE_CASES, PIPELINE_CASES, cases_for, descs, go_binds, go_body, go_source, header_protos

GOOD = (20, 1000, 0.2, 1.1)
NEGATIVE = (-30, 10, 0.2, 1.1)        # the ladder reaches a negative window size
LONG = (0, 200000, 0.2, 1.0)          # 100001 ladder entries, more than the 65536 the library accepts


def scan(images, nimages, params=(GOOD,) * 4, angles=True, cap=4, with_n_out=True, with_out=True, face=None):
    """pigo_run_cascade_images_params with NULL cascade (or `face`).  Returns (status, message)."""
    L = pigo_b200.lib()
    out = np.zeros((4, max(cap, 1)), dtype=pigo_b200.DET_DTYPE)
    cnt = np.zeros(4, dtype=np.int32)
    ang = np.zeros(4, dtype=np.float64)
    prm = pigo_b200.cascade_params_array(params) if params is not None else None
    rc = L.pigo_run_cascade_images_params(face, images, nimages, prm, ang.ctypes.data if angles else None, out.ctypes.data if with_out else None,
                                          cap, cnt.ctypes.data if with_n_out else None, pigo_b200.MEM_HOST, None)
    return rc, L.pigo_last_error().decode()


def detect(images, nimages, cparams=(GOOD,) * 8, face=None, puploc=None, flp="default", ncalls=2, face_cap=4, prm_kw=None, faces=True,
           n_faces=True, points=True, params=True):
    """pigo_detect_images_params with NULL cascades unless given.  Returns (status, message)."""
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
    cp = pigo_b200.cascade_params_array(cparams) if cparams is not None else None
    rc = L.pigo_detect_images_params(face, puploc, hs, fl.ctypes.data, ncalls, images, nimages, cp, None, C.byref(prm) if params else None, None, 0,
                                     out_f.ctypes.data if faces else None, face_cap, out_n.ctypes.data if n_faces else None,
                                     out_p.ctypes.data if points else None, pigo_b200.MEM_HOST, None)
    return rc, L.pigo_last_error().decode()


# the cases of the shared-parameter call, then the ones of the parameter array: a handle that validation never dereferences
# (the bad parameters fail first) lets the per-image checks run, since the cascade is validated before the ladders
PARAM_CASES = [
    ("null params", descs((8, 8, 8)), 1, {"params": None}, "null params"),
    ("negative window, image 1", descs((64, 64, 64), (64, 64, 64)), 2, {"params": (GOOD, NEGATIVE), "face": FAKE}, "image 1: negative window size"),
    ("long ladder, image 2", descs((64, 64, 64), (8, 8, 8), (1, 1, 1)), 3, {"params": (GOOD, GOOD, LONG), "face": FAKE},
     "image 2: scale ladder longer than 65536"),
    ("negative window, image 0", descs((8, 8, 8)), 1, {"params": (NEGATIVE,), "face": FAKE}, "image 0: negative window size"),
]


@pytest.mark.parametrize("case,images,nimages,kw,msg", IMAGE_CASES + PARAM_CASES)
def test_invalid_arguments_are_rejected_before_the_device(case, images, nimages, kw, msg):
    rc, err = scan(images, nimages, **kw)
    assert rc == pigo_b200.PIGO_E_INVALID, case
    assert msg in err, (case, err)


def test_angles_may_be_null_and_valid_arguments_reach_the_cascade_check():
    """Control for the cases above: valid images and parameters, with or without angles, fail only on the NULL cascade."""
    for angles in (True, False):
        rc, err = scan(descs((64, 64, 64), (1, 1, 1), (0, 0, 0)), 3, params=(GOOD, (60, 600, 0.1, 1.1), (200, 480, 0.1, 1.1)), angles=angles)
        assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err, err


PIPELINE_PARAM_CASES = [
    ("null cparams", descs((8, 8, 8)), 1, {"cparams": None}, "null cparams"),
    ("negative window, image 1", descs((64, 64, 64), (64, 64, 64)), 2,
     {"cparams": (GOOD, NEGATIVE), "face": FAKE, "puploc": FAKE, "flp": (C.c_void_p * 2)(FAKE, FAKE)}, "image 1: negative window size"),
    ("long ladder, image 0", descs((64, 64, 64)), 1, {"cparams": (LONG,), "face": FAKE, "puploc": FAKE, "flp": (C.c_void_p * 2)(FAKE, FAKE)},
     "image 0: scale ladder longer than 65536"),
]


@pytest.mark.parametrize("case,images,nimages,kw,msg", cases_for(PIPELINE_CASES, last=LATER_PIPELINE_CASES) + PIPELINE_PARAM_CASES)
def test_pipeline_invalid_arguments_are_rejected_before_the_device(case, images, nimages, kw, msg):
    rc, err = detect(images, nimages, **kw)
    assert rc == pigo_b200.PIGO_E_INVALID, case
    assert msg in err, (case, err)


def test_pipeline_valid_arguments_reach_the_cascade_check():
    """The scan fields of the pipeline parameters are not read: values pigo_run_cascade would reject still reach the handle check."""
    rc, err = detect(descs((64, 64, 64), (8, 8, 8)), 2, cparams=(GOOD, (60, 600, 0.1, 1.1)),
                     prm_kw={"min_size": -30, "max_size": 10, "shift_factor": float("nan"), "scale_factor": 1.0})
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err, err


def test_cascade_params_layout_matches_the_header():
    P = pigo_b200.PigoCascadeParams
    assert C.sizeof(P) == 24
    assert [P.min_size.offset, P.max_size.offset, P.shift_factor.offset, P.scale_factor.offset] == [0, 4, 8, 16]
    a = pigo_b200.cascade_params_array([pigo_b200.CascadeParams(pigo_b200.ImageParams(), 60, 600, 0.1, 1.1), (20, 1000, 0.2, 1.1)])
    assert (a[0].min_size, a[0].max_size, a[0].shift_factor, a[0].scale_factor) == (60, 600, 0.1, 1.1)
    assert (a[1].min_size, a[1].max_size, a[1].shift_factor, a[1].scale_factor) == (20, 1000, 0.2, 1.1)


def test_go_shim_binds_both_calls():
    protos, go = header_protos(), go_source()
    assert protos["pigo_run_cascade_images_params"] == 10 and go_binds(go, "pigo_run_cascade_images_params", protos)
    assert protos["pigo_detect_images_params"] == 18 and go_binds(go, "pigo_detect_images_params", protos)
    assert re.search(r"^func \(pg \*Pigo\) RunCascadeImagesParams\(cps \[\]CascadeParams, angles \[\]float64\) \[\]\[\]Detection \{", go, flags=re.M)
    assert re.search(r"^func \(pg \*Pigo\) DetectImagesParams\(plc \*PuplocCascade, calls \[\]LandmarkCall, cps \[\]CascadeParams, pp PipelineParams, "
                     r"angles \[\]float64\) \[\]\[\]FaceResult \{", go, flags=re.M)
    for fn in ("RunCascadeImagesParams", "DetectImagesParams"):
        assert "packImages(images)" in go_body(go, fn), fn   # host pixels listed several times are copied once
