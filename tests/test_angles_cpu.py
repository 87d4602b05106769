"""CPU-side checks of the per-image angle calls (pigo_run_cascade_images_angles, pigo_detect_images_angles): every invalid
argument, a null `angles` among them, is rejected with PIGO_E_INVALID and a message that names it before any device work,
and the Go shim binds both calls."""
import re

import pytest

import pigo_b200
from abi_cases import (IMAGE_CASES, LATER_PIPELINE_CASES, PIPELINE_CASES, cases_for, descs, detect, go_binds, go_body, go_source, header_protos,
                       scan)

NULL_ANGLES = ("null angles", descs((8, 8, 8)), 1, {"angles": False}, "null angles")


@pytest.mark.parametrize("case,images,nimages,kw,msg", cases_for(IMAGE_CASES, first=[NULL_ANGLES]))
def test_run_cascade_images_angles_rejects_invalid_arguments_before_the_device(case, images, nimages, kw, msg):
    rc, err = scan("pigo_run_cascade_images_angles", images, nimages, **kw)
    assert rc == pigo_b200.PIGO_E_INVALID, case
    assert msg in err, (case, err)


def test_run_cascade_images_angles_valid_arguments_reach_the_cascade_check():
    """Control: valid images (repeated descriptors, no windows) and any angles, NaN and > 1 included, fail only on the NULL
    cascade; with no images a null `angles` is allowed."""
    rc, err = scan("pigo_run_cascade_images_angles", descs((64, 64, 64), (64, 64, 64), (1, 1, 1), (0, 0, 0)), 4)
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err
    rc, err = scan("pigo_run_cascade_images_angles", descs((8, 8, 8)), 0, angles=False)
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err


@pytest.mark.parametrize("case,images,nimages,kw,msg", cases_for(PIPELINE_CASES, first=[NULL_ANGLES], last=LATER_PIPELINE_CASES))
def test_detect_images_angles_rejects_invalid_arguments_before_the_device(case, images, nimages, kw, msg):
    rc, err = detect("pigo_detect_images_angles", images, nimages, **kw)
    assert rc == pigo_b200.PIGO_E_INVALID, case
    assert msg in err, (case, err)


def test_detect_images_angles_valid_arguments_reach_the_cascade_check():
    rc, err = detect("pigo_detect_images_angles", descs((64, 64, 64), (1, 1, 1), (64, 64, 64), (40, 30, 31)), 4)
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err


def test_go_shim_binds_the_angle_calls():
    protos, go = header_protos(), go_source()
    assert protos["pigo_run_cascade_images_angles"] == 13 and protos["pigo_detect_images_angles"] == 17
    for name in ("pigo_run_cascade_images_angles", "pigo_detect_images_angles"):
        assert go_binds(go, name, protos), name
    assert re.search(r"^func \(pg \*Pigo\) RunCascadeImagesAngles\(images \[\]ImageParams, cp CascadeParams, angles \[\]float64\) "
                     r"\[\]\[\]Detection \{", go, flags=re.M)
    assert re.search(r"^func \(pg \*Pigo\) DetectImagesAngles\(plc \*PuplocCascade, calls \[\]LandmarkCall, images \[\]ImageParams, "
                     r"cp CascadeParams, pp PipelineParams, angles \[\]float64\) \[\]\[\]FaceResult \{", go, flags=re.M)
    for fn in ("RunCascadeImagesAngles", "DetectImagesAngles"):
        body = go_body(go, fn)
        assert "len(angles) != len(images)" in body and "panic(" in body, fn
    assert "pp.Sharded" in go_body(go, "DetectImagesAngles")
