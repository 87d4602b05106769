"""CPU-side checks of the angle sweep (pigo_run_cascade_images_sweep, pigo_detect_images_sweep): every invalid argument is
rejected with PIGO_E_INVALID before any device work, valid ones reach the cascade check, the Go shim binds both calls, and
the oracle restatement of the merge (tests/sweep_oracle.py) recovers the tilt of the rotated sample within one slot."""
import re

import numpy as np
import pytest

import oracle_lib as O
import pigo_b200
import sweep_oracle as S
from abi_cases import IMAGE_CASES, LATER_PIPELINE_CASES, PIPELINE_CASES, cases_for, descs, detect, go_binds, go_source, header_protos, scan

NULL_ANGLES = ("null angles", descs((8, 8, 8)), 1, {"angles": False}, "null angles")
NO_ANGLES = ("no angles", descs((8, 8, 8)), 1, {"nangles": 0}, "nangles")
# with four angles, 65536 images (or 65535 images of 4096 faces) first exceed the 65535 scan entries: one angle reaches the
# nimages (or the pupil work) check
TOO_MANY_IMAGES = ("too many images", descs((8, 8, 8)), 65536, {"nangles": 1}, "nimages")


@pytest.mark.parametrize("case,images,nimages,kw,msg", cases_for(IMAGE_CASES, own=[TOO_MANY_IMAGES], last=("too many images",), first=[
    NULL_ANGLES, NO_ANGLES,
    ("negative nangles", descs((8, 8, 8)), 1, {"nangles": -1}, "nangles"),
    ("entries > 65535", descs((8, 8, 8)), 16384, {"nangles": 4}, "exceeds 65535"),
    ("negative det_cap", descs((8, 8, 8)), 1, {"det_cap": -1}, "det_cap"),
    ("merged > 2^31-1", descs((8, 8, 8)), 16383, {"det_cap": 1 << 16}, "exceeds 2^31-1"),
]))
def test_run_cascade_images_sweep_rejects_invalid_arguments_before_the_device(case, images, nimages, kw, msg):
    rc, err = scan("pigo_run_cascade_images_sweep", images, nimages, **kw)
    assert rc == pigo_b200.PIGO_E_INVALID, case
    assert msg in err, (case, err)


def test_run_cascade_images_sweep_valid_arguments_reach_the_cascade_check():
    rc, err = scan("pigo_run_cascade_images_sweep", descs((64, 64, 64), (64, 64, 64), (1, 1, 1), (0, 0, 0)), 4)
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err
    rc, err = scan("pigo_run_cascade_images_sweep", descs((8, 8, 8)), 0, nangles=1)
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err


@pytest.mark.parametrize("case,images,nimages,kw,msg", cases_for(PIPELINE_CASES, last=LATER_PIPELINE_CASES, first=[
    NULL_ANGLES, NO_ANGLES,
    ("entries > 65535", descs((8, 8, 8)), 32768, {"nangles": 2}, "exceeds 65535"),
    ("merged > 2^31-1", descs((8, 8, 8)), 16000, {"prm_kw": {"det_cap": 1 << 16}}, "exceeds 2^31-1"),
], own=[
    TOO_MANY_IMAGES,
    ("pupil work > 2^31-1", descs((8, 8, 8)), 65535, {"nangles": 1, "face_cap": 4096, "ncalls": 30}, "exceeds 2^31-1 pupil"),
]))
def test_detect_images_sweep_rejects_invalid_arguments_before_the_device(case, images, nimages, kw, msg):
    rc, err = detect("pigo_detect_images_sweep", images, nimages, **kw)
    assert rc == pigo_b200.PIGO_E_INVALID, case
    assert msg in err, (case, err)


def test_detect_images_sweep_valid_arguments_reach_the_cascade_check():
    rc, err = detect("pigo_detect_images_sweep", descs((64, 64, 64), (1, 1, 1), (64, 64, 64), (40, 30, 31)), 4)
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err
    rc, err = detect("pigo_detect_images_sweep", descs((64, 64, 64)), 1, nangles=1)
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err


def test_go_shim_binds_the_sweep_calls():
    protos, go = header_protos(), go_source()
    assert protos["pigo_run_cascade_images_sweep"] == 17 and protos["pigo_detect_images_sweep"] == 19
    for name in ("pigo_run_cascade_images_sweep", "pigo_detect_images_sweep"):
        assert go_binds(go, name, protos), name
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
