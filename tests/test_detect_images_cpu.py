"""CPU-side checks of the mixed-size pipeline (pigo_detect_images) and mixed-size RunDetector (pigo_puploc_run_images):
every invalid argument is rejected with PIGO_E_INVALID and a message that names it before any device work, and the Go shim
binds the pipeline call."""
import re

import numpy as np
import pytest

import pigo_b200
from abi_cases import PIPELINE_CASES, descs, detect, go_binds, go_body, go_source, header_protos


@pytest.mark.parametrize("case,images,nimages,kw,msg", PIPELINE_CASES)
def test_detect_images_rejects_invalid_arguments_before_the_device(case, images, nimages, kw, msg):
    rc, err = detect("pigo_detect_images", images, nimages, **kw)
    assert rc == pigo_b200.PIGO_E_INVALID, case
    assert msg in err, (case, err)


def test_detect_images_valid_arguments_reach_the_cascade_check():
    """Control for the cases above: valid images (odd pitches, one pixel, no windows) fail only on the NULL cascade."""
    rc, err = detect("pigo_detect_images", descs((64, 64, 64), (1, 1, 1), (10, 10, 16), (40, 30, 31)), 4)
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
    ("negative nseeds", (_seeds(1), -1, None, descs((8, 8, 8)), 1), "negative nseeds"),
    ("null seeds", (None, 1, None, descs((8, 8, 8)), 1), "null seeds"),
    ("no images", (_seeds(1), 1, None, descs((8, 8, 8)), 0), "nimages"),
    ("too many images", (_seeds(1), 1, [0], descs((8, 8, 8)), 65536), "nimages"),
    ("null images", (_seeds(1), 1, None, None, 1), "null images"),
    ("seed_image missing", (_seeds(1), 1, None, descs((8, 8, 8), (9, 9, 9)), 2), "seed_image is required"),
    ("zero rows", (_seeds(1), 1, [0], descs((8, 8, 8), (0, 9, 9)), 2), "image 1: bad geometry"),
    ("dim < cols", (_seeds(1), 1, None, descs((8, 9, 8)), 1), "image 0: bad geometry"),
    ("rows*dim >= 2^31", (_seeds(1), 1, None, descs((65536, 32768, 32768)), 1), "image 0: larger than 2^31"),
    ("null pixels", (_seeds(1), 1, None, descs((8, 8, 8), pixels=None), 1), "image 0: null pixels"),
    ("perturbs > 63", (_seeds(3, 64), 2, None, descs((8, 8, 8)), 1), "seed 1: Perturbs=64"),
    ("negative perturbs", (_seeds(-1), 1, None, descs((8, 8, 8)), 1), "seed 0: Perturbs=-1"),
    ("image index past the end", (_seeds(1, 1), 2, [1, 2], descs((8, 8, 8), (9, 9, 9)), 2), "seed 1: image index out of range"),
    ("negative image index", (_seeds(1), 1, [-1], descs((8, 8, 8), (9, 9, 9)), 2), "seed 0: image index out of range"),
])
def test_puploc_run_images_rejects_invalid_arguments_before_the_device(case, args, msg):
    rc, err = _run_images(*args)
    assert rc == pigo_b200.PIGO_E_INVALID, case
    assert msg in err, (case, err)


def test_puploc_run_images_null_out_and_valid_arguments():
    rc, err = _run_images(_seeds(1), 1, None, descs((8, 8, 8)), 1, out=False)
    assert rc == pigo_b200.PIGO_E_INVALID and "null out" in err
    rc, err = _run_images(_seeds(0, 63, 7), 3, [0, 2, 1], descs((8, 8, 8), (1, 1, 1), (30, 40, 41)), 3)
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err


def test_go_shim_binds_detect_images():
    protos, go = header_protos(), go_source()
    assert protos["pigo_detect_images"] == 16 and protos["pigo_puploc_run_images"] == 13
    assert go_binds(go, "pigo_detect_images", protos)
    assert re.search(r"^func \(pg \*Pigo\) DetectImages\(plc \*PuplocCascade, calls \[\]LandmarkCall, images \[\]ImageParams, "
                     r"cp CascadeParams, pp PipelineParams\) \[\]\[\]FaceResult \{", go, flags=re.M)
    body = go_body(go, "DetectImages")
    assert "pp.Sharded" in body and "panic(" in body and "C.PIGO_E_CAP" in body
    assert "C.pigo_alloc_pinned" in body and "C.malloc" in body
