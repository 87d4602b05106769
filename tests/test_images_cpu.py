"""CPU-side checks of pigo_run_cascade_images (mixed-size RunCascade): every invalid argument is rejected with
PIGO_E_INVALID before any device work, and the Go shim binds the entry point."""
import re

import pytest

import pigo_b200
from abi_cases import IMAGE_CASES, descs, go_binds, go_source, header_protos, scan


@pytest.mark.parametrize("case,images,nimages,kw,msg", IMAGE_CASES)
def test_invalid_arguments_are_rejected_before_the_device(case, images, nimages, kw, msg):
    rc, err = scan("pigo_run_cascade_images", images, nimages, **kw)
    assert rc == pigo_b200.PIGO_E_INVALID, case
    assert msg in err, (case, err)


def test_valid_arguments_reach_the_cascade_check():
    """Control for the cases above: the same call with valid images fails only on the NULL cascade."""
    rc, err = scan("pigo_run_cascade_images", descs((64, 64, 64), (1, 1, 1), (0, 0, 0)), 3)
    assert rc == pigo_b200.PIGO_E_INVALID and "null cascade" in err


def test_descriptor_layout_matches_the_header():
    import ctypes as C
    assert C.sizeof(pigo_b200.PigoImage) == 24
    assert [pigo_b200.PigoImage.pixels.offset, pigo_b200.PigoImage.rows.offset, pigo_b200.PigoImage.cols.offset,
            pigo_b200.PigoImage.dim.offset] == [0, 8, 12, 16]


def test_go_shim_binds_run_cascade_images():
    protos, go = header_protos(), go_source()
    assert protos["pigo_run_cascade_images"] == 13 and go_binds(go, "pigo_run_cascade_images", protos)
    assert re.search(r"^func \(pg \*Pigo\) RunCascadeImages\(images \[\]ImageParams, cp CascadeParams, angle float64\) \[\]\[\]Detection \{",
                     go, flags=re.M)
    assert "C.pigo_alloc_pinned" in go and "C.malloc" in go   # pixels and descriptors in C memory (cgo pointer rules)
