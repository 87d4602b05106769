"""CPU-side check of the fused kernel's region role plan (no GPU): the regions of every band PARTITION the windows of the
band's scales, every pixel a window can sample lies inside its region buffer, two buffers and the cascade prefix fit the
227 KB of shared memory, no TMA box dimension exceeds 256, and the planner picks the region role by the call's windows (more
than 2 M, at most one per frame pixel) unless an option names another role."""
import numpy as np
import pytest

import pigo_b200
from option_guard import options, options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)

GEOMS = [(1080, 1920), (2160, 3840), (400, 320), (97, 131), (720, 1280), (33, 4000)]
PARAMS = [(20, 1000, 0.2, 1.1), (20, 1000, 0.1, 1.1), (20, 1000, 0.15, 1.15), (12, 90, 0.05, 1.05), (64, 400, 0.3, 1.3)]
SMEM_PER_CTA = 232448   # 227 KB opt-in maximum on sm_90


def _check_regions(rows, cols, prm, nframes=None):
    p = pigo_b200.describe_plan(rows, cols, *prm, nframes=nframes)
    scales = p["scales"]
    if not p["regions"]:
        assert p["region"] == 0
        return p
    assert p["region_bytes"] % 256 == 0
    assert p["tiles_off"] <= SMEM_PER_CTA and 2 * p["region_bytes"] + 384 + 48 * 520 <= SMEM_PER_CTA
    covered = 0
    for b in p["regions"]:
        assert 1 <= b["nscales"] <= 32
        assert b["pitch"] == 256 and b["box_rows"] <= 256 and b["pitch"] <= 256
        nbox = -(-b["rows_r"] // b["box_rows"])
        assert nbox * b["box_rows"] * b["pitch"] <= p["region_bytes"]
        assert b["core_x"] % 16 == 0 and (b["org_x"] - b["halo_lo"]) % 16 == 0   # 16-byte aligned region origins
        regions_y = b["nregions"] // b["regions_x"]
        assert b["nregions"] == b["regions_x"] * regions_y
        for s, step, off, nrows, ncols, wbase in scales[b["scale_lo"]:b["scale_lo"] + b["nscales"]]:
            r = off + step * np.arange(nrows)
            c = off + step * np.arange(ncols)
            ry, rx = r // b["core_y"], (c - b["org_x"]) // b["core_x"]
            # every window centre falls into exactly one region core (floor division), and that region exists
            assert ry.min() >= 0 and ry.max() < regions_y and rx.min() >= 0 and rx.max() < b["regions_x"]
            # sample offsets of classifyRegion: (code*s) >> 8 for code in [-128, 127]  (core/pigo.go:126-127)
            lo, hi = (-128 * s) >> 8, (127 * s) >> 8
            ly = r - (ry * b["core_y"] - b["halo_lo"])
            lx = c - (b["org_x"] + rx * b["core_x"] - b["halo_lo"])
            assert (ly + lo).min() >= 0 and (ly + hi).max() < b["rows_r"]
            assert (lx + lo).min() >= 0 and (lx + hi).max() < b["pitch"]
            covered += nrows * ncols
    assert p["regions"][0]["scale_lo"] == 0
    for a, b in zip(p["regions"], p["regions"][1:]):
        assert b["scale_lo"] == a["scale_lo"] + a["nscales"]
    last = p["regions"][-1]
    assert p["region_first_untiled"] == last["scale_lo"] + last["nscales"]
    untiled = sum(e[3] * e[4] for e in scales[p["region_first_untiled"]:])
    assert covered + untiled == p["windows"]
    return p


@pytest.mark.parametrize("geom", GEOMS)
@pytest.mark.parametrize("prm", PARAMS)
def test_regions_partition_windows_and_contain_all_samples(geom, prm):
    with options(tile_region=1):
        p = _check_regions(geom[0], geom[1], prm)
    assert p["region"] == (1 if p["regions"] and geom[1] % 16 == 0 else 0)


def test_region_role_follows_the_call_and_the_options():
    """Auto: calls of more than 2 M windows with at most one window per frame pixel -- off at one or two 1080p frames of the
    test parameters (0.9 M windows, 0.43 per pixel), on from three frames up, off at ShiftFactor 0.1 (2 windows per pixel)
    at any frame count; 1 runs the region role for any call, 2 never; the options that name another tile role keep it."""
    prm = (20, 1000, 0.2, 1.1)
    auto = [pigo_b200.describe_plan(1080, 1920, *prm, nframes=n)["region"] for n in (1, 2, 3, 256)]
    assert auto == [0, 0, 1, 1]
    assert [pigo_b200.describe_plan(1080, 1920, 20, 1000, 0.1, 1.1, nframes=n)["region"] for n in (1, 64, 256)] == [0, 0, 0]
    with options(tile_region=1):
        assert [pigo_b200.describe_plan(1080, 1920, 20, 1000, 0.1, 1.1, nframes=n)["region"] for n in (1, 64)] == [1, 1]
    with options(tile_region=1):
        assert _check_regions(1080, 1920, prm, nframes=1)["region"] == 1
        assert _check_regions(400, 320, prm, nframes=1)["region"] == 1
        assert pigo_b200.describe_plan(301, 500, *prm, nframes=1)["region"] == 0            # Dim % 16 != 0: no tensor map
        for opt in ({"tile_head": 2}, {"tile_ptab": 1}, {"fused_smem_kb": 200}, {"tile_ni": 2}, {"tile_prefetch": 1}, {"tile_tmap": 0}):
            with options(**opt):
                assert pigo_b200.describe_plan(1080, 1920, *prm, nframes=256)["region"] == 0, opt
    with options(tile_region=2):
        assert pigo_b200.describe_plan(1080, 1920, *prm, nframes=256)["region"] == 0
    # the classic keys keep describing the per-warp tiles whatever the role
    with options(tile_region=2):
        off = pigo_b200.describe_plan(1080, 1920, *prm)
    on = pigo_b200.describe_plan(1080, 1920, *prm)
    assert on["region"] == 1 and off["region"] == 0
    for k in ("bands", "tile_bytes", "first_untiled", "tiles_off", "band_ratio", "ks", "head", "ptab_kt"):
        assert on[k] == off[k], k


@pytest.mark.parametrize("frames", [1, 3, 64])
def test_region_plan_for_the_call_s_frame_count(frames):
    with options(tile_region=1):
        for geom in GEOMS:
            for prm in PARAMS:
                _check_regions(geom[0], geom[1], prm, nframes=frames)
