"""CPU-side check of the scan schedule (no GPU): the per-warp tiles of every band must PARTITION the windows of the band's
scales (each window centre falls into exactly one tile core), every pixel a window of that tile can sample must lie inside
the tile buffer, and the tile must fit the per-warp shared-memory budget.  Geometry bugs here would silently corrupt the
GPU result, so they are pinned on the host, in the `-m "not gpu"` part of the suite."""
import numpy as np
import pytest

import pigo_b200
from option_guard import options, options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)


def _check(rows, cols, prm, nframes=None):
    p = pigo_b200.describe_plan(rows, cols, *prm, nframes=nframes)
    scales = p["scales"]
    assert sum(e[3] * e[4] for e in scales) == p["windows"] == pigo_b200.count_windows(rows, cols, *prm)
    covered = 0
    for b in p["bands"]:
        tiles_y = b["ntiles"] // b["tiles_x"]
        assert b["ntiles"] == b["tiles_x"] * tiles_y
        assert b["rows_t"] * b["pitch"] <= p["tile_bytes"] and b["pitch"] % 16 == 0 and b["pitch"] >= b["rows_t"]
        assert (b["org_x"] - b["halo_lo"]) % 16 == 0          # TMA row copies need 16-byte aligned tile origins
        for s, step, off, nrows, ncols, wbase in scales[b["scale_lo"]:b["scale_lo"] + b["nscales"]]:
            r = off + step * np.arange(nrows)
            c = off + step * np.arange(ncols)
            ty, tx = r // b["core"], (c - b["org_x"]) // b["core"]
            assert ty.min() >= 0 and ty.max() < tiles_y and tx.min() >= 0 and tx.max() < b["tiles_x"]
            # sample offsets of classifyRegion: (code*s) >> 8 for code in [-128, 127]  (core/pigo.go:126-127)
            lo, hi = (-128 * s) >> 8, (127 * s) >> 8
            # tile-local coordinates of the extreme samples of every window
            ly = r - (ty * b["core"] - b["halo_lo"])
            lx = c - (b["org_x"] + tx * b["core"] - b["halo_lo"])
            assert (ly + lo).min() >= 0 and (ly + hi).max() < b["rows_t"]
            assert (lx + lo).min() >= 0 and (lx + hi).max() < b["pitch"]
            covered += nrows * ncols
    untiled = sum(e[3] * e[4] for e in scales[p["first_untiled"]:])
    assert covered + untiled == p["windows"]
    return p


@pytest.mark.parametrize("geom", [(1080, 1920), (2160, 3840), (400, 320), (97, 131), (720, 1280), (33, 4000)])
@pytest.mark.parametrize("prm", [(20, 1000, 0.2, 1.1), (20, 1000, 0.1, 1.1), (20, 1000, 0.15, 1.15), (12, 90, 0.05, 1.05), (64, 400, 0.3, 1.3)])
def test_tiles_partition_windows_and_contain_all_samples(geom, prm):
    _check(geom[0], geom[1], prm)


def test_plan_follows_the_tuning_options():
    base = _check(1080, 1920, (20, 1000, 0.2, 1.1))
    assert base["bands"] and base["bands"][0]["scale_lo"] == 0
    with options(tile_warps=8):
        big = _check(1080, 1920, (20, 1000, 0.2, 1.1))
        assert big["tile_bytes"] > base["tile_bytes"] and big["first_untiled"] >= base["first_untiled"]
        with options(tile_max_scale=24):
            small = _check(1080, 1920, (20, 1000, 0.2, 1.1))
        assert small["first_untiled"] == 3      # scales 20, 22, 24


def test_offset_table_kernel_plan_keeps_the_tile_invariants():
    """tile_ptab=1 (scan_ptab_kernel) moves the tiles behind two table buffers: same partition / containment invariants, a smaller
    tile budget, offsets that fit 16 bits, at most 32 tiled ladder entries."""
    base = _check(1080, 1920, (20, 1000, 0.2, 1.1))
    for kt, ks, warps in ((16, 24, 24), (4, 6, 7), (60, 48, 12), (1, 1, 24)):
        with options(tile_ptab=1, ptab_kt=kt, ptab_ks=ks, tile_warps=warps):
            for geom, prm in (((1080, 1920), (20, 1000, 0.2, 1.1)), ((2160, 3840), (20, 1000, 0.1, 1.1)), ((97, 131), (12, 90, 0.05, 1.05))):
                p = _check(geom[0], geom[1], prm)
                if p["ptab_kt"] == 0:        # more than 32 tiled ladder entries: the planner falls back to the classic kernel
                    assert p["first_untiled"] > 32
                    continue
                assert p["ptab_kt"] == min(kt, 60) and p["first_untiled"] <= 32
                for b in p["bands"]:
                    assert b["rows_t"] * (b["pitch"] + 1) < 65536
                if warps == 24 and geom == (1080, 1920) and kt == 16:
                    assert p["tiles_off"] > base["tiles_off"] and p["tile_bytes"] <= base["tile_bytes"]


GEOMS = [(1080, 1920), (2160, 3840), (400, 320), (97, 131), (720, 1280), (33, 4000)]
PARAMS = [(20, 1000, 0.2, 1.1), (20, 1000, 0.1, 1.1), (20, 1000, 0.15, 1.15), (12, 90, 0.05, 1.05), (64, 400, 0.3, 1.3)]


@pytest.mark.parametrize("geom", GEOMS)
@pytest.mark.parametrize("ratio", [0, 110, 130, 400])
@pytest.mark.parametrize("head", [1, 2, 3, 4])
def test_single_frame_plans_keep_the_invariants_and_the_dense_head_rules(geom, ratio, head):
    """What one-frame calls run: the band ratio the library picks for them (0 = auto: 140 up to 2 M windows per call, else
    200) or a forced one, with the dense head asked for.  The tiles keep the partition / containment invariants, and
    where the planner keeps the head, the geometry satisfies what the head kernel needs: a resident prefix longer than
    the head and short enough for a ring entry's 6-bit tree field, at most 16 tiled ladder entries (its table slots),
    window sizes that fit the ring entry's 8-bit field, and int16 tile offsets."""
    for prm in PARAMS:
        with options(tile_head=head, tile_band_ratio=ratio):
            p = _check(geom[0], geom[1], prm, nframes=1)
        assert p["band_ratio"] == (ratio if ratio else (140 if p["windows"] <= 2000000 else 200))
        assert p["head"] in (0, head) and p["ptab_kt"] == 0
        if p["head"]:
            assert head < p["ks"] <= 63
            assert p["bands"] and p["first_untiled"] <= 16
            for b in p["bands"]:
                assert p["scales"][b["scale_lo"] + b["nscales"] - 1][0] <= 255
                assert (b["halo_lo"] + 1) * (b["pitch"] + 1) < 32768


def test_describe_plan_plans_for_the_call_s_frame_count():
    """A call of <= 2 M windows plans bands of 1.4x its first scale, a larger one 2x (run_scan's rule); the default
    description is that of a call of many frames."""
    one = pigo_b200.describe_plan(1080, 1920, 20, 1000, 0.2, 1.1, nframes=1)     # 0.9 M windows
    two = pigo_b200.describe_plan(1080, 1920, 20, 1000, 0.2, 1.1, nframes=2)     # 1.8 M
    three = pigo_b200.describe_plan(1080, 1920, 20, 1000, 0.2, 1.1, nframes=3)   # 2.7 M
    many = pigo_b200.describe_plan(1080, 1920, 20, 1000, 0.2, 1.1)
    assert (one["band_ratio"], two["band_ratio"], three["band_ratio"], many["band_ratio"]) == (140, 140, 200, 200)
    assert three["bands"] == many["bands"] and one["bands"] == two["bands"] != many["bands"]
    assert one["head"] == 0 and one["ptab_kt"] == 0 and one["ks"] == pigo_b200.get_option("tile_ks")
    with pytest.raises(pigo_b200.PigoError):
        pigo_b200.describe_plan(1080, 1920, 20, 1000, 0.2, 1.1, nframes=0)
