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
    assert p["tiles_off"] <= SMEM_PER_CTA and 2 * p["region_bytes"] + 384 + p["ks"] * 520 <= SMEM_PER_CTA
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


def _ceil_div_pos(num, den):
    return np.where(num <= 0, 0, (num + den - 1) // den)


def _row_of(kk, nj, magic):
    """region_role's kk / nj: __umulhi(kk, magic) for nj > 1, kk itself for nj <= 1."""
    kk = np.asarray(kk, dtype=np.uint64)
    return np.where(nj > 1, (kk * np.asarray(magic, dtype=np.uint64)) >> np.uint64(32), kk).astype(np.int64)


def _partitions(lo, hi, n):
    """The non-empty intervals [lo, hi) cover 0..n-1 exactly once (and nothing outside)."""
    keep = hi > lo
    assert (lo[keep] >= 0).all() and (hi[keep] <= n).all()
    cover = np.zeros(n + 1, dtype=np.int64)
    np.add.at(cover, lo[keep], 1)
    np.add.at(cover, hi[keep], -1)
    assert (np.cumsum(cover)[:n] == 1).all()


def _deal_regions(p, checked_nj):
    """region_fill's sub-grid arithmetic (scan_tiled.cu) restated in numpy for every band, region and scale of the plan, and
    the dealing of region_role: window k of a sub-grid is row i = kk / nj (by __umulhi(kk, magic)), column kk - i * nj, id
    wid0 + i * ncols + j, buffer offset base + i * step * pitch + j * step.  Region (ry, rx) deals the windows of rows
    [i0, i1) x columns [j0, j1) of each scale, so every window of a band's scales is dealt exactly once iff the row intervals
    of the ry and the column intervals of the rx each partition the scale's rows and columns, and the division is exact for
    every kk < n (checked for each distinct nj over all kk below the largest n it occurs with; checked_nj caches those).
    The id and buffer offset are checked against the window's centre at the four corners of every sub-grid.  Returns the
    windows dealt."""
    scales = p["scales"]
    dealt = 0
    for b in p["regions"]:
        regions_y = b["nregions"] // b["regions_x"]
        for s, step, off, nrows, ncols, wbase in scales[b["scale_lo"]:b["scale_lo"] + b["nscales"]]:
            cy0 = np.arange(regions_y, dtype=np.int64) * b["core_y"]
            cx0 = b["org_x"] + np.arange(b["regions_x"], dtype=np.int64) * b["core_x"]
            i0 = _ceil_div_pos(cy0 - off, step)
            i1 = np.minimum(nrows, _ceil_div_pos(cy0 + b["core_y"] - off, step))
            j0 = _ceil_div_pos(cx0 - off, step)
            j1 = np.minimum(ncols, _ceil_div_pos(cx0 + b["core_x"] - off, step))
            _partitions(i0, i1, nrows)
            _partitions(j0, j1, ncols)
            # per region (ry, rx): lane l's RegionSub of region_fill
            I0, J0 = np.meshgrid(i0, j0, indexing="ij")
            NI, NJ = np.meshgrid(np.maximum(0, i1 - i0), np.maximum(0, j1 - j0), indexing="ij")
            gy0 = (cy0 - b["halo_lo"])[:, None]
            gx0 = (cx0 - b["halo_lo"])[None, :]
            n = NI * NJ
            magic = np.where(NJ > 1, ((1 << 32) + NJ - 1) // np.maximum(NJ, 1), 0)
            assert magic.max() < (1 << 32)
            base = (off + I0 * step - gy0) * 256 + (off + J0 * step - gx0)
            wid0 = wbase + I0 * ncols + J0
            for nj_ in np.unique(NJ[n > 0]):
                top = int(n[NJ == nj_].max())
                if checked_nj.get(int(nj_), 0) < top:
                    kk = np.arange(top, dtype=np.int64)
                    m = ((1 << 32) + int(nj_) - 1) // int(nj_) if nj_ > 1 else 0
                    np.testing.assert_array_equal(_row_of(kk, nj_, m), kk // nj_)   # __umulhi(kk, magic) == kk / nj
                    checked_nj[int(nj_)] = top
            live = n > 0
            for kk in (np.zeros_like(n), NJ - 1, n - NJ, n - 1):   # the corners of each sub-grid
                kk, nj_, m = kk[live], NJ[live], magic[live]
                i = _row_of(kk, nj_, m)
                j = kk - i * nj_
                wid = wid0[live] + i * ncols + j
                r, c = off + step * ((wid - wbase) // ncols), off + step * ((wid - wbase) % ncols)
                assert ((wid >= wbase) & (wid < wbase + nrows * ncols)).all()
                np.testing.assert_array_equal(base[live] + i * step * 256 + j * step,
                                              (r - np.broadcast_to(gy0, n.shape)[live]) * 256 + (c - np.broadcast_to(gx0, n.shape)[live]))
            dealt += int(n.sum())
    return dealt


# option settings that change the region plan: the resident prefix (and with it the buffer size: at 400 trees the buffers
# are about 11 KB and may hold no band), the band width, the largest tiled scale, and the core limits at their extremes
PLAN_OPTIONS = ([{"tile_ks": k} for k in (1, 6, 120, 250, 400)] + [{"tile_band_ratio": r} for r in (100, 110, 400)] +
                [{"tile_max_scale": m} for m in (24, 40, 80)] +
                [{"tile_min_core": 16, "tile_min_core_steps": 1}, {"tile_min_core": 240}, {"tile_min_core": 4000},
                 {"tile_min_core_steps": 40}, {"tile_min_core": 16, "tile_min_core_steps": 1, "tile_ks": 250}])
# settings under which no geometry of the grid gets a region band: 11 KB buffers, a core limit above every region's core
NO_BANDS = [{"tile_ks": 400}, {"tile_min_core": 4000}]


@pytest.mark.parametrize("opt", PLAN_OPTIONS, ids=["-".join(f"{k}{v}" for k, v in o.items()) for o in PLAN_OPTIONS])
def test_region_plan_under_options(opt):
    """_check_regions over the geometry / parameter grid under options that change the region plan, and the sub-grid
    arithmetic of region_fill over every band, region and scale of those plans."""
    planned = 0
    checked_nj = {}
    with options(tile_region=1, **opt):
        for geom in GEOMS:
            for prm in PARAMS:
                p = _check_regions(geom[0], geom[1], prm, nframes=3)
                if "tile_ks" in opt:
                    assert p["ks"] == min(opt["tile_ks"], 468)
                if p["regions"]:
                    planned += 1
                    last = p["regions"][-1]
                    covered = sum(e[3] * e[4] for e in p["scales"][:last["scale_lo"] + last["nscales"]])
                    assert _deal_regions(p, checked_nj) == covered
                    assert p["scales"][last["scale_lo"] + last["nscales"] - 1][0] <= opt.get("tile_max_scale", 1 << 30)
                    assert min(min(b["core_x"], b["core_y"]) for b in p["regions"]) >= opt.get("tile_min_core", 32)
    assert (planned == 0) == (opt in NO_BANDS)
