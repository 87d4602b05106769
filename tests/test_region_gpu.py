"""The fused kernel's region role (tile warps dealing windows from two shared, double-buffered region buffers per CTA),
forced with tile_region=1, against the C oracle; and the full-size bench batch with the role the planner picks (the region
role) against the per-warp tiles (tile_region=2), byte for byte."""
import numpy as np
import pytest

import pigo_b200
from pigo_b200 import synth
from option_guard import options, options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)
from test_gpu_parity import CLI_PARAMS, DOC_PARAMS, TEST_PARAMS, assert_same, cp_of

pytestmark = pytest.mark.gpu


def run_timed(fn):
    with options(timing=1):
        out = fn()
        launches = {k: pigo_b200.get_option(k) for k in ("t_tiled_n", "t_gather_n", "t_deep_n", "t_region_n")}
    return out, launches


def assert_region_ran(launches, rows, cols, prm, nframes, groups=1, gather=False):
    """Every fused launch of the call ran the region role (t_region_n counts those, after their tensor maps were encoded:
    a fallback to the per-warp tiles shows as 0), and the planner says so too."""
    assert launches == {"t_tiled_n": groups, "t_gather_n": groups * gather, "t_deep_n": groups, "t_region_n": groups}, launches
    assert pigo_b200.describe_plan(rows, cols, *prm, nframes=nframes)["region"] == 1


REGION_VARIANTS = [
    {},
    {"gather_warps": 0},
    {"queue_cap": 40, "tile_ks": 4, "gather_ks": 6},     # deep queue full: old-region flush and tail fail, windows finish in place
    {"queue_cap": 3000},
    {"tile_tail_min": 0},
    {"tile_tail_min": 33},
]


@pytest.mark.parametrize("variant", REGION_VARIANTS, ids=[f"variant{i}" for i in range(len(REGION_VARIANTS))])
def test_region_role_agrees_with_oracle(gpu_face, oracle_face, sample_gray, variant):
    frames = synth.make_batch(3, 720, 1280, "SFU", seed0=21)
    cases = [(frames[0], 720, 1280, 1280, TEST_PARAMS), (frames[1], 720, 1280, 1280, DOC_PARAMS),
             (frames[2], 720, 1280, 1280, CLI_PARAMS), (sample_gray, 400, 320, 320, (20, 1000, 0.05, 1.05)),
             (sample_gray, 400, 320, 320, TEST_PARAMS)]
    gather = variant.get("gather_warps", 8) == 0
    with options(tile_region=1, **variant):
        _, launches = run_timed(lambda: gpu_face.run_cascade_array(cp_of(frames[0], 720, 1280, 1280, TEST_PARAMS), 0.0))
        assert_region_ran(launches, 720, 1280, TEST_PARAMS, 1, gather=gather)
        for img, r, c, d, prm in cases:
            assert_same(gpu_face.run_cascade_array(cp_of(img, r, c, d, prm), 0.0), oracle_face.run_cascade(img, r, c, d, *prm, 0.0))
        dets, cnt = gpu_face.RunCascadeBatch(frames, cp_of(None, 720, 1280, 1280, TEST_PARAMS), 0.0, cap_per_frame=512)
    for f in range(3):
        o = oracle_face.run_cascade(frames[f], 720, 1280, 1280, *TEST_PARAMS, 0.0)
        assert cnt[f] == len(o) and dets[f, :cnt[f]].tobytes() == o.tobytes()


@pytest.mark.parametrize("variant,groups", [({"host_stream": 1, "copy_chunk": 1, "sub_batch": 4}, 3), ({"host_stream": 1, "copy_chunk": 3}, 1),
                                            ({"host_stream": 0, "sub_batch": 4}, 3)])
def test_region_role_batches_and_host_streamed_frames(gpu_face, oracle_face, variant, groups):
    """An 11-frame batch over several pipeline groups, frames streamed from the host behind the copy: the filling warp waits
    for a region's frame before it issues the region's copies."""
    frames = synth.make_batch(11, 270, 480, "USF", seed0=77)
    with options(tile_region=1, **variant):
        for prm in (TEST_PARAMS, DOC_PARAMS):
            (dets, cnt), launches = run_timed(lambda: gpu_face.RunCascadeBatch(frames, cp_of(None, 270, 480, 480, prm), 0.0, cap_per_frame=256))
            assert_region_ran(launches, 270, 480, prm, 11, groups)
            for f in range(11):
                o = oracle_face.run_cascade(frames[f], 270, 480, 480, *prm, 0.0)
                assert cnt[f] == len(o) and dets[f, :cnt[f]].tobytes() == o.tobytes()


def test_full_size_batch_region_role_equals_per_warp_tiles(gpu_face, oracle_face):
    """configs[2] (256 x 1080p, the bench workload, device resident): the default plan runs the region role and gives the
    same counts and detections as the per-warp tiles, byte for byte; sampled frames equal the oracle."""
    import torch
    nf, R, C = 256, 1080, 1920
    base = synth.make_batch(12, R, C, "USF")
    frames = np.concatenate([base] * ((nf + 11) // 12))[:nf]
    cap = 256
    d = torch.from_numpy(frames).cuda()

    def run():
        d_out = torch.zeros((nf, cap, 4), dtype=torch.int32, device="cuda")
        d_cnt = torch.zeros(nf, dtype=torch.int32, device="cuda")
        gpu_face.run_cascade_batch_device(d.data_ptr(), nf, R * C, R, C, C, *TEST_PARAMS, 0.0, d_out.data_ptr(), cap, d_cnt.data_ptr())
        torch.cuda.synchronize()
        return d_cnt.cpu().numpy(), d_out.cpu().numpy()

    (cnt, dets), launches = run_timed(run)
    assert_region_ran(launches, R, C, TEST_PARAMS, nf, groups=2)
    with options(tile_region=2):
        (cnt2, dets2), launches2 = run_timed(run)
        assert pigo_b200.describe_plan(R, C, *TEST_PARAMS, nframes=nf)["region"] == 0
    assert launches2 == dict(launches, t_region_n=0)
    assert int(cnt.max()) <= cap
    assert cnt.tobytes() == cnt2.tobytes() and dets.tobytes() == dets2.tobytes()
    for f in (0, 5, 255):
        o = oracle_face.run_cascade(frames[f], R, C, C, *TEST_PARAMS, 0.0)
        assert cnt[f] == len(o) and dets[f, :cnt[f]].tobytes() == o.tobytes()
    del d
