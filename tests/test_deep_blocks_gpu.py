"""The unrotated deep kernel reads the face cascade from a block-interleaved copy (trees 8b..8b+7 side by side, node by
node), so that the 8 lanes of a group share cache lines.  The copy must be the reference tables byte for byte, and the
detections must stay what the reference computes, whatever tree a deep-queue item starts at (gather hand-over point,
resident prefix of the tile warps, straggler threshold) and whatever the lane-group width and queue capacity."""
import ctypes as C

import numpy as np
import pytest

import pigo_b200
from pigo_b200 import CascadeParams, ImageParams, synth
from option_guard import options, options_at_defaults   # noqa: F401 (autouse: every test ends with the options at their defaults)
from oracle.np_oracle import FaceCascade

pytestmark = pytest.mark.gpu

PARAMS = (20, 1000, 0.2, 1.1)
R, C_ = 1080, 1920
NF = 6   # 5.4 M windows: above the 4 M-window threshold of the image-ordered deep queue
KNOBS = ("gather_limit", "tile_ks", "tile_tail_min", "deep_group", "queue_cap")


def pack_blocks(cas: FaceCascade) -> bytes:
    """Host restatement of the device layout: 4096-byte blocks of 8 trees; the last block's pad slots repeat the last tree."""
    n = cas.ntrees
    nblk = (n + 7) // 8
    t = np.minimum(np.arange(nblk * 8), n - 1).reshape(nblk, 8)
    words = cas.codes.reshape(n, 64, 4).view("<i4").reshape(n, 64)      # code word of node idx
    blk = np.zeros((nblk, 64, 8, 2), dtype="<u4")                        # [block][row p][slot][pair]
    blk[:, 0, :4, :] = cas.thresh[t].view("<u4").reshape(nblk, 4, 2)     # bytes 0..31: thresholds
    blk[:, 0, 4:, :] = words[t, 1].view("<u4").reshape(nblk, 4, 2)       # bytes 32..63: root code words
    p = np.arange(1, 32)
    blk[:, 1:32, :, 0] = words[t][:, :, 2 * p].transpose(0, 2, 1).view("<u4")
    blk[:, 1:32, :, 1] = words[t][:, :, 2 * p + 1].transpose(0, 2, 1).view("<u4")
    p = np.arange(32, 64)
    leaves = cas.preds.view("<u4")
    blk[:, 32:, :, 0] = leaves[t][:, :, 2 * p - 64].transpose(0, 2, 1)
    blk[:, 32:, :, 1] = leaves[t][:, :, 2 * p - 63].transpose(0, 2, 1)
    return blk.tobytes()


def device_blocks(face) -> bytes:
    L = pigo_b200.lib()
    n = C.c_size_t(0)
    assert L.pigo_cascade_block_table(face._h, None, C.byref(n)) == pigo_b200.PIGO_OK
    buf = (C.c_uint8 * n.value)()
    assert L.pigo_cascade_block_table(face._h, buf, C.byref(n)) == pigo_b200.PIGO_OK
    return bytes(buf)


def test_block_table_matches_host_packing(gpu_face, facefinder_bytes):
    cas = FaceCascade(facefinder_bytes)
    assert cas.depth == 6 and cas.ntrees % 8 != 0          # 468 trees: the last block is padded
    got = device_blocks(gpu_face)
    assert len(got) == (cas.ntrees + 7) // 8 * 4096
    assert got == pack_blocks(cas)


@pytest.fixture(scope="module")
def frames():
    return synth.make_batch(NF, R, C_, "USF", seed0=31)


@pytest.fixture(scope="module")
def oracle_dets(oracle_face, frames):
    return [oracle_face.run_cascade(frames[f], R, C_, C_, *PARAMS, 0.0) for f in range(NF)]


# every value of each knob at least once: gather hand-over 8/16/24, tile-resident prefix 32/48, straggler threshold 2/16 (items
# start at every tree mod 8), lane groups of 8/16/32, and a queue so small that every producer overflows it
CASES = [
    (16, 48, 6, 8, 0),
    (8, 32, 2, 8, 0),
    (24, 48, 16, 8, 0),
    (16, 32, 16, 16, 0),
    (8, 48, 2, 32, 0),
    (24, 32, 6, 16, 50),
]


@pytest.mark.parametrize("gather_limit,tile_ks,tile_tail_min,deep_group,queue_cap", CASES)
def test_deep_blocks_batch_matches_oracle_and_single_frames(gpu_face, frames, oracle_dets,
                                                            gather_limit, tile_ks, tile_tail_min, deep_group, queue_cap):
    cp = CascadeParams(ImageParams(None, R, C_, C_), *PARAMS)
    with options(**dict(zip(KNOBS, (gather_limit, tile_ks, tile_tail_min, deep_group, queue_cap)))):
        dets, cnt = gpu_face.RunCascadeBatch(frames, cp, 0.0)
        for f in range(NF):
            one = gpu_face.run_cascade_array(CascadeParams(ImageParams(frames[f], R, C_, C_), *PARAMS), 0.0)
            assert cnt[f] == len(one) and dets[f, :cnt[f]].tobytes() == one.tobytes(), f"frame {f}"
            assert one.tobytes() == oracle_dets[f].tobytes(), f"frame {f}"
    assert sum(len(o) for o in oracle_dets) > 0


@pytest.mark.parametrize("deep_group", [8, 32])
def test_deep_blocks_ragged_images_match_single_image_calls(gpu_face, frames, deep_group):
    with options(deep_group=deep_group):
        _ragged_images_match_single_image_calls(gpu_face, frames)


def _ragged_images_match_single_image_calls(gpu_face, frames):
    cp = CascadeParams(ImageParams(None, R, C_, C_), *PARAMS)
    sizes = [(R, C_), (720, 1280), (1000, 1900), (480, 640), (1080, 1500), (333, 517), (900, 1920), (1079, 1919)]
    imgs = [ImageParams(np.ascontiguousarray(frames[i % NF][:r, :c]), r, c, c) for i, (r, c) in enumerate(sizes)]
    for group in (imgs, imgs[3:6]):   # > 4 M windows (image-ordered deep queue) and a small call
        dets, cnt = gpu_face.RunCascadeImages(group, cp, 0.0)
        for i, im in enumerate(group):
            d1, c1 = gpu_face.RunCascadeImages([im], cp, 0.0)
            assert cnt[i] == c1[0] and dets[i, :cnt[i]].tobytes() == d1[0, :c1[0]].tobytes(), f"image {i}"
