#!/usr/bin/env python
"""Line-touch model of the deep kernel's loads (CPU only, numpy oracle; needs no GPU and measures no time).

The deep kernel walks one window per group of 8 lanes, trees t0 .. t0+7 of it per step, one tree per lane.  An L1 load
instruction costs a tag look-up per distinct 128-byte line its lanes touch, so this counts, per 8-lane group step, the
distinct lines of each load instruction summed over the step's loads:
  cascade   1 threshold + 1 root word + 6 child-pair loads (the last one the leaf pair), in two layouts:
            reference  codes[t][256 B], preds[t][256 B], thresh[t]   (what the deep walk read before)
            blocks     the block-interleaved copy of common.cuh (kBlockBytes): 8 trees per 4096-byte block
  pixels    12 one-byte gathers (two per level)
The windows are those of bench.py's batch (configs[2], 1080p, its frame generator) that reach the deep queue, approximated:
tile-role scales (< 55) alive at tree 48, gather-role scales alive at tree 16, plus one in --straggler-every tile-role windows
alive at a random tree in [1, 48) (the drained tiles' stragglers, which start at any tree).  Each is replayed to the step in
which the reference rejects it.

Usage: python tools/deep_lines.py [--frames 3] [--seed 0] ; prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.np_oracle import FaceCascade, grid, scale_ladder  # noqa: E402

ROWS, COLS = 1080, 1920
PARAMS = (20, 1000, 0.2, 1.1)
GATHER_MIN_SCALE, TILE_KS, GATHER_LIMIT, GROUP = 55, 48, 16, 8


def bench_frames(n: int, seed0: int) -> np.ndarray:
    """bench.py's make_frames for the first n frames (n <= 24: base frames only)."""
    from pigo_b200 import synth
    return synth.make_batch(n, ROWS, COLS, "USF", seed0=seed0)


def distinct(a: np.ndarray) -> np.ndarray:
    """Distinct values per row of a [n, GROUP] array."""
    s = np.sort(a, axis=1)
    return 1 + (np.diff(s, axis=1) != 0).sum(axis=1)


def walk(cas: FaceCascade, t: np.ndarray, pos: np.ndarray, s: np.ndarray, flat: np.ndarray):
    """Walks trees t (any shape) at window centre pos (flat pixel index) and size s: leaf value, the node index at each of
    the 6 levels (the node whose children the level loads) and the 12 pixel addresses."""
    idx = np.ones(t.shape, dtype=np.int64)
    nodes, pix = [], []
    for _ in range(cas.depth):
        nodes.append(idx)
        cd = cas.codes[t, idx].astype(np.int64)
        x1 = pos + ((cd[..., 0] * s) >> 8) * COLS + ((cd[..., 1] * s) >> 8)
        x2 = pos + ((cd[..., 2] * s) >> 8) * COLS + ((cd[..., 3] * s) >> 8)
        pix += [x1, x2]
        idx = 2 * idx + (flat[x1] <= flat[x2])
    return cas.preds[t, idx - cas.leaves], nodes, pix


def lines_per_step(t: np.ndarray, nodes, pix, frame_base: int):
    """Summed distinct lines over the step's load instructions, per group step ([n, GROUP] inputs)."""
    ref = distinct((4 * t) >> 7)                                        # thresh[t] (own allocation, 128-aligned)
    ref += distinct((256 * t + 4) >> 7)                                  # root word, codes[t][4]
    blk = distinct((4096 * (t >> 3) + 4 * (t & 7)) >> 7)
    blk += distinct((4096 * (t >> 3) + 32 + 4 * (t & 7)) >> 7)
    for j, idx in enumerate(nodes):
        if j < 5:
            ref += distinct((256 * t + 8 * idx) >> 7)                    # codes[t][8 idx ..]
        else:
            ref += distinct((256 * t + 8 * (idx - 32)) >> 7)             # preds[t][2 idx - 64 ..]
        blk += distinct((4096 * (t >> 3) + 64 * idx + 8 * (t & 7)) >> 7)
    px = sum(distinct((frame_base + x) >> 7) for x in pix)
    return ref, blk, px


def deep_items(cas: FaceCascade, flat: np.ndarray, rng: np.random.Generator, straggler_every: int):
    """(pos, s, start tree, partial sum) of the windows of one frame that reach the deep queue (see the module doc)."""
    items = []
    for s in scale_ladder(PARAMS[0], PARAMS[1], PARAMS[3]):
        rr, cc = grid(ROWS, COLS, s, PARAMS[2])
        if len(rr) == 0 or len(cc) == 0:
            continue
        R, C = np.meshgrid(rr, cc, indexing="ij")
        pos = (R * COLS + C).ravel()
        n = pos.size
        tile = s < GATHER_MIN_SCALE
        limit = TILE_KS if tile else GATHER_LIMIT
        strag_at = np.full(n, -1)
        if tile:
            pick = rng.random(n) < 1.0 / straggler_every
            strag_at[pick] = rng.integers(1, TILE_KS, pick.sum())
        acc = np.zeros(n, dtype=np.float32)
        alive = np.arange(n)
        for t in range(limit):
            if alive.size == 0:
                break
            hit = alive[strag_at[alive] == t]
            items += [(pos[hit], np.full(hit.size, s), np.full(hit.size, t), acc[hit])]
            alive = alive[strag_at[alive] != t]
            leaf, _, _ = walk(cas, np.full(alive.size, t), pos[alive], s, flat)
            acc[alive] = acc[alive] + leaf
            alive = alive[acc[alive] > cas.thresh[t]]
        items += [(pos[alive], np.full(alive.size, s), np.full(alive.size, limit), acc[alive])]
    return [np.concatenate(a) for a in zip(*items)]


def replay(cas: FaceCascade, flat: np.ndarray, pos, s, t0, acc, frame_base: int):
    """Group steps of every item until the reference rejects it: summed line counts and the number of steps."""
    tot = np.zeros(3, dtype=np.int64)
    steps = 0
    sub = np.arange(GROUP)
    while pos.size:
        t = np.minimum(t0[:, None] + sub[None, :], cas.ntrees - 1)
        leaf, nodes, pix = walk(cas, t, pos[:, None], s[:, None], flat)
        for k, v in enumerate(lines_per_step(t, nodes, pix, frame_base)):
            tot[k] += int(v.sum())
        steps += pos.size
        live = np.ones(pos.size, dtype=bool)
        nvalid = np.minimum(GROUP, cas.ntrees - t0)
        for j in range(GROUP):                                           # the sequential accumulation, tree order
            on = live & (j < nvalid)
            acc = np.where(on, acc + leaf[:, j], acc)
            live &= ~(on & (acc <= cas.thresh[t[:, j]]))
        t0 = t0 + GROUP
        keep = live & (t0 < cas.ntrees)
        pos, s, t0, acc = pos[keep], s[keep], t0[keep], acc[keep]
    return tot, steps


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--frames", type=int, default=3, help="bench.py base frames to model (one of each class U/S/F)")
    ap.add_argument("--seed", type=int, default=0, help="bench.py's seed0 (rank 0: 0)")
    ap.add_argument("--straggler-every", type=int, default=64, help="one in N tile-role windows becomes a straggler sample")
    args = ap.parse_args()
    import pigo_b200
    cas = FaceCascade(pigo_b200.load_cascade("facefinder"))
    frames = bench_frames(args.frames, args.seed)
    rng = np.random.default_rng(12345)
    tot, steps, nitems, per_frame = np.zeros(3, dtype=np.int64), 0, 0, []
    for f in range(args.frames):
        flat = frames[f].reshape(-1)
        pos, s, t0, acc = deep_items(cas, flat, rng, args.straggler_every)
        base = f * ROWS * COLS
        ft, fs = replay(cas, flat, pos, s, t0, acc, base)
        per_frame.append({"items": int(pos.size), "group_steps": fs,
                          "cascade_reference": round(ft[0] / max(fs, 1), 2), "cascade_blocks": round(ft[1] / max(fs, 1), 2),
                          "pixels": round(ft[2] / max(fs, 1), 2)})
        tot += ft
        steps += fs
        nitems += pos.size
    ref, blk, px = (tot / max(steps, 1)).tolist()
    print(json.dumps({
        "metric": "distinct 128-byte lines per 8-lane group step, summed over its load instructions (model, not measured)",
        "frames": args.frames, "items": nitems, "group_steps": steps,
        "cascade_reference": round(ref, 2), "cascade_blocks": round(blk, 2), "pixels": round(px, 2),
        "total_reference": round(ref + px, 2), "total_blocks": round(blk + px, 2),
        "line_touches_saved": round(1 - (blk + px) / (ref + px), 3), "per_frame": per_frame}))


if __name__ == "__main__":
    main()
