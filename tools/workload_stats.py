#!/usr/bin/env python
"""Workload statistics of the scan (CPU only, numpy restatement of classifyRegion): for one 1080p frame of each synthetic
content class (pigo_b200/synth.py: U noise, S smooth + faces, F faces on noise) and the reference's test parameters, how
many trees each window evaluates before it is rejected, per scale.  These numbers are what the kernel schedule is built on
(which share of the tree walks happens in the tile warps, in the gather role, in Q2/deep) -- see DESIGN.md section 7.

    python tools/workload_stats.py > profiles/workload_stats_r01.md
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import np_oracle as NP  # noqa: E402  (test infrastructure: this tool only measures the workload)
from pigo_b200 import synth  # noqa: E402

ROWS, COLS = 1080, 1920
PRM = (20, 1000, 0.2, 1.1)
KS = 48          # trees resident in the fused kernel (tile_ks)
FIRST_GATHER = 60  # smallest scale scanned by the gather role with the default options


def main():
    pk = open(os.path.join(ROOT, "pigo_b200", "data", "cascade", "facefinder"), "rb").read()
    face = NP.FaceCascade(pk)
    print("# Scan workload statistics (numpy restatement, one 1080p frame per class, MinSize 20 MaxSize 1000 Shift 0.2 Scale 1.1)\n")
    print("`walks` = tree walks (one window evaluating one tree); `>=K` = share of the class's walks that happen at tree index >= K.\n")
    for cls in "USF":
        img = synth.make_batch(1, ROWS, COLS, cls)[0]
        rows_out = []
        tot_w = tot_walks = 0
        walks_ge = {16: 0, 32: 0, KS: 0, 128: 0}
        surv = {1: 0, 2: 0, 4: 0, 16: 0, KS: 0, 467: 0}
        q2_by_band = {"tile (s<60)": [0, 0], "gather (s>=60)": [0, 0]}
        for s in NP.scale_ladder(PRM[0], PRM[1], PRM[3]):
            rr, cc = NP.grid(ROWS, COLS, s, PRM[2])
            if len(rr) == 0 or len(cc) == 0:
                continue
            R, C = np.meshgrid(rr, cc, indexing="ij")
            _, nt = face.classify(R.ravel(), C.ravel(), s, img, ROWS, COLS, COLS, 0.0, return_ntrees=True)
            n, walks = nt.size, int(nt.sum())
            tot_w += n
            tot_walks += walks
            for k in walks_ge:
                walks_ge[k] += int(np.maximum(nt - k, 0).sum())
            for k in surv:
                surv[k] += int((nt > k).sum())
            band = "tile (s<60)" if s < FIRST_GATHER else "gather (s>=60)"
            q2_by_band[band][0] += int((nt > KS).sum())
            q2_by_band[band][1] += int(np.maximum(nt - KS, 0).sum())
            rows_out.append((s, n, walks, walks / n, int((nt > KS).sum()), int(np.maximum(nt - KS, 0).sum())))
        print(f"## class {cls}: {tot_w} windows, {tot_walks} walks, {tot_walks / tot_w:.2f} walks/window\n")
        print("| survive more than k trees | " + " | ".join(f"k={k}" for k in surv) + " |")
        print("|---|" + "---|" * len(surv))
        print("| share of windows | " + " | ".join(f"{100.0 * v / tot_w:.3f} %" for v in surv.values()) + " |\n")
        print("| walks at tree index | " + " | ".join(f">={k}" for k in walks_ge) + " |")
        print("|---|" + "---|" * len(walks_ge))
        print("| share of walks | " + " | ".join(f"{100.0 * v / tot_walks:.1f} %" for v in walks_ge.values()) + " |\n")
        print(f"Windows handed to Q2 (alive after tree {KS}) and their remaining walks, by producer:\n")
        for band, (nw, wk) in q2_by_band.items():
            print(f"* {band}: {nw} windows, {wk} walks ({100.0 * wk / tot_walks:.1f} % of all walks)")
        print("\n| scale | windows | walks | walks/window | alive after tree 48 | walks past tree 48 |")
        print("|---|---|---|---|---|---|")
        for s, n, walks, avg, a48, w48 in rows_out:
            if s <= 124 or a48 > 0:
                print(f"| {s} | {n} | {walks} | {avg:.2f} | {a48} | {w48} |")
        print()


if __name__ == "__main__":
    main()
