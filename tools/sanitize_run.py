#!/usr/bin/env python
"""Exercises every kernel of libpigo_b200 on small inputs, for use under compute-sanitizer:

    compute-sanitizer --tool memcheck --error-exitcode 3 python tools/sanitize_run.py
    compute-sanitizer --tool racecheck --error-exitcode 3 python tools/sanitize_run.py --quick

No torch (ctypes mirror only), a few hundred thousand windows in total, so that the instrumented run ends in minutes.
Covers: fused kernel (tile + gather role, aligned TMA fill and byte-wise fill), gather-v2, deep kernel with Q2,
queue-overflow fallbacks (tiny KS, tail policy on), universal gather kernel (rotated, scan_mode=1), finalize, cluster,
RunDetector / landmark kernels over resident frames, grayscale, and the mixed-size pipeline and RunDetector (image-table
kernel variants; --images runs only those), and the per-image angle calls (--angles runs only those).  Prints the detection counts (compare with a plain run).
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pigo_b200  # noqa: E402
from pigo_b200 import CascadeParams, ImageParams, pipeline, synth  # noqa: E402

PRM = (20, 1000, 0.2, 1.1)


def cp_of(img, rows, cols, dim, prm=PRM):
    return CascadeParams(ImageParams(img, rows, cols, dim), *prm)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="scan kernels only, fewer variants (racecheck is slow)")
    ap.add_argument("--new", action="store_true", help="only the kernels added late in round 2 (offset tables, shared-memory deep, queue overflow)")
    ap.add_argument("--images", action="store_true", help="only the mixed-size pipeline and RunDetector (image-table kernel variants)")
    ap.add_argument("--angles", action="store_true", help="only the per-image angle calls (several node tables, unrotated and rotated passes)")
    ap.add_argument("--decoded", action="store_true", help="only pigo_gray_images (every decoded format, host and device planes)")
    args = ap.parse_args()
    pigo_b200.init(0)
    clf = pigo_b200.NewPigo().Unpack(pigo_b200.load_cascade("facefinder"))
    sample = synth.sample_gray()
    counts = []
    if args.decoded:
        counts += decoded_case()
        print("sanitize_run counts:", counts, "launches:", pigo_b200.launch_count())
        return
    if args.images or args.angles:
        counts += angles_case(clf, sample) if args.angles else images_case(clf, sample)
        print("sanitize_run counts:", counts, "launches:", pigo_b200.launch_count())
        return

    variants = [{}, {"tile_warps": 4, "tile_ks": 5, "gather_ks": 7, "tile_tail_min": 33},
                {"scan_mode": 3, "gather_ks": 4}, {"scan_mode": 1}, {"tile_ni": 2, "tile_warps": 8, "gather_warps": 0, "tile_prefetch": 1},
                {"tile_head": 2, "tile_warps": 22}, {"tile_head": 1, "tile_warps": 6, "tile_ks": 5, "tile_tail_min": 33},
                {"host_stream": 1, "copy_chunk": 1, "sub_batch": 1, "deep_flat": 1}, {"host_stream": 0}, {"walk_stats": 1}]
    late = [{"tile_ptab": 1}, {"tile_ptab": 1, "ptab_kt": 4, "ptab_ks": 6, "tile_warps": 7, "gather_warps": 3, "tile_tail_min": 33},
            {"deep_smem": 1, "deep_smem_k": 468, "deep_smem_lo": 0}, {"deep_smem": 1, "deep_group": 4, "gather_limit": 4, "tile_ks": 6, "deep_smem_k": 30, "deep_smem_lo": 11},
            {"queue_cap": 9, "tile_ks": 4, "gather_ks": 6, "tile_tail_min": 33}, {"queue_cap": 7, "tile_ptab": 1, "ptab_kt": 3, "ptab_ks": 5, "tile_tail_min": 33}]
    variants = late if args.new else variants + late
    if args.quick:
        variants = variants[:2]
    keys = sorted({k for v in variants for k in v})
    saved = {k: pigo_b200.get_option(k) for k in keys}
    frames = np.stack([synth.frame_faces(sample, 360, 640, shift=(20 * i, 10 * i), noise_seed=3 + i) for i in range(2)])
    odd = np.zeros((203, 331), dtype=np.uint8)
    odd[:, :320] = synth.frame_faces(None, 203, 320, shift=(3, 1), noise_seed=8)
    for v in variants:
        for k, val in saved.items():
            pigo_b200.set_option(k, val)
        for k, val in v.items():
            pigo_b200.set_option(k, val)
        counts.append(len(clf.run_cascade_array(cp_of(sample, 400, 320, 320), 0.0)))
        counts.append(len(clf.run_cascade_array(cp_of(odd, 203, 320, 331), 0.0)))       # Dim % 16 != 0: byte-wise tile fill
        dets, cnt = clf.RunCascadeBatch(frames, cp_of(None, 360, 640, 640), 0.0, cap_per_frame=256)
        counts += [int(c) for c in cnt]
    for k, val in saved.items():
        pigo_b200.set_option(k, val)
    for a in (0.3, 0.97):                                                                # rotated: table-driven block + deep kernels
        counts.append(len(clf.run_cascade_array(cp_of(sample, 400, 320, 320), a)))
        dets, cnt = clf.RunCascadeBatch(frames, cp_of(None, 360, 640, 640), a, cap_per_frame=256)
        counts += [int(c) for c in cnt]
    pigo_b200.set_option("rot_mode", 1)                                                  # rotated: universal gather kernel
    counts.append(len(clf.run_cascade_array(cp_of(sample, 400, 320, 320), 0.3)))
    pigo_b200.set_option("rot_mode", 0)

    if not args.quick:
        dets = clf.RunCascade(cp_of(sample, 400, 320, 320), 0.0)
        counts.append(len(clf.ClusterDetections(dets, 0.1)))
        plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
        names = sorted(set(pipeline.EYE_CASCADES + pipeline.MOUTH_CASCADES))
        flp = {n: pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("lps/" + n)) for n in names}
        faces = pipeline.detect_batch(clf, plc, flp, frames, cp_of(None, 360, 640, 640), iou=0.1)
        counts.append(sum(len(f) for f in faces))
        counts.append(sum(1 for f in faces for fc in f if fc.landmarks))
        rgba = np.random.default_rng(0).integers(0, 256, size=(37, 53, 4), dtype=np.uint8)
        counts.append(int(pigo_b200.RgbToGrayscale(rgba).sum()))
        # device-sequenced pipeline (seed kernels + pair kernel, staged and unstaged, rotated eyes), sharded entry point
        for stage, ang in ((1, 0.0), (0, 0.0), (1, 0.05)):
            pigo_b200.set_option("puploc_stage", stage)
            f, n, p = pipeline.detect_batch_device(clf, plc, flp, frames, cp_of(None, 360, 640, 640), face_cap=16, rng_seed=3, angle=ang, raw=True)
            counts += [int(n.sum()), int((p["row"] > 0).sum())]
        pigo_b200.set_option("puploc_stage", 1)
        pigo_b200.init_devices(1)
        f, n, p = pipeline.detect_batch_device(clf, plc, flp, frames, cp_of(None, 360, 640, 640), face_cap=16, rng_seed=3, raw=True, sharded=True)
        counts.append(int(n.sum()))
        pigo_b200.set_option("puploc_mode", 1)
        faces2 = pipeline.detect_batch(clf, plc, flp, frames[:1], cp_of(None, 360, 640, 640), iou=0.1)
        counts.append(sum(len(x) for x in faces2))
        pigo_b200.set_option("puploc_mode", 0)
        yy = np.random.default_rng(1).integers(0, 256, size=(21, 40), dtype=np.uint8)
        cb = np.random.default_rng(2).integers(0, 256, size=(11, 20), dtype=np.uint8)
        cr = np.random.default_rng(3).integers(0, 256, size=(11, 20), dtype=np.uint8)
        out, gy = pigo_b200.YCbCrToNRGBA(yy, cb, cr, 2, 37, 21, want_gray=True)
        counts += [int(out.sum()), int(gy.sum())]
        counts += images_case(clf, sample)
        counts += angles_case(clf, sample)
        counts += decoded_case()
    print("sanitize_run counts:", counts, "launches:", pigo_b200.launch_count() if hasattr(pigo_b200, "launch_count") else "n/a")


def images_case(clf, sample):
    """pigo_detect_images over images of three geometries (one with Dim % 16 != 0: the patch falls back to global gathers),
    every puploc_stage; pigo_puploc_run_images with seeds on and past the borders on both RunDetector kernels."""
    counts = []
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
    names = sorted(set(pipeline.EYE_CASCADES + pipeline.MOUTH_CASCADES))
    flp = {n: pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("lps/" + n)) for n in names}
    wide = np.zeros((300, 712), dtype=np.uint8)
    wide[:, :700] = synth.frame_faces(sample, 300, 700, noise_seed=2)
    images = [ImageParams(sample, 400, 320, 320), ImageParams(wide, 300, 700, 712),
              ImageParams(synth.frame_faces(sample, 540, 960, shift=(30, 200), noise_seed=4), 540, 960, 960), ImageParams(np.zeros(64, np.uint8), 8, 8, 8)]
    cp = CascadeParams(ImageParams(), *PRM)
    for stage, ang in ((2, 0.0), (1, 0.05), (0, 0.0)):
        pigo_b200.set_option("puploc_stage", stage)
        f, n, p = pipeline.detect_images_device(clf, plc, flp, images, cp, face_cap=8, rng_seed=3, angle=ang, raw=True)
        counts += [int(n.sum()), int((p["row"] > 0).sum())]
    pigo_b200.set_option("puploc_stage", 1)
    rng = np.random.default_rng(5)
    seeds = [pigo_b200.Puploc(int(rng.integers(-30, 560)), int(rng.integers(-30, 980)), float(rng.uniform(4, 200)), int(rng.integers(0, 64)))
             for _ in range(24)]
    which = [k % 3 for k in range(24)]
    for mode in (0, 1):
        pigo_b200.set_option("puploc_mode", mode)
        out = plc.run_detector_images(seeds, which, images[:3], 0.2, [k % 2 == 0 for k in range(24)], rng_seed=9)
        counts.append(sum(o.Row for o in out))
    pigo_b200.set_option("puploc_mode", 0)
    return counts


def angles_case(clf, sample):
    """pigo_run_cascade_images_angles on two wide images and the sample, each listed at several angles (repeated host
    descriptors, unrotated and rotated passes, one node table per slot), and pigo_detect_images_angles (per-image eye slots)."""
    counts = []
    wide = np.zeros((300, 712), dtype=np.uint8)
    wide[:, :700] = synth.frame_faces(sample, 300, 700, noise_seed=2)
    base = [ImageParams(sample, 400, 320, 320), ImageParams(wide, 300, 700, 712), ImageParams(np.zeros(64, np.uint8), 8, 8, 8)]
    angles = [0.0, 0.05, 0.3, 1.0]
    ims = [im for im in base for _ in angles]
    ang = [0.0 if im.Cols < im.Rows else a for im in base for a in angles]   # tall images unrotated (the rotated column clamp)
    cp = CascadeParams(ImageParams(), *PRM)
    dets, cnt = clf.RunCascadeImagesAngles(ims, cp, ang, 256)
    counts += [int(c) for c in cnt]
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
    names = sorted(set(pipeline.EYE_CASCADES + pipeline.MOUTH_CASCADES))
    flp = {n: pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("lps/" + n)) for n in names}
    for stage in (2, 1):
        pigo_b200.set_option("puploc_stage", stage)
        f, n, p = pipeline.detect_images_angles_device(clf, plc, flp, ims, cp, ang, face_cap=8, rng_seed=3, raw=True)
        counts += [int(n.sum()), int((p["row"] > 0).sum())]
    pigo_b200.set_option("puploc_stage", 1)
    return counts


def decoded_case():
    """pigo_gray_images over every decoded format (odd sizes and origins, padded strides, 16-byte aligned and unaligned rows,
    a short palette, one repeated source) from host planes into a device arena, and again from device planes."""
    import ctypes as C
    rng = np.random.default_rng(6)
    y, cb, cr = (rng.integers(0, 256, size=(21, 43), dtype=np.uint8) for _ in range(3))
    px = rng.integers(0, 256, size=(9, 40 * 4 + 4), dtype=np.uint8)
    g = rng.integers(0, 256, size=(5, 35), dtype=np.uint8)
    src = [pigo_b200.DecodedImage.ycbcr(y, cb, cr, sub, 37, 20, min_x=1, min_y=1) for sub in range(6)]
    src += [pigo_b200.DecodedImage.nrgba(px, 40, 9), pigo_b200.DecodedImage.rgba(px, 33, 9), pigo_b200.DecodedImage.gray(g, 32, 5),
            pigo_b200.DecodedImage.gray(g, 35, 5), pigo_b200.DecodedImage.gray(g, 1, 1)]
    pal = rng.integers(0, 256, size=(7, 4), dtype=np.uint8)   # indices past it give 0
    flat = px.reshape(-1)
    src += [pigo_b200.DecodedImage.gray16(px, 82, 9), pigo_b200.DecodedImage.gray16(flat[3:], 75, 9, stride=164),
            pigo_b200.DecodedImage.rgba64(px, 20, 9), pigo_b200.DecodedImage.nrgba64(flat[5:], 19, 9, stride=164),
            pigo_b200.DecodedImage.cmyk(px, 40, 9), pigo_b200.DecodedImage.paletted(g, pal, 35, 5)]
    src.append(src[2])
    need = pigo_b200.gray_images_bytes(src)
    L = pigo_b200.lib()
    counts = []
    for flags in (pigo_b200.MEM_HOST, pigo_b200.FRAMES_DEVICE):
        gray = C.c_void_p()
        pigo_b200._check(L.pigo_device_alloc(C.byref(gray), need))
        bufs = []
        cur = src
        if flags == pigo_b200.FRAMES_DEVICE:   # the same planes uploaded with pigo_device_upload
            cur, seen = [], {}
            for s in src:
                if id(s) in seen:   # a repeated source stays byte-identical
                    cur.append(seen[id(s)])
                    continue
                pl = []
                for p in s.planes:
                    d = C.c_void_p()
                    pigo_b200._check(L.pigo_device_alloc(C.byref(d), p.nbytes))
                    pigo_b200._check(L.pigo_device_upload(d, p.ctypes.data, p.nbytes))
                    bufs.append(d.value)
                    pl.append(d.value)
                seen[id(s)] = pigo_b200.DecodedImage(s.format, s.width, s.height, tuple(pl), s.strides, s.subsample, s.min_x, s.min_y)
                cur.append(seen[id(s)])
        imgs = (pigo_b200.PigoImage * len(cur))()
        size = C.c_size_t(need)
        pigo_b200._check(L.pigo_gray_images(pigo_b200.decoded_descs(cur), len(cur), gray.value, C.byref(size), imgs, flags, None))
        out = np.zeros(need, dtype=np.uint8)
        pigo_b200._check(L.pigo_device_download(out.ctypes.data, gray.value, need))
        counts.append(int(out.astype(np.int64).sum()))
        for b in bufs:
            L.pigo_device_free(b)
        L.pigo_device_free(gray.value)
    return counts


if __name__ == "__main__":
    main()
