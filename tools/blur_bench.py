#!/usr/bin/env python
"""Face blur benchmark: prints one JSON line with the card's name and power limit and
  decoded_ms         : pigo_blur_decoded on tools/ragged_bench.py's 256 images as pinned 4:2:0 planes (luma = the image, seeded
                       chroma, as its decoded section builds them), end to end, host clock, median of 5
  detect_only_ms     : the same call's first three steps without the blur: pigo_gray_images, pigo_run_cascade_images_params,
                       pigo_cluster_batch, from the same pinned planes, host clock, median of 5
  blur_faces_ms      : pigo_blur_faces alone on device-resident copies of those planes with the faces the first call found,
                       CUDA events, median of 5
  crowd_4k_ms        : pigo_blur_faces on one 3840x2160 4:2:0 device image with 2,000 faces, CUDA events, median of 5
  numpy_cpu_s        : tests/blur_oracle.py's numpy restatement on the 256 images and their faces, on the CPU, one run
The planes are restored before every timed run.  Writes nothing to the tree."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)
from bench import PARAMS  # noqa: E402
from ragged_bench import ragged_images  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def main():
    import torch
    import blur_oracle as B
    import pigo_b200
    from pigo_b200 import DET_DTYPE, BlurParams, DecodedImage
    L = pigo_b200.lib()
    clf = pigo_b200.NewPigo().Unpack(pigo_b200.load_cascade("facefinder"))
    rng = np.random.default_rng(77)
    imgs = ragged_images()
    n = len(imgs)
    bp = BlurParams(5.0, 0.5, 0.0, 15)
    iou, det_cap, face_cap = 0.1, 4096, 4096

    def check(rc):
        if rc != 0:
            raise RuntimeError(L.pigo_last_error().decode())

    planes, keep = [], []
    for b, r, c, d in imgs:
        cw, ch = (c + 1) // 2, (r + 1) // 2
        y = torch.from_numpy(np.ascontiguousarray(b)).pin_memory()
        cb = torch.from_numpy((128 + rng.integers(-20, 21, size=(ch, cw + 3))).astype(np.uint8)).pin_memory()
        cr = torch.from_numpy((128 + rng.integers(-20, 21, size=(ch, cw + 3))).astype(np.uint8)).pin_memory()
        planes.append((y, cb, cr))
        keep.append((y.clone(), cb.clone(), cr.clone()))
    src = [DecodedImage.ycbcr(y, cb, cr, 2, c, r, y_stride=d, c_stride=cb.shape[1]) for (y, cb, cr), (_, r, c, d) in zip(planes, imgs)]
    descs = pigo_b200.decoded_descs(src)
    cps = pigo_b200.cascade_params_array([PARAMS] * n)

    def restore():
        for pl, k in zip(planes, keep):
            for a, b in zip(pl, k):
                a.copy_(b)

    faces = np.zeros((n, face_cap), dtype=DET_DTYPE)
    nf = np.zeros(n, dtype=np.int32)

    def blur_decoded():
        check(L.pigo_blur_decoded(clf._h, descs, n, cps, None, iou, det_cap, C.byref(bp), faces.ctypes.data, face_cap, nf.ctypes.data, 0, None))

    need = pigo_b200.gray_images_bytes(src)
    arena = torch.empty(need, dtype=torch.uint8, device="cuda")
    out_imgs = (pigo_b200.PigoImage * n)()
    size = C.c_size_t(need)
    raw = np.zeros((n, det_cap), dtype=DET_DTYPE)
    cnt = np.zeros(n, dtype=np.int32)
    cl = np.zeros((n, face_cap), dtype=DET_DTYPE)
    ncl = np.zeros(n, dtype=np.int32)

    def detect_only():
        check(L.pigo_gray_images(descs, n, arena.data_ptr(), C.byref(size), out_imgs, pigo_b200.MEM_HOST, None))
        check(L.pigo_run_cascade_images_params(clf._h, out_imgs, n, cps, None, raw.ctypes.data, det_cap, cnt.ctypes.data, pigo_b200.FRAMES_DEVICE, None))
        check(L.pigo_cluster_batch(raw.ctypes.data, cnt.ctypes.data, n, det_cap, iou, cl.ctypes.data, face_cap, ncl.ctypes.data, 0, None))

    def host_clock(fn):
        fn()
        ts = []
        for _ in range(5):
            restore()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        return round(1e3 * float(np.median(ts)), 3)

    res = {"card": card(), "images": n, "params": list(PARAMS), "blur": [5.0, 0.5, 0.0, 15]}
    res["decoded_ms"] = host_clock(blur_decoded)
    res["detect_only_ms"] = host_clock(detect_only)
    restore()
    blur_decoded()
    assert nf.tolist() == ncl.tolist() and all(faces[i, :nf[i]].tobytes() == cl[i, :ncl[i]].tobytes() for i in range(n))
    res["faces"] = int(nf.sum())
    blurred = [tuple(p.clone() for p in pl) for pl in planes]

    def events(fn, prep):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ms = []
        for _ in range(6):
            prep()
            torch.cuda.synchronize()
            ev[0].record()
            fn()
            ev[1].record()
            ev[1].synchronize()
            ms.append(ev[0].elapsed_time(ev[1]))
        return round(float(np.median(ms[1:])), 4)

    dev = [tuple(p.cuda() for p in k) for k in keep]
    dev_keep = [tuple(p.clone() for p in pl) for pl in dev]
    dsrc = pigo_b200.decoded_descs([DecodedImage.ycbcr(y, cb, cr, 2, c, r, y_stride=d, c_stride=cb.shape[1])
                                    for (y, cb, cr), (_, r, c, d) in zip(dev, imgs)])

    def restore_dev(pl=dev, k=dev_keep):
        for a, b in zip(pl, k):
            for x, y in zip(a, b):
                x.copy_(y)

    res["blur_faces_ms"] = events(lambda: check(L.pigo_blur_faces(dsrc, n, faces.ctypes.data, face_cap, nf.ctypes.data, C.byref(bp),
                                                                  pigo_b200.FRAMES_DEVICE, None)), restore_dev)
    assert all(torch.equal(a.cpu(), b) for pl, bl in zip(dev, blurred) for a, b in zip(pl, bl)), "blur_faces differs from blur_decoded"

    crowd = B.make_src(0, 3840, 2160, np.random.default_rng(11), sub=2, pad=8)
    cf = np.zeros((1, 2000), dtype=DET_DTYPE)
    cf["row"], cf["col"] = rng.integers(-20, 2180, (1, 2000)), rng.integers(-20, 3860, (1, 2000))
    cf["scale"], cf["q"] = rng.integers(20, 160, (1, 2000)), rng.uniform(4, 12, (1, 2000))
    cn = np.array([2000], dtype=np.int32)
    cdev = [torch.from_numpy(p).cuda() for p in crowd.planes]
    ckeep = [p.clone() for p in cdev]
    cdesc = pigo_b200.decoded_descs([crowd.decoded(cdev)])
    res["crowd_4k_ms"] = events(lambda: check(L.pigo_blur_faces(cdesc, 1, cf.ctypes.data, 2000, cn.ctypes.data, C.byref(bp), pigo_b200.FRAMES_DEVICE,
                                                                None)), lambda: restore_dev([cdev], [ckeep]))

    srcs = []
    for (y, cb, cr), (_, r, c, d) in zip(keep, imgs):
        srcs.append(B.BlurSrc(0, c, r, [y.numpy().reshape(-1), cb.numpy().reshape(-1), cr.numpy().reshape(-1)], (d, cb.shape[1]), 2))
    t0 = time.perf_counter()
    for i, s in enumerate(srcs):
        B.blur_np(s, faces[i, :nf[i]], 5.0, 0.5, 0.0, 15)
    res["numpy_cpu_s"] = round(time.perf_counter() - t0, 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
