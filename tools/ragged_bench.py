#!/usr/bin/env python
"""Mixed-size images benchmark: pigo_run_cascade_images against the ways a caller without it would scan the same images.

Usage: `python tools/ragged_bench.py [--frames 256]` on one GPU prints one JSON line:
  one_images_call / batch_call_per_geometry / call_per_image : 256 seeded images of mixed sizes, device resident, CUDA
              events; the three outputs are asserted identical
  one_images_call_e2e_host : the mixed call from pageable host images, wall clock
  uniform_1080p : the mixed call on --frames identical-geometry 1080p frames (bench.py's batch) against pigo_run_cascade_batch
              with the default schedule and with scan_mode=3 (the gather-v2 + deep pair the mixed call runs), alternated
  pipeline : face -> cluster -> pupils -> 15 landmarks on the same 256 images: one pigo_detect_images call against one
              pigo_detect_batch per geometry and one per image (device resident, CUDA events; faces and counts asserted
              identical, points compared in an untimed run with injected randoms), and pigo_detect_images against
              pigo_detect_batch on --pipeline-frames uniform 1080p frames, alternated
  angles : angle sweeps, one per-image-angle call against one call per angle (device resident, CUDA events, outputs
              asserted identical): (1) one 1080p frame at 0 and k/32 (k = 1..32) against 33 single-frame calls; (2) bench.py's
              configs[3] batch, 8 x 4K frames at the 32 rotated slots, against 32 batch calls; (3) 16 wide images x 8 angles
              through the pipeline, listed image-major and angle-major, against 8 pigo_detect_images calls
  decoded : the same 256 images as 4:2:0 YCbCr (luma = the image, seeded chroma) in pinned host memory through face -> pupils
              -> 15 landmarks, host clock around each whole way, median of 5, outputs asserted identical: (a) one
              pigo_gray_images + one pigo_detect_images on the device images; (b) per image pigo_ycbcr_to_nrgba (gray only)
              to the host, then one pigo_detect_images from host gray; (c) per image pigo_ycbcr_to_nrgba (NRGBA) +
              pigo_rgba_to_gray, then one pigo_detect_images.  Also pigo_gray_images alone from device-resident planes
              (CUDA events) and from pinned host planes (host clock).
  formats : the same 256 images as NRGBA, Gray16, RGBA64, NRGBA64, CMYK and Paletted sources whose gray is exactly the
              image, detections asserted equal: pigo_gray_images alone (device and pinned planes) and with
              pigo_detect_images end to end (formats_bench)
  sharded : the same 256 images (a quarter of the wide ones rotated) from host memory: one single-device call against the
              sharded calls with shard_split 1, 2, 4, 8, outputs asserted identical; per-shard modelled cost against
              measured time (sharded_bench)
  sweep   : one 1080p frame and 16 wide images of the mix, each x 32 angles: one pigo_detect_images_sweep against
              pigo_detect_images_angles over the expanded list plus a merge through host memory; the merge kernels' own time
              (sweep_bench)
`--sections scan,pipeline` (the default) selects the sections; `--sections angles` runs the sweeps alone.  Writes nothing
to the tree.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
from bench import COLS, PARAMS, ROWS, make_frames  # noqa: E402  (the headline batch's frames and parameters)


# Mixed-size workload: common sizes from 320x240 to 3840x2160 (weighted towards photos and HD) and
# odd sizes with Dim > Cols, what a detector serving uploaded photos, thumbnails and several cameras is fed.
RAGGED_COMMON = [(240, 320), (360, 640), (480, 640), (540, 960), (600, 800), (720, 1280), (768, 1024), (1080, 1440), (1080, 1920),
                 (1200, 1600), (1536, 2048), (2160, 3840)]


def ragged_images(n: int = 256, seed: int = 2024):
    """Seeded mix of n images, (pixels [rows][dim], rows, cols, dim): 60 % common sizes, 40 % odd sizes with 1..63 bytes of
    row padding; content classes F and S alternate, cut at random offsets from one 4K frame of each class."""
    from pigo_b200 import synth
    rng = np.random.default_rng(seed)
    base = {"F": synth.frame_faces(None, 2160, 3840, noise_seed=seed), "S": synth.frame_smooth(2160, 3840, seed)}
    out = []
    for i in range(n):
        if rng.random() < 0.6:
            r, c = RAGGED_COMMON[int(rng.integers(len(RAGGED_COMMON)))]
            d = c
        else:
            r, c = int(rng.integers(48, 1600)), int(rng.integers(48, 2400))
            d = c + int(rng.integers(1, 64))
        r0, c0 = int(rng.integers(0, 2160 - r + 1)), int(rng.integers(0, 3840 - c + 1))
        buf = np.zeros((r, d), dtype=np.uint8)
        buf[:, :c] = base["FS"[i % 2]][r0:r0 + r, c0:c0 + c]
        out.append((buf, r, c, d))
    return out


def ragged_bench(clf, dev: int, stream, d_frames, nf: int) -> dict:
    """One pigo_run_cascade_images call on a mixed-size batch against one pigo_run_cascade_batch per
    distinct geometry and one call per image (all device resident, CUDA events, outputs asserted identical), the mixed call
    end to end from host images, and the mixed call on the uniform 1080p batch against the batch call (default schedule and
    scan_mode=3, the gather-v2 + deep pair the mixed call runs)."""
    import torch
    import pigo_b200
    L = pigo_b200.lib()
    st = stream.cuda_stream
    cap = 4096
    imgs = ragged_images()
    n = len(imgs)
    wins = [pigo_b200.count_windows(r, c, *PARAMS) for _, r, c, _ in imgs]
    W = int(sum(wins))
    offs, total = [], 0
    for b, r, c, d in imgs:
        offs.append(total)
        total += (r * d + 255) & ~255
    host = np.zeros(total, dtype=np.uint8)
    for (b, r, c, d), o in zip(imgs, offs):
        host[o:o + r * d] = b.reshape(-1)
    dev_all = torch.from_numpy(host).to(f"cuda:{dev}")
    base = dev_all.data_ptr()
    descs = [(base + o, r, c, d) for (b, r, c, d), o in zip(imgs, offs)]
    geo = {}
    for i, (_, r, c, d) in enumerate(imgs):
        geo.setdefault((r, c, d), []).append(i)
    # (b): every geometry's images contiguous, frame_stride = rows*dim
    geo_frames = {g: torch.stack([dev_all[offs[i]:offs[i] + g[0] * g[2]] for i in idx]) for g, idx in geo.items()}
    out = {k: torch.zeros((n, cap, 4), dtype=torch.int32, device=f"cuda:{dev}") for k in "abc"}
    cnt = {k: torch.zeros(n, dtype=torch.int32, device=f"cuda:{dev}") for k in "abc"}
    geo_out = {g: (torch.zeros((len(idx), cap, 4), dtype=torch.int32, device=f"cuda:{dev}"),
                   torch.zeros(len(idx), dtype=torch.int32, device=f"cuda:{dev}")) for g, idx in geo.items()}

    def run_a():
        clf.run_cascade_images_device(descs, *PARAMS, 0.0, out["a"].data_ptr(), cap, cnt["a"].data_ptr(), st)

    def run_b():
        for (r, c, d), fr in geo_frames.items():
            o, k = geo_out[(r, c, d)]
            clf.run_cascade_batch_device(fr.data_ptr(), fr.shape[0], r * d, r, c, d, *PARAMS, 0.0, o.data_ptr(), cap, k.data_ptr(), st)

    def run_c():
        for i, (p, r, c, d) in enumerate(descs):
            clf.run_cascade_batch_device(p, 1, r * d, r, c, d, *PARAMS, 0.0, out["c"][i].data_ptr(), cap, cnt["c"].data_ptr() + 4 * i, st)

    def timed(fn, reps=5, warm=2):
        for _ in range(warm):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            fn()
            b.record(stream)
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return float(np.median(ts))

    ms = {k: timed(f) for k, f in (("a", run_a), ("b", run_b), ("c", run_c))}
    for (g, idx) in geo.items():
        o, k = geo_out[g]
        out["b"][idx] = o
        cnt["b"][idx] = k
    counts = {k: cnt[k].cpu().numpy() for k in "abc"}
    assert int(counts["a"].max()) <= cap, "raise cap: an image has more detections than the bench buffer"
    dets = {k: out[k].cpu().numpy() for k in "abc"}
    for k in "bc":
        assert np.array_equal(counts["a"], counts[k]), f"ragged: counts of ({k}) differ from the mixed call"
        for i in range(n):
            assert dets["a"][i, :counts["a"][i]].tobytes() == dets[k][i, :counts["a"][i]].tobytes(), f"ragged: image {i} of ({k}) differs"
    # (a) end to end: pageable host images in, detections out
    hdesc = pigo_b200.image_descs([(b.ctypes.data, r, c, d) for b, r, c, d in imgs])
    out_h = np.zeros((n, cap), dtype=pigo_b200.DET_DTYPE)
    cnt_h = np.zeros(n, dtype=np.int32)

    def run_host():
        rc = L.pigo_run_cascade_images(clf._h, hdesc, n, *PARAMS, 0.0, out_h.ctypes.data, cap, cnt_h.ctypes.data, 0, None)
        if rc != 0:
            raise RuntimeError(L.pigo_last_error().decode())
    run_host()
    hts = []
    for _ in range(3):
        t0 = time.perf_counter()
        run_host()
        hts.append((time.perf_counter() - t0) * 1e3)
    assert np.array_equal(cnt_h, counts["a"])
    ms_host = float(np.median(hts))

    # uniform batch: the bench's 1080p frames through the mixed call, the batch call and the batch call with scan_mode=3,
    # alternated in rounds so that drift hits the three alike
    Wf = pigo_b200.count_windows(ROWS, COLS, *PARAMS)
    ucap = 1024
    uo = {k: torch.zeros((nf, ucap, 4), dtype=torch.int32, device=f"cuda:{dev}") for k in ("images", "batch", "batch_scan_mode3")}
    uc = {k: torch.zeros(nf, dtype=torch.int32, device=f"cuda:{dev}") for k in uo}
    udesc = [(d_frames[i].data_ptr(), ROWS, COLS, COLS) for i in range(nf)]
    mode0 = pigo_b200.get_option("scan_mode")

    def u_run(k):
        if k == "images":
            clf.run_cascade_images_device(udesc, *PARAMS, 0.0, uo[k].data_ptr(), ucap, uc[k].data_ptr(), st)
            return
        pigo_b200.set_option("scan_mode", 3 if k == "batch_scan_mode3" else mode0)
        clf.run_cascade_batch_device(d_frames.data_ptr(), nf, ROWS * COLS, ROWS, COLS, COLS, *PARAMS, 0.0, uo[k].data_ptr(), ucap,
                                     uc[k].data_ptr(), st)
        torch.cuda.synchronize()   # the option is process-global: it must not change under a queued call
        pigo_b200.set_option("scan_mode", mode0)

    uts = {k: [] for k in uo}
    for rnd in range(7):
        for k in uo:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            u_run(k)
            b.record(stream)
            torch.cuda.synchronize()
            if rnd >= 2:
                uts[k].append(a.elapsed_time(b))
    ums = {k: float(np.median(v)) for k, v in uts.items()}
    same_u = all(torch.equal(uc["images"], uc[k]) for k in uo)
    return {"workload": f"{n} images of {len(geo)} geometries (seeded: common sizes 320x240..3840x2160 and odd sizes with Dim > Cols, "
                        "classes F/S), test parameters, device resident, CUDA events, median of 5 after 2 warm-ups",
            "images": n, "geometries": len(geo), "windows": W, "unit": "windows/s",
            "one_images_call": {"ms": ms["a"], "windows_per_s": W / (ms["a"] * 1e-3), "calls": 1},
            "batch_call_per_geometry": {"ms": ms["b"], "windows_per_s": W / (ms["b"] * 1e-3), "calls": len(geo)},
            "call_per_image": {"ms": ms["c"], "windows_per_s": W / (ms["c"] * 1e-3), "calls": n},
            "one_images_call_e2e_host": {"ms": ms_host, "windows_per_s": W / (ms_host * 1e-3), "h2d_bytes": int(sum(b.nbytes for b, *_ in imgs))},
            "outputs_identical": True, "detections": int(counts["a"].sum()),
            "uniform_1080p": {"frames": nf, "ms_images_call": ums["images"], "ms_batch_default": ums["batch"],
                              "ms_batch_scan_mode3": ums["batch_scan_mode3"],
                              "windows_per_s_images_call": Wf * nf / (ums["images"] * 1e-3),
                              "images_call_over_scan_mode3": ums["images"] / ums["batch_scan_mode3"],
                              "images_call_over_default": ums["images"] / ums["batch"], "counts_identical": bool(same_u),
                              "note": "median of 5 alternated rounds after 2"}}


def pipeline_bench(clf, dev: int, stream, d_frames, nf: int) -> dict:
    """The whole per-face sequence (pigo_detect_images / pigo_detect_batch, the reference's 15 landmark calls) on the mixed
    set three ways, and on uniform 1080p frames two ways; see the module docstring."""
    import ctypes as C
    import torch
    import pigo_b200
    from pigo_b200 import pipeline
    L = pigo_b200.lib()
    st = C.c_void_p(stream.cuda_stream)
    cuda = f"cuda:{dev}"
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
    names = sorted(set(pipeline.EYE_CASCADES + pipeline.MOUTH_CASCADES))
    flp = {nm: pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("lps/" + nm)) for nm in names}
    hs, fl = pipeline.landmark_call_arrays(flp)
    ncalls = len(fl)
    face_cap, det_cap = 128, 4096
    prm = pigo_b200.PipelineParams(*PARAMS, 0.0, 0.1, 50, 50, 63, det_cap)
    flags = pigo_b200.FRAMES_DEVICE | pigo_b200.OUT_DEVICE
    imgs = ragged_images()
    n = len(imgs)
    offs, total = [], 0
    for b, r, c, d in imgs:
        offs.append(total)
        total += (r * d + 255) & ~255
    host = np.zeros(total, dtype=np.uint8)
    for (b, r, c, d), o in zip(imgs, offs):
        host[o:o + r * d] = b.reshape(-1)
    dev_all = torch.from_numpy(host).to(cuda)
    descs = pigo_b200.image_descs([(dev_all.data_ptr() + o, r, c, d) for (b, r, c, d), o in zip(imgs, offs)])
    geo = {}
    for i, (_, r, c, d) in enumerate(imgs):
        geo.setdefault((r, c, d), []).append(i)
    geo_frames = {g: torch.stack([dev_all[offs[i]:offs[i] + g[0] * g[2]] for i in idx]) for g, idx in geo.items()}
    outs = {k: (torch.zeros((n, face_cap, 4), dtype=torch.int32, device=cuda), torch.zeros(n, dtype=torch.int32, device=cuda),
                torch.zeros((n, face_cap, 2 + ncalls, 4), dtype=torch.int32, device=cuda)) for k in "abc"}
    geo_out = {g: tuple(torch.zeros((len(idx),) + t.shape[1:], dtype=torch.int32, device=cuda) for t in outs["b"]) for g, idx in geo.items()}

    def check(rc):
        if rc != 0:
            raise RuntimeError(L.pigo_last_error().decode())

    def batch(frames_ptr, k, stride, r, c, d, o, rnd):
        check(L.pigo_detect_batch(clf._h, plc._h, hs, fl.ctypes.data, ncalls, frames_ptr, k, stride, r, c, d, C.byref(prm), rnd, 7,
                                  o[0].data_ptr(), face_cap, o[1].data_ptr(), o[2].data_ptr(), flags, st))

    def run_a(rnd=None):
        check(L.pigo_detect_images(clf._h, plc._h, hs, fl.ctypes.data, ncalls, descs, n, C.byref(prm), rnd.data_ptr() if rnd is not None else None,
                                   7, outs["a"][0].data_ptr(), face_cap, outs["a"][1].data_ptr(), outs["a"][2].data_ptr(), flags, st))

    def run_b(rnd=None):
        for g, fr in geo_frames.items():
            rg = rnd[geo[g]].contiguous() if rnd is not None else None
            batch(fr.data_ptr(), fr.shape[0], g[0] * g[2], *g, geo_out[g], rg.data_ptr() if rg is not None else None)
            if rnd is not None:
                torch.cuda.synchronize()   # rg must outlive the asynchronous call

    def run_c(rnd=None):
        for i, (b, r, c, d) in enumerate(imgs):
            o = tuple(t[i:i + 1] for t in outs["c"])
            batch(dev_all.data_ptr() + offs[i], 1, r * d, r, c, d, o, rnd[i].data_ptr() if rnd is not None else None)

    def gather_b():
        for g, idx in geo.items():
            for t, u in zip(outs["b"], geo_out[g]):
                t[idx] = u

    def timed(fn, reps=5, warm=2):
        for _ in range(warm):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            fn()
            b.record(stream)
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return float(np.median(ts))

    ms = {k: timed(f) for k, f in (("a", run_a), ("b", run_b), ("c", run_c))}
    gather_b()
    res = {k: [t.cpu().numpy() for t in outs[k]] for k in "abc"}
    assert int(res["a"][1].max()) <= face_cap, "raise face_cap: an image has more faces than the bench buffer"
    for k in "bc":
        assert np.array_equal(res["a"][1], res[k][1]), f"pipeline: face counts of ({k}) differ"
        assert res["a"][0].tobytes() == res[k][0].tobytes(), f"pipeline: faces of ({k}) differ"
    # points: generator keys depend on the frame index, so compare with the same injected randoms (untimed)
    rnd = torch.from_numpy(np.random.default_rng(11).random((n, face_cap, 2 + ncalls, 63, 3), dtype=np.float32)).to(cuda)
    run_a(rnd); run_b(rnd); run_c(rnd)
    torch.cuda.synchronize()
    gather_b()
    pts = {k: outs[k][2].cpu().numpy() for k in "abc"}
    assert pts["a"].tobytes() == pts["b"].tobytes() == pts["c"].tobytes(), "pipeline: points differ with injected randoms"
    del rnd
    refined = int((res["a"][0][..., 2] > 50).sum())

    # uniform 1080p: the mixed call against the batch call on the same frames, alternated
    uo = {k: (torch.zeros((nf, face_cap, 4), dtype=torch.int32, device=cuda), torch.zeros(nf, dtype=torch.int32, device=cuda),
              torch.zeros((nf, face_cap, 2 + ncalls, 4), dtype=torch.int32, device=cuda)) for k in ("images", "batch")}
    udesc = pigo_b200.image_descs([(d_frames[i].data_ptr(), ROWS, COLS, COLS) for i in range(nf)])

    def u_run(k):
        o = uo[k]
        if k == "images":
            check(L.pigo_detect_images(clf._h, plc._h, hs, fl.ctypes.data, ncalls, udesc, nf, C.byref(prm), None, 7, o[0].data_ptr(), face_cap,
                                       o[1].data_ptr(), o[2].data_ptr(), flags, st))
        else:
            batch(d_frames.data_ptr(), nf, ROWS * COLS, ROWS, COLS, COLS, o, None)

    uts = {k: [] for k in uo}
    for r in range(7):
        for k in uo:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            u_run(k)
            b.record(stream)
            torch.cuda.synchronize()
            if r >= 2:
                uts[k].append(a.elapsed_time(b))
    ums = {k: float(np.median(v)) for k, v in uts.items()}
    same_u = all(torch.equal(x, y) for x, y in zip(uo["images"], uo["batch"]))
    return {"workload": f"{n} images of {len(geo)} geometries (the scan section's set), test parameters, eye Perturbs 50, 15 landmark calls, "
                        "device resident, device outputs, CUDA events, median of 5 after 2 warm-ups",
            "one_detect_images_call_ms": ms["a"], "detect_batch_per_geometry_ms": ms["b"], "detect_batch_per_image_ms": ms["c"],
            "calls": {"a": 1, "b": len(geo), "c": n}, "faces": int(res["a"][1].sum()), "refined_faces": refined,
            "faces_counts_identical": True, "points_identical_with_injected_randoms": True,
            "uniform_1080p": {"frames": nf, "ms_detect_images": ums["images"], "ms_detect_batch": ums["batch"],
                              "images_over_batch": ums["images"] / ums["batch"], "outputs_identical": bool(same_u),
                              "note": "median of 5 alternated rounds after 2"}}


def angles_bench(clf, dev: int, stream) -> dict:
    """Angle sweeps as one pigo_run_cascade_images_angles / pigo_detect_images_angles call against one call per angle (device
    resident, CUDA events, outputs asserted identical); see the module docstring."""
    import ctypes as C
    import torch
    import pigo_b200
    from pigo_b200 import pipeline, synth
    L = pigo_b200.lib()
    st = stream.cuda_stream
    cuda = f"cuda:{dev}"

    def timed(fn, reps=7, warm=2):
        for _ in range(warm):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            fn()
            b.record(stream)
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return float(np.median(ts))

    def zeros(*shape):
        return torch.zeros(shape, dtype=torch.int32, device=cuda)

    res = {}
    # (1) one 1080p frame at angle 0 and k/32, k = 1..32: one call over 33 pointers to the frame against 33 single-frame calls
    cap = 1024
    fr = torch.from_numpy(synth.frame_faces(None, 1080, 1920, noise_seed=3)).to(cuda)
    sweep = [0.0] + [k / 32 for k in range(1, 33)]
    na = len(sweep)
    desc = [(fr.data_ptr(), 1080, 1920, 1920)] * na
    o1, c1, o2, c2 = zeros(na, cap, 4), zeros(na), zeros(na, cap, 4), zeros(na)
    W1 = pigo_b200.count_windows(1080, 1920, *PARAMS) * na
    ms_one = timed(lambda: clf.run_cascade_images_angles_device(desc, sweep, *PARAMS, o1.data_ptr(), cap, c1.data_ptr(), st))
    ms_lone = timed(lambda: [clf.run_cascade_batch_device(fr.data_ptr(), 1, 1080 * 1920, 1080, 1920, 1920, *PARAMS, a, o2[k].data_ptr(), cap,
                                                          c2.data_ptr() + 4 * k, st) for k, a in enumerate(sweep)])
    assert torch.equal(c1, c2) and int(c1.max()) <= cap
    assert all(torch.equal(o1[k, :c1[k]], o2[k, :c1[k]]) for k in range(na)), "angles (1): outputs differ"
    res["sweep_1080p"] = {"workload": "one 1080p frame (class F) at angle 0 and k/32, k = 1..32", "entries": na, "windows": W1,
                          "ms_one_call": ms_one, "ms_call_per_angle": ms_lone, "calls": {"one": 1, "per_angle": na},
                          "speedup": ms_lone / ms_one, "detections": int(c1.sum()), "outputs_identical": True}

    # (2) bench.py's configs[3] workload: 8 x 4K frames at the 32 rotated slots, one call over pointers into the batch against
    #     one batch call per slot
    R4, C4, n4, cap4 = 2160, 3840, 8, 4096
    fr4 = torch.from_numpy(np.stack([synth.frame_faces(None, R4, C4, shift=(31 * i, 17 * i), noise_seed=i) for i in range(n4)])).to(cuda)
    rot = [k / 32 for k in range(1, 33)]
    desc4 = [(fr4[i].data_ptr(), R4, C4, C4) for a in rot for i in range(n4)]   # angle-major: slot k's frames contiguous
    ang4 = [a for a in rot for _ in range(n4)]
    o1, c1, o2, c2 = zeros(len(desc4), cap4, 4), zeros(len(desc4)), zeros(len(desc4), cap4, 4), zeros(len(desc4))
    W4 = pigo_b200.count_windows(R4, C4, *PARAMS) * n4 * len(rot)
    ms_one = timed(lambda: clf.run_cascade_images_angles_device(desc4, ang4, *PARAMS, o1.data_ptr(), cap4, c1.data_ptr(), st), reps=5)
    ms_lone = timed(lambda: [clf.run_cascade_batch_device(fr4.data_ptr(), n4, R4 * C4, R4, C4, C4, *PARAMS, a, o2[k * n4].data_ptr(), cap4,
                                                          c2.data_ptr() + 4 * k * n4, st) for k, a in enumerate(rot)], reps=5)
    assert torch.equal(c1, c2) and int(c1.max()) <= cap4
    assert all(torch.equal(o1[k, :c1[k]], o2[k, :c1[k]]) for k in range(len(desc4))), "angles (2): outputs differ"
    res["config4_sweep"] = {"workload": f"{n4} x 3840x2160 frames (class F, bench.py configs[3]) at angle k/32, k = 1..32", "entries": len(desc4),
                            "windows": W4, "ms_one_call": ms_one, "ms_batch_call_per_angle": ms_lone, "calls": {"one": 1, "per_angle": len(rot)},
                            "speedup": ms_lone / ms_one, "windows_per_s_one_call": W4 / (ms_one * 1e-3), "detections": int(c1.sum()),
                            "outputs_identical": True}
    del fr4, o1, c1, o2, c2

    # (3) pipeline: 16 mixed images x 8 angles, one pigo_detect_images_angles call (listed image-major and angle-major) against
    #     one pigo_detect_images call per angle
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
    names = sorted(set(pipeline.EYE_CASCADES + pipeline.MOUTH_CASCADES))
    flp = {nm: pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("lps/" + nm)) for nm in names}
    hs, fl = pipeline.landmark_call_arrays(flp)
    ncalls = len(fl)
    face_cap = 256
    prm = pigo_b200.PipelineParams(*PARAMS, 0.0, 0.1, 50, 50, 63, 4096)
    flags = pigo_b200.FRAMES_DEVICE | pigo_b200.OUT_DEVICE
    imgs = [im for im in ragged_images(64, seed=7) if im[2] >= im[1]][:16]   # wide images: the rotated column clamp stays inside
    offs, total = [], 0
    for b, r, c, d in imgs:
        offs.append(total)
        total += (r * d + 255) & ~255
    host = np.zeros(total, dtype=np.uint8)
    for (b, r, c, d), o in zip(imgs, offs):
        host[o:o + r * d] = b.reshape(-1)
    dev_all = torch.from_numpy(host).to(cuda)
    base = [(dev_all.data_ptr() + o, r, c, d) for (b, r, c, d), o in zip(imgs, offs)]
    pang = [0.0, 0.02, 0.05, 0.1, 0.25, 0.5, 0.75, 1.0]
    ni, nk = len(base), len(pang)
    n = ni * nk
    listings = {"image_major": [(i, k) for i in range(ni) for k in range(nk)], "angle_major": [(i, k) for k in range(nk) for i in range(ni)]}
    outs = {key: (zeros(n, face_cap, 4), zeros(n), zeros(n, face_cap, 2 + ncalls, 4)) for key in ("image_major", "angle_major", "per_angle")}
    pdesc = pigo_b200.image_descs(base)

    def check(rc):
        if rc != 0:
            raise RuntimeError(L.pigo_last_error().decode())

    def one(key):
        lst = listings[key]
        d = pigo_b200.image_descs([base[i] for i, _ in lst])
        a = np.array([pang[k] for _, k in lst], dtype=np.float64)
        o = outs[key]
        return lambda rnd=None: check(L.pigo_detect_images_angles(clf._h, plc._h, hs, fl.ctypes.data, ncalls, d, n, a.ctypes.data, C.byref(prm),
                                                                  rnd.data_ptr() if rnd is not None else None, 7, o[0].data_ptr(), face_cap,
                                                                  o[1].data_ptr(), o[2].data_ptr(), flags, C.c_void_p(st)))

    def per_angle(rnd=None):
        o = outs["per_angle"]   # angle-major slices: angle k's images at rows k*ni .. (k+1)*ni
        for k, a in enumerate(pang):
            p = pigo_b200.PipelineParams(*PARAMS, a, 0.1, 50, 50, 63, 4096)
            check(L.pigo_detect_images(clf._h, plc._h, hs, fl.ctypes.data, ncalls, pdesc, ni, C.byref(p), rnd[k * ni].data_ptr() if rnd is not None else None,
                                       7, o[0][k * ni].data_ptr(), face_cap, o[1].data_ptr() + 4 * k * ni, o[2][k * ni].data_ptr(), flags,
                                       C.c_void_p(st)))

    run_im, run_am = one("image_major"), one("angle_major")
    pms = {"image_major": [], "angle_major": [], "per_angle": []}
    for f in (run_im, run_am, per_angle):
        f(); f()
    torch.cuda.synchronize()
    for rnd in range(7):   # alternated rounds, so that drift hits the three alike
        for key, f in (("image_major", run_im), ("angle_major", run_am), ("per_angle", per_angle)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            f()
            b.record(stream)
            torch.cuda.synchronize()
            if rnd >= 2:
                pms[key].append(a.elapsed_time(b))
    pm = {k: float(np.median(v)) for k, v in pms.items()}
    # faces and counts of the timed runs must agree; points (the generator's key is the slot index) are compared in an untimed
    # run with the same injected randoms per (image, angle)
    r = {k: [t.cpu().numpy() for t in v] for k, v in outs.items()}
    assert int(r["per_angle"][1].max()) <= face_cap
    am_pos = {ik: p for p, ik in enumerate(listings["angle_major"])}
    for key in ("image_major", "angle_major"):
        for p, ik in enumerate(listings[key]):
            q = am_pos[ik]   # the per-angle calls' outputs are angle-major
            assert r[key][1][p] == r["per_angle"][1][q] and r[key][0][p].tobytes() == r["per_angle"][0][q].tobytes(), f"angles (3): {key} differs"
    rnd = torch.from_numpy(np.random.default_rng(13).random((n, face_cap, 2 + ncalls, 63, 3), dtype=np.float32)).to(cuda)   # angle-major
    rnd_im = rnd[[am_pos[ik] for ik in listings["image_major"]]].contiguous()
    run_im(rnd_im); run_am(rnd); per_angle(rnd)
    torch.cuda.synchronize()
    pts = {k: v[2].cpu().numpy() for k, v in outs.items()}
    assert pts["angle_major"].tobytes() == pts["per_angle"].tobytes(), "angles (3): points differ with injected randoms"
    assert all(pts["image_major"][p].tobytes() == pts["per_angle"][am_pos[ik]].tobytes() for p, ik in enumerate(listings["image_major"]))
    del rnd, rnd_im
    res["pipeline_sweep"] = {"workload": f"{ni} wide images of the scan section's mix x {nk} angles {pang}, 15 landmark calls, device outputs",
                             "entries": n, "ms_one_call_image_major": pm["image_major"], "ms_one_call_angle_major": pm["angle_major"],
                             "ms_detect_images_per_angle": pm["per_angle"], "calls": {"one": 1, "per_angle": nk},
                             "speedup": pm["per_angle"] / pm["angle_major"], "faces": int(r["per_angle"][1].sum()),
                             "refined_faces": int((r["per_angle"][0][..., 2] > 50).sum()), "outputs_identical": True,
                             "note": "median of 5 alternated rounds after 2"}
    res["note"] = "device resident, CUDA events; (1) and (2) median of 7 / 5 after 2 warm-ups"
    return res


def sweep_bench(clf, dev: int, stream) -> dict:
    """An angle sweep merged per image: one pigo_detect_images_sweep call against pigo_detect_images_angles over the expanded
    (image x angle) list followed by a merge through host memory (D2H of its faces, then pigo_cluster_batch of each image's
    concatenated faces).  Host clock around each way ending in a synchronise, median of 5 after 2; the merge kernels' own
    time from the library's CUDA-event timing (option "timing") in a separate run."""
    import ctypes as C
    import time
    import torch
    import pigo_b200
    from pigo_b200 import pipeline, synth
    L = pigo_b200.lib()
    st = stream.cuda_stream
    cuda = f"cuda:{dev}"
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
    names = sorted(set(pipeline.EYE_CASCADES + pipeline.MOUTH_CASCADES))
    flp = {nm: pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("lps/" + nm)) for nm in names}
    hs, fl = pipeline.landmark_call_arrays(flp)
    ncalls = len(fl)
    angles = [k / 32 for k in range(32)]
    ang = np.array(angles, dtype=np.float64)
    na = len(angles)
    flags = pigo_b200.FRAMES_DEVICE | pigo_b200.OUT_DEVICE

    def check(rc):
        if rc != 0:
            raise RuntimeError(L.pigo_last_error().decode())

    def wall(fn, reps=5, warm=2):
        for _ in range(warm):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(ts))

    def workload(base, face_cap):
        n = len(base)
        prm = pigo_b200.PipelineParams(*PARAMS, 0.0, 0.1, 50, 50, 63, 4096)
        desc = pigo_b200.image_descs(base)
        f = torch.zeros((n, face_cap, 4), dtype=torch.int32, device=cuda)
        fa = torch.zeros((n, face_cap), dtype=torch.int32, device=cuda)
        nf = torch.zeros(n, dtype=torch.int32, device=cuda)
        pts = torch.zeros((n, face_cap, 2 + ncalls, 4), dtype=torch.int32, device=cuda)

        def sweep():
            check(L.pigo_detect_images_sweep(clf._h, plc._h, hs, fl.ctypes.data, ncalls, desc, n, ang.ctypes.data, na, C.byref(prm), None, 7,
                                             f.data_ptr(), fa.data_ptr(), face_cap, nf.data_ptr(), pts.data_ptr(), flags, C.c_void_p(st)))

        ex = pigo_b200.image_descs([b for b in base for _ in angles])
        exa = np.array([a for _ in base for a in angles], dtype=np.float64)
        m = n * na
        ef = torch.zeros((m, face_cap, 4), dtype=torch.int32, device=cuda)
        enf = torch.zeros(m, dtype=torch.int32, device=cuda)
        epts = torch.zeros((m, face_cap, 2 + ncalls, 4), dtype=torch.int32, device=cuda)
        merged = {}

        def per_entry():
            check(L.pigo_detect_images_angles(clf._h, plc._h, hs, fl.ctypes.data, ncalls, ex, m, exa.ctypes.data, C.byref(prm), None, 7,
                                              ef.data_ptr(), face_cap, enf.data_ptr(), epts.data_ptr(), flags, C.c_void_p(st)))
            faces = ef.cpu().numpy().view(pigo_b200.DET_DTYPE).reshape(n, na * face_cap)
            cnt = enf.cpu().numpy().reshape(n, na)
            cat = np.zeros((n, na * face_cap), dtype=pigo_b200.DET_DTYPE)
            k = np.zeros(n, dtype=np.int32)
            for i in range(n):
                parts = [faces[i, a * face_cap:a * face_cap + cnt[i, a]] for a in range(na)]
                k[i] = sum(len(p) for p in parts)
                cat[i, :k[i]] = np.concatenate(parts)
            merged["clusters"], merged["n"] = clf.cluster_batch_array(cat, k, 0.1)
            merged["refined"] = int((cat["scale"] > 50).sum())

        ms_sweep = wall(sweep)
        ms_entry = wall(per_entry)
        pigo_b200.set_option("timing", 1)
        sweep()
        torch.cuda.synchronize()
        merge_ms = pigo_b200.get_option("t_merge_ns") / 1e6
        merge_n = pigo_b200.get_option("t_merge_n")
        pigo_b200.set_option("timing", 0)
        nfh, fh = nf.cpu().numpy(), f.cpu().numpy().view(pigo_b200.DET_DTYPE).reshape(n, face_cap)
        assert int(nfh.max()) <= face_cap and int(enf.max()) <= face_cap, (int(nfh.max()), int(enf.max()), face_cap)
        refined = int(sum((fh[i, :nfh[i]]["scale"] > 50).sum() for i in range(n)))
        return {"images": n, "angles": na, "ms_sweep": ms_sweep, "ms_angles_plus_host_merge": ms_entry, "speedup": ms_entry / ms_sweep,
                "merge_kernels_ms": merge_ms, "merge_launches": merge_n, "faces_sweep": int(nfh.sum()), "refined_sweep": refined,
                "faces_host_merge": int(merged["n"].sum()), "refined_per_entry": merged["refined"]}

    res = {}
    fr = torch.from_numpy(synth.frame_faces(None, 1080, 1920, noise_seed=3)).to(cuda)
    res["frame_1080p"] = workload([(fr.data_ptr(), 1080, 1920, 1920)], 1024)
    imgs = [im for im in ragged_images(64, seed=7) if im[2] >= im[1]][:16]   # wide images: the rotated column clamp stays inside
    offs, total = [], 0
    for b, r, c, d in imgs:
        offs.append(total)
        total += (r * d + 255) & ~255
    host = np.zeros(total, dtype=np.uint8)
    for (b, r, c, d), o in zip(imgs, offs):
        host[o:o + r * d] = b.reshape(-1)
    dev_all = torch.from_numpy(host).to(cuda)
    res["mixed_16"] = workload([(dev_all.data_ptr() + o, r, c, d) for (b, r, c, d), o in zip(imgs, offs)], 1024)
    res["note"] = ("k/32, k = 0..31; test parameters, IoU 0.1, eye Perturbs 50, 15 landmark calls, device images; host clock, median of 5 "
                   "after 2; merge_kernels_ms = compaction + segmented sort + tagged clustering of one sweep call (CUDA events)")
    return res


def decoded_bench(clf, dev: int, stream) -> dict:
    """Decoded JPEG-like sources to detector results three ways, and the conversion alone; see the module docstring."""
    import ctypes as C
    import torch
    import pigo_b200
    from pigo_b200 import DecodedImage, pipeline
    L = pigo_b200.lib()
    st = C.c_void_p(stream.cuda_stream)
    cuda = f"cuda:{dev}"
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
    names = sorted(set(pipeline.EYE_CASCADES + pipeline.MOUTH_CASCADES))
    flp = {nm: pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("lps/" + nm)) for nm in names}
    hs, fl = pipeline.landmark_call_arrays(flp)
    ncalls = len(fl)
    face_cap = 128
    prm = pigo_b200.PipelineParams(*PARAMS, 0.0, 0.1, 50, 50, 63, 4096)
    rng = np.random.default_rng(77)
    imgs = ragged_images()
    n = len(imgs)

    def check(rc):
        if rc != 0:
            raise RuntimeError(L.pigo_last_error().decode())

    # 4:2:0 planes of every image in pinned host memory (YStride = the image's Dim, CStride = chroma width + 3)
    planes, src_bytes = [], 0
    for b, r, c, d in imgs:
        cw, ch = (c + 1) // 2, (r + 1) // 2
        y = torch.from_numpy(np.ascontiguousarray(b)).pin_memory()
        cb = torch.from_numpy((128 + rng.integers(-20, 21, size=(ch, cw + 3))).astype(np.uint8)).pin_memory()
        cr = torch.from_numpy((128 + rng.integers(-20, 21, size=(ch, cw + 3))).astype(np.uint8)).pin_memory()
        planes.append((y, cb, cr))
        src_bytes += r * c + 2 * ch * cw
    gray_px = sum(r * c for _, r, c, _ in imgs)
    host_src = [DecodedImage.ycbcr(y, cb, cr, 2, c, r, y_stride=d, c_stride=cb.shape[1]) for (y, cb, cr), (_, r, c, d) in zip(planes, imgs)]
    dev_planes = [tuple(p.to(cuda) for p in pl) for pl in planes]
    dev_src = [DecodedImage.ycbcr(y, cb, cr, 2, c, r, y_stride=d, c_stride=cb.shape[1]) for (y, cb, cr), (_, r, c, d) in zip(dev_planes, imgs)]
    need = pigo_b200.gray_images_bytes(host_src)
    arena = torch.empty(need, dtype=torch.uint8, device=cuda)
    host_descs, dev_descs = pigo_b200.decoded_descs(host_src), pigo_b200.decoded_descs(dev_src)
    out_imgs = (pigo_b200.PigoImage * n)()
    size = C.c_size_t(need)

    def outputs():
        return (np.zeros((n, face_cap), dtype=pigo_b200.DET_DTYPE), np.zeros(n, dtype=np.int32),
                np.zeros((n, face_cap, 2 + ncalls), dtype=pigo_b200.POINT_DTYPE))

    def detect(descs, flags, o):
        check(L.pigo_detect_images(clf._h, plc._h, hs, fl.ctypes.data, ncalls, descs, n, C.byref(prm), None, 7, o[0].ctypes.data, face_cap,
                                   o[1].ctypes.data, o[2].ctypes.data, flags, st))

    gray_host = [np.zeros((r, c), dtype=np.uint8) for _, r, c, _ in imgs]
    nrgba_host = [np.zeros((r, c, 4), dtype=np.uint8) for _, r, c, _ in imgs]
    gray_descs = pigo_b200.image_descs([(g.ctypes.data, r, c, c) for g, (_, r, c, _) in zip(gray_host, imgs)])

    def way_a(o):
        check(L.pigo_gray_images(host_descs, n, arena.data_ptr(), C.byref(size), out_imgs, pigo_b200.MEM_HOST, st))
        detect(out_imgs, pigo_b200.FRAMES_DEVICE, o)

    def ycc(i, nrgba, gray):
        (y, cb, cr), (_, r, c, d) = planes[i], imgs[i]
        check(L.pigo_ycbcr_to_nrgba(y.data_ptr(), cb.data_ptr(), cr.data_ptr(), d, cb.shape[1], 2, 0, 0, c, r, nrgba, gray, pigo_b200.MEM_HOST, st))

    def way_b(o):
        for i in range(n):
            ycc(i, None, gray_host[i].ctypes.data)
        detect(gray_descs, pigo_b200.MEM_HOST, o)

    def way_c(o):
        for i in range(n):
            ycc(i, nrgba_host[i].ctypes.data, None)
            check(L.pigo_rgba_to_gray(nrgba_host[i].ctypes.data, nrgba_host[i].size // 4, gray_host[i].ctypes.data, pigo_b200.MEM_HOST, st))
        detect(gray_descs, pigo_b200.MEM_HOST, o)

    res, outs = {}, {}
    for name, fn in (("a_gray_images_then_detect", way_a), ("b_ycbcr_gray_per_image", way_b), ("c_nrgba_then_gray_per_image", way_c)):
        o = outputs()
        fn(o)   # warm-up
        ts = []
        for _ in range(5):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn(o)
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        res[name + "_ms"] = round(1e3 * float(np.median(ts)), 3)
        outs[name] = o
    ref = outs["a_gray_images_then_detect"]
    for name, o in outs.items():
        assert all(x.tobytes() == y.tobytes() for x, y in zip(o, ref)), f"{name} differs from the one-call way"
    res["faces"] = int(ref[1].sum())

    # the conversion alone: device-resident planes (CUDA events), pinned host planes (host clock)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ks = []
    for _ in range(6):
        ev[0].record(stream)
        check(L.pigo_gray_images(dev_descs, n, arena.data_ptr(), C.byref(size), out_imgs, pigo_b200.FRAMES_DEVICE, st))
        ev[1].record(stream)
        ev[1].synchronize()
        ks.append(ev[0].elapsed_time(ev[1]))
    k_ms = float(np.median(ks[1:]))
    moved = src_bytes + gray_px
    res["gray_images_device_ms"] = round(k_ms, 4)
    res["gray_images_device_bytes"] = moved
    res["gray_images_device_tb_s"] = round(moved / (k_ms * 1e-3) / 1e12, 3)
    res["gray_images_device_of_3_35_tb_s"] = round(moved / (k_ms * 1e-3) / 3.35e12, 3)
    hs_ = []
    for _ in range(6):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        check(L.pigo_gray_images(host_descs, n, arena.data_ptr(), C.byref(size), out_imgs, pigo_b200.MEM_HOST, st))
        torch.cuda.synchronize()
        hs_.append(time.perf_counter() - t0)
    h_s = float(np.median(hs_[1:]))
    res["gray_images_pinned_ms"] = round(1e3 * h_s, 3)
    res["gray_images_pinned_source_gb_s"] = round(src_bytes / h_s / 1e9, 2)
    res["source_bytes"], res["gray_pixels"], res["images"] = src_bytes, gray_px, n
    return res


FORMATS = {"nrgba": (1, 4), "gray16": (5, 2), "rgba64": (6, 8), "nrgba64": (7, 8), "cmyk": (8, 4), "paletted": (9, 1)}   # code, bytes/px


def encode_gray(fmt: str, b: np.ndarray, noise: np.ndarray, inv: np.ndarray, out: np.ndarray) -> None:
    """Writes into out [rows][dim * bytes/px] the Pix rows of gray image b [rows][dim] in format fmt such that
    RgbToGrayscale(ImgToNRGBA(img)) is b: NRGBA opaque (g, g, g); Gray16 g<<8 | noise; RGBA64 and NRGBA64 opaque with each
    channel g<<8 | noise; CMYK (0, 0, 0, 255-g); Paletted the index inv[g] of a permuted gray palette."""
    r, d = b.shape
    bpp = FORMATS[fmt][1]
    px = out.reshape(r, d, bpp)
    if fmt == "nrgba":
        px[..., :3] = b[..., None]
        px[..., 3] = 255
    elif fmt == "gray16":
        px[..., 0], px[..., 1] = b, noise
    elif fmt in ("rgba64", "nrgba64"):
        px[..., 0:6:2] = b[..., None]
        px[..., 1:6:2] = noise[..., None]
        px[..., 6:] = 255
    elif fmt == "cmyk":
        px[..., :3] = 0
        px[..., 3] = 255 - b
    else:
        px[..., 0] = inv[b]


def formats_bench(clf, dev: int, stream) -> dict:
    """The 256 ragged images encoded in each format pigo_gray_images takes beyond YCbCr and Gray, each such that its gray
    is exactly the image (encode_gray): detections asserted equal to those of the plain gray images; pigo_gray_images alone
    from device-resident planes (CUDA events) and from pinned host planes (host clock), and pigo_gray_images +
    pigo_detect_images end to end from pinned planes (host clock), medians of 5.  NRGBA is what a caller converting on
    the CPU first (the Go shim's ImgToNRGBA for these types) sends; that CPU pass itself is not measured here."""
    import ctypes as C
    import torch
    import pigo_b200
    from pigo_b200 import DecodedImage, pipeline
    L = pigo_b200.lib()
    st = C.c_void_p(stream.cuda_stream)
    cuda = f"cuda:{dev}"
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
    names = sorted(set(pipeline.EYE_CASCADES + pipeline.MOUTH_CASCADES))
    flp = {nm: pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("lps/" + nm)) for nm in names}
    hs, fl = pipeline.landmark_call_arrays(flp)
    ncalls, face_cap = len(fl), 128
    prm = pigo_b200.PipelineParams(*PARAMS, 0.0, 0.1, 50, 50, 63, 4096)
    imgs = ragged_images()
    n = len(imgs)
    gray_px = sum(r * c for _, r, c, _ in imgs)

    def check(rc):
        if rc != 0:
            raise RuntimeError(L.pigo_last_error().decode())

    def outputs():
        return (np.zeros((n, face_cap), dtype=pigo_b200.DET_DTYPE), np.zeros(n, dtype=np.int32),
                np.zeros((n, face_cap, 2 + ncalls), dtype=pigo_b200.POINT_DTYPE))

    def detect(descs, flags, o):
        check(L.pigo_detect_images(clf._h, plc._h, hs, fl.ctypes.data, ncalls, descs, n, C.byref(prm), None, 7, o[0].ctypes.data, face_cap,
                                   o[1].ctypes.data, o[2].ctypes.data, flags, st))

    def host_ms(fn, reps=5):
        fn()
        ts = []
        for _ in range(reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        return 1e3 * float(np.median(ts))

    gray = [np.ascontiguousarray(b[:, :c]) for b, _, c, _ in imgs]
    ref = outputs()
    detect(pigo_b200.image_descs([(g.ctypes.data, r, c, c) for g, (_, r, c, _) in zip(gray, imgs)]), pigo_b200.MEM_HOST, ref)
    rng = np.random.default_rng(78)
    perm = rng.permutation(256)
    palette = torch.from_numpy(np.stack([perm, perm, perm, np.full(256, 255)], axis=-1).astype(np.uint8)).pin_memory()
    inv = np.argsort(perm).astype(np.uint8)
    res = {}
    for fmt, (code, bpp) in FORMATS.items():
        pinned = []
        for b, r, c, d in imgs:
            t = torch.empty((r, d * bpp), dtype=torch.uint8, pin_memory=True)
            encode_gray(fmt, b, rng.integers(0, 256, size=(r, d), dtype=np.uint8), inv, t.numpy())
            pinned.append(t)
        dev_planes = [t.to(cuda) for t in pinned]
        d_palette = palette.to(cuda)

        def src(planes, pal):
            return [DecodedImage(code, c, r, (p, pal) if fmt == "paletted" else (p,), (d * bpp, len(pal) if fmt == "paletted" else 0))
                    for p, (_, r, c, d) in zip(planes, imgs)]
        host_descs, dev_descs = pigo_b200.decoded_descs(src(pinned, palette)), pigo_b200.decoded_descs(src(dev_planes, d_palette))
        need = pigo_b200.gray_images_bytes(src(pinned, palette))
        arena = torch.empty(need, dtype=torch.uint8, device=cuda)
        out_imgs = (pigo_b200.PigoImage * n)()
        size = C.c_size_t(need)

        def convert(descs, flags):
            check(L.pigo_gray_images(descs, n, arena.data_ptr(), C.byref(size), out_imgs, flags, st))

        o = outputs()

        def e2e():
            convert(host_descs, pigo_b200.MEM_HOST)
            detect(out_imgs, pigo_b200.FRAMES_DEVICE, o)
        row = {"e2e_ms": round(host_ms(e2e), 3)}
        assert all(x.tobytes() == y.tobytes() for x, y in zip(o, ref)), f"{fmt}: detections differ from the gray images'"
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ks = []
        for _ in range(6):
            ev[0].record(stream)
            convert(dev_descs, pigo_b200.FRAMES_DEVICE)
            ev[1].record(stream)
            ev[1].synchronize()
            ks.append(ev[0].elapsed_time(ev[1]))
        k_ms = float(np.median(ks[1:]))
        src_bytes = gray_px * bpp + (1024 if fmt == "paletted" else 0)
        row["gray_images_device_ms"] = round(k_ms, 4)
        row["gray_images_device_tb_s"] = round((src_bytes + gray_px) / (k_ms * 1e-3) / 1e12, 3)
        row["gray_images_device_of_3_35_tb_s"] = round((src_bytes + gray_px) / (k_ms * 1e-3) / 3.35e12, 3)
        p_ms = host_ms(lambda: convert(host_descs, pigo_b200.MEM_HOST))
        row["gray_images_pinned_ms"] = round(p_ms, 3)
        row["gray_images_pinned_source_gb_s"] = round(src_bytes / (p_ms * 1e-3) / 1e9, 2)
        row["source_bytes"] = src_bytes
        res[fmt] = row
        del pinned, dev_planes, arena
        torch.cuda.empty_cache()
    res["faces"], res["gray_pixels"], res["images"] = int(ref[1].sum()), gray_px, n
    res["go_cpu_pass"] = "not measured"
    return res


def sharded_bench(clf, dev: int) -> dict:
    """The sharded mixed-size calls on the 256 images, host inputs and outputs, host clock, median of 5 alternated rounds:
    one pigo_run_cascade_images_angles / pigo_detect_images_angles call against pigo_run_cascade_images_sharded /
    pigo_detect_images_sharded with shard_split 1, 2, 4 and 8 on the visible devices (outputs asserted identical).  On one
    GPU every shard shares the card: the difference is the cost of splitting, not scaling.  Then the cost model: every
    shard of the 4- and 8-way splits timed alone as a single-device call against its modelled cost, and a least-squares fit
    of time = a * unrotated windows + b * rotated windows + c * images over those shards (k_rot = b / a, k_img = c / a)."""
    import torch
    import pigo_b200
    from pigo_b200 import CascadeParams, ImageParams, pipeline
    imgs = ragged_images()
    n = len(imgs)
    rng = np.random.default_rng(7)
    # a quarter of the wide images rotated (tall images stay unrotated: see tests/test_angles_gpu.py)
    angles = [float(rng.choice([0.1, 0.25, 0.5])) if c >= r and rng.random() < 0.25 else 0.0 for _, r, c, _ in imgs]
    images = [ImageParams(b, r, c, d) for b, r, c, d in imgs]
    cp = CascadeParams(ImageParams(), *PARAMS)
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
    flp = {k: pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("lps/" + k))
           for k in sorted(set(pipeline.EYE_CASCADES + pipeline.MOUTH_CASCADES))}
    splits = [1, 2, 4, 8]
    ways = {"one_call": None, **{f"sharded_{k}": k for k in splits}}
    old = pigo_b200.get_option("shard_split")

    def scan(k):
        if k is None:
            return clf.RunCascadeImagesAngles(images, cp, angles, 4096)
        pigo_b200.set_option("shard_split", k)
        return clf.run_cascade_images_sharded(images, cp, angles, 4096)

    def detect(k):
        if k is None:
            return pipeline.detect_images_angles_device(clf, plc, flp, images, cp, angles, face_cap=64, rng_seed=5, raw=True)
        pigo_b200.set_option("shard_split", k)
        return pipeline.detect_images_sharded(clf, plc, flp, images, cp, angles, face_cap=64, rng_seed=5, raw=True)

    def timed(fn):
        torch.cuda.synchronize(dev)
        t = time.perf_counter()
        r = fn()
        return r, (time.perf_counter() - t) * 1e3

    res = {"images": n, "rotated": int(sum(a > 0 for a in angles)), "devices": torch.cuda.device_count()}
    try:
        for name, fn in (("scan", scan), ("pipeline", detect)):
            ref = fn(None)
            for k in splits:   # warm-up, and the outputs
                got = fn(k)
                assert all(a.tobytes() == b.tobytes() for a, b in zip(got, ref)), (name, k)
            ms = {w: [] for w in ways}
            for _ in range(5):
                for w, k in ways.items():
                    ms[w].append(timed(lambda: fn(k))[1])
            res[name] = {w: round(float(np.median(v)), 2) for w, v in ms.items()}
        # cost model against per-shard times (each shard alone, one device, host in and out)
        wins = [pigo_b200.count_windows(r, c, *PARAMS) for _, r, c, _ in imgs]
        rows, times, model = [], [], []
        for k in (4, 8):
            first = pigo_b200.shard_plan(images, *PARAMS, angles=angles, nshards=k)
            for s in range(len(first) - 1):
                lo, hi = first[s], first[s + 1]
                sub, sa = images[lo:hi], angles[lo:hi]
                clf.RunCascadeImagesAngles(sub, cp, sa, 4096)
                t = float(np.median([timed(lambda: clf.RunCascadeImagesAngles(sub, cp, sa, 4096))[1] for _ in range(5)]))
                un = sum(wins[i] for i in range(lo, hi) if not angles[i] > 0)
                ro = sum(wins[i] for i in range(lo, hi) if angles[i] > 0)
                rows.append([un, ro, hi - lo])
                times.append(t)
                model.append((10 * un + 14 * ro + 40960 * (hi - lo)) / 10)
        ratio = np.array(times) / np.array(model)
        a, b, c = np.linalg.lstsq(np.array(rows, dtype=np.float64), np.array(times), rcond=None)[0]
        res["shards"] = [{"model_windows": int(m), "ms": round(t, 3)} for m, t in zip(model, times)]
        res["ms_per_model_window_spread"] = round(float(ratio.max() / ratio.min()), 3)
        res["fit"] = {"k_rot": round(float(b / a), 3) if a > 0 else None, "k_img_windows": round(float(c / a), 1) if a > 0 else None,
                      "ns_per_unrotated_window": round(float(a * 1e6), 5)}
    finally:
        pigo_b200.set_option("shard_split", old)
    res["multi_gpu_scaling"] = "measured" if res["devices"] > 1 else "not measured (one visible GPU: every shard shares it)"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256, help="frames of the uniform 1080p comparison")
    ap.add_argument("--pipeline-frames", type=int, default=64, help="frames of the uniform 1080p pipeline comparison")
    ap.add_argument("--sections", default="scan,pipeline", help="comma-separated: scan, pipeline, angles, decoded, formats, sharded, sweep")
    args = ap.parse_args()
    sections = set(args.sections.split(","))
    import torch
    import pigo_b200
    pigo_b200.init(0)
    clf = pigo_b200.NewPigo().Unpack(pigo_b200.load_cascade("facefinder"))
    d_frames = torch.from_numpy(make_frames(max(args.frames, args.pipeline_frames), seed0=0)).to("cuda:0")
    stream = torch.cuda.Stream(device=0)
    torch.cuda.set_stream(stream)
    res = ragged_bench(clf, 0, stream, d_frames[:args.frames], args.frames) if "scan" in sections else {}
    if "pipeline" in sections:
        res["pipeline"] = pipeline_bench(clf, 0, stream, d_frames[:args.pipeline_frames], args.pipeline_frames)
    if "angles" in sections:
        res["angles"] = angles_bench(clf, 0, stream)
    if "decoded" in sections:
        res["decoded"] = decoded_bench(clf, 0, stream)
    if "formats" in sections:
        res["formats"] = formats_bench(clf, 0, stream)
    if "sharded" in sections:
        res["sharded"] = sharded_bench(clf, 0)
    if "sweep" in sections:
        res["sweep"] = sweep_bench(clf, 0, stream)
    res["gpu"] = torch.cuda.get_device_name(0)
    try:   # read-only query: the power limit belongs beside the numbers
        import subprocess
        res["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:   # noqa: BLE001
        res["power_limit_w"] = None
    print(json.dumps(res))


if __name__ == "__main__":
    main()
