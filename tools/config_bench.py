#!/usr/bin/env python
"""Measures the BASELINE.json configs that are parity-test cases rather than the bench line (written to
profiles/configs_r01.json): configs[3] 3840x2160 rotated sweep (classifyRotatedRegion path) and configs[4] the
face -> cluster -> pupils -> landmarks pipeline, plus the RgbToGrayscale kernel (section 8f N2).  Device-resident
inputs, CUDA events on the launching stream."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pigo_b200  # noqa: E402
from pigo_b200 import CascadeParams, ImageParams, pipeline, synth  # noqa: E402


def timed(fn, reps, stream):
    fn(); torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream); fn(); b.record(stream); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    pigo_b200.init(0)
    clf = pigo_b200.NewPigo().Unpack(pigo_b200.load_cascade("facefinder"))
    stream = torch.cuda.Stream(); torch.cuda.set_stream(stream); st = stream.cuda_stream
    out = {}
    # ---- configs[3]: 4K frames, rotated path, table slots k/32
    R, C = 2160, 3840
    nf = 8
    frames = np.stack([synth.frame_faces(None, R, C, shift=(31 * i, 17 * i), noise_seed=i) for i in range(nf)])
    d = torch.from_numpy(frames).cuda()
    cap = 4096
    d_out = torch.zeros((nf, cap, 4), dtype=torch.int32, device="cuda"); d_cnt = torch.zeros(nf, dtype=torch.int32, device="cuda")
    W4k = pigo_b200.count_windows(R, C, 20, 1000, 0.2, 1.1)
    rot = {}
    for k in (0, 4, 8, 16, 27, 32):
        ms = timed(lambda: clf.run_cascade_batch_device(d.data_ptr(), nf, R * C, R, C, C, 20, 1000, 0.2, 1.1, k / 32.0, d_out.data_ptr(), cap,
                                                       d_cnt.data_ptr(), st), 3, stream)
        rot[f"angle_{k}_32"] = {"ms_per_8_frames": ms, "windows_per_s": nf * W4k / (ms * 1e-3), "detections": int(d_cnt.sum())}
    out["configs3_4k_rotated"] = {"frames": nf, "windows_per_frame": W4k, "by_angle": rot,
                                  "note": "angle 0 = unrotated fused path; angle > 0 = scan_gather_kernel<6,true> (64-bit coordinate math, nrows-1 clamp quirk)"}
    # ---- configs[4]: full pipeline on 1080p class-F frames through the host API
    plc = pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("puploc"))
    names = sorted(set(pipeline.EYE_CASCADES + pipeline.MOUTH_CASCADES))
    flp = {n: pigo_b200.NewPuplocCascade().UnpackCascade(pigo_b200.load_cascade("lps/" + n)) for n in names}
    nfp = 64
    fr = np.stack([synth.frame_faces(None, 1080, 1920, shift=(37 * i, 53 * i), noise_seed=100 + i) for i in range(nfp)])
    cp = CascadeParams(ImageParams(None, 1080, 1920, 1920), 20, 1000, 0.2, 1.1)
    pipeline.detect_batch(clf, plc, flp, fr, cp)   # warm-up: buffers, plans
    dts = []
    for _ in range(3):
        t0 = time.perf_counter()
        res = pipeline.detect_batch(clf, plc, flp, fr, cp)
        dts.append(time.perf_counter() - t0)
    dt = min(dts)
    nfaces = sum(1 for f in res for face in f if face.left_eye is not None)
    out["configs4_pipeline_host_api"] = {"frames": nfp, "seconds": dt, "frames_per_s": nfp / dt, "faces_with_landmarks": nfaces,
                                         "landmark_points": sum(len(face.landmarks) for f in res for face in f),
                                         "note": "frames uploaded once; batched RunCascade + ClusterDetections, one RunDetector launch for all eye seeds and "
                                                 "one per landmark cascade for all frames (host sequencing only between the ~12 launches)"}
    # ---- RgbToGrayscale (N2), device resident, HBM-bound streaming kernel: 5 B/pixel
    npx = 64 * 1080 * 1920
    rgba = torch.randint(0, 256, (npx, 4), dtype=torch.uint8, device="cuda"); gray = torch.empty(npx, dtype=torch.uint8, device="cuda")
    L = pigo_b200.lib()
    ms = timed(lambda: L.pigo_rgba_to_gray(rgba.data_ptr(), npx, gray.data_ptr(), 3, st), 5, stream)
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
    gbs = 5 * npx / (ms * 1e-3) / 1e9
    out["rgb_to_grayscale"] = {"pixels": npx, "ms": ms, "GBps": gbs, "frac_of_measured_hbm": gbs / peaks.get("hbm_gbs", 3350.0)}
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, "gpurun_out", "configs_r01.json"), "w"), indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
