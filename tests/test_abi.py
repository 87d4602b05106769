"""CPU-side checks of the drop-in boundary: the C-ABI library builds, loads and exports every symbol
include/pigo_b200.h declares, and fails LOUDLY (no CPU fallback) when no sm_90 device is present."""
import os
import re

import numpy as np
import pytest

import pigo_b200

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "pigo_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(pigo_[a-z_0-9]+)\s*\(", src)))


def test_library_builds_and_exports_every_declared_symbol():
    from pigo_b200 import build
    so = build.build()
    assert os.path.exists(so)
    L = pigo_b200.lib()
    declared = _header_symbols()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(L, name), f"{name} declared in include/pigo_b200.h but not exported"
    assert sorted(declared) == sorted(pigo_b200.ABI_SYMBOLS)
    assert L.pigo_version() == 200


def test_host_side_ladder_matches_oracle():
    import oracle_lib as O
    for (mn, mx, sf) in [(20, 1000, 1.1), (20, 1000, 1.15), (9, 300, 1.1), (100, 99, 1.1), (1, 50, 1.0), (24, 2000, 1.33)]:
        assert pigo_b200.scale_ladder(mn, mx, sf) == O.scale_ladder(mn, mx, sf)
    for (r, c, mn, mx, sh, sf) in [(1080, 1920, 20, 1000, 0.2, 1.1), (1080, 1920, 20, 1000, 0.1, 1.1),
                                   (2160, 3840, 20, 1000, 0.2, 1.1), (400, 320, 20, 1000, 0.2, 1.1),
                                   (480, 640, 20, 1000, 0.15, 1.15), (10, 10, 20, 1000, 0.2, 1.1), (64, 48, 8, 64, 0.0, 1.2)]:
        assert pigo_b200.count_windows(r, c, mn, mx, sh, sf) == O.count_windows(r, c, mn, mx, sh, sf)
    # SURVEY.md section 8(a) figures
    assert pigo_b200.count_windows(1080, 1920, 20, 1000, 0.2, 1.1) == 894448
    assert pigo_b200.count_windows(2160, 3840, 20, 1000, 0.2, 1.1) == 3669137
    assert pigo_b200.count_windows(400, 320, 20, 1000, 0.2, 1.1) == 48015


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="this check is about the no-device behaviour")
def test_no_cpu_fallback_without_device(facefinder_bytes):
    with pytest.raises(pigo_b200.PigoError) as ei:
        pigo_b200.NewPigo().Unpack(facefinder_bytes)
    assert ei.value.status in (pigo_b200.PIGO_E_NODEVICE, pigo_b200.PIGO_E_CUDA)


def test_malformed_cascade_is_rejected_before_touching_the_device():
    with pytest.raises(pigo_b200.PigoError) as ei:
        pigo_b200.NewPigo().Unpack(b"\x00" * 8)
    assert ei.value.status == pigo_b200.PIGO_E_INVALID
    bad = bytearray(pigo_b200.load_cascade("facefinder")[:1000])
    with pytest.raises(pigo_b200.PigoError) as ei:
        pigo_b200.NewPigo().Unpack(bytes(bad))
    assert ei.value.status == pigo_b200.PIGO_E_INVALID


def test_options_round_trip_and_unknown_names():
    """pigo_set_option / pigo_get_option (no device needed): every tuning knob the docs name is readable and writable,
    unknown names are rejected, timing counters read as zero launches before anything ran."""
    names = ["scan_mode", "chunk", "gather_ctas_per_sm", "tile_max_scale", "tile_warps", "tile_ni", "gather_warps", "tile_ks",
             "gather_ks", "gather_ni", "fused_smem_kb", "tile_min_core", "tile_min_core_steps", "tile_prefetch", "gather_block",
             "deep_group", "sub_batch", "lanes", "tile_tail_min", "tile_band_ratio", "timing"]
    for n in names:
        old = pigo_b200.get_option(n)
        assert old >= 0, n
        pigo_b200.set_option(n, old + 1)
        assert pigo_b200.get_option(n) == old + 1
        pigo_b200.set_option(n, old)
    assert pigo_b200.get_option("no_such_option") == -1
    with pytest.raises(pigo_b200.PigoError):
        pigo_b200.set_option("no_such_option", 1)
    assert pigo_b200.get_option("t_tiled_n") == 0


def _split_top_level(argtext: str):
    args, depth, cur = [], 0, ""
    for ch in argtext:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
        if ch == "," and depth == 0:
            args.append(cur)
            cur = ""
        else:
            cur += ch
    if cur.strip():
        args.append(cur)
    return args


def _calls(text: str, prefix: str):
    """(name, number of top-level arguments) of every `<prefix>pigo_xxx(...)` call / prototype in text."""
    out = []
    for m in re.finditer(re.escape(prefix) + r"(pigo_[a-z_]+)\s*\(", text):
        i, depth = m.end(), 1
        while depth and i < len(text):
            depth += text[i] == "("
            depth -= text[i] == ")"
            i += 1
        body = text[m.end():i - 1].strip()
        out.append((m.group(1), 0 if body in ("", "void") else len(_split_top_level(body))))
    return out


def test_go_shim_calls_match_the_header():
    """go/pigo/pigo.go cannot be compiled here (no Go toolchain): at least every C function it calls must be declared in
    include/pigo_b200.h with the same number of arguments, so the shim cannot silently drift from the ABI."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "pigo_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    protos = dict(_calls(header, ""))
    import glob
    go = "\n".join(open(f).read() for f in sorted(glob.glob(os.path.join(root, "go", "pigo", "*.go"))))
    go = re.sub(r"//[^\n]*", "", go)
    calls = _calls(go, "C.")
    assert len(calls) >= 16
    for needed in ("pigo_rgba_to_gray", "pigo_ycbcr_to_nrgba", "pigo_detect_batch", "pigo_detect_batch_sharded", "pigo_run_cascade_batch_sharded",
                   "pigo_init_devices"):
        assert needed in dict(calls), f"the Go shim does not bind {needed}"
    for name, nargs in calls:
        assert name in protos, f"{name} is not declared in pigo_b200.h"
        assert nargs == protos[name], f"{name}: Go passes {nargs} arguments, the header declares {protos[name]}"


def test_go_shim_exports_what_the_reference_callers_use():
    """cmd/pigo/main.go:288-353 and the examples call pigo.GetImage, pigo.RgbToGrayscale, NewPigo, Unpack, RunCascade,
    ClusterDetections, NewPuplocCascade, UnpackCascade, RunDetector, ReadCascadeDir, GetLandmarkPoint: the shim package must
    export each of them (compile-drop-in), plus the additive entry points."""
    import glob
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    go = "\n".join(open(f).read() for f in sorted(glob.glob(os.path.join(root, "go", "pigo", "*.go"))))
    funcs = set(re.findall(r"^func (?:\([^)]*\) )?([A-Z][A-Za-z0-9]*)\(", go, flags=re.M))
    types = set(re.findall(r"^type ([A-Z][A-Za-z0-9]*) ", go, flags=re.M))
    for name in ("GetImage", "DecodeImage", "ImgToNRGBA", "RgbToGrayscale", "NewPigo", "Unpack", "RunCascade", "ClusterDetections", "NewPuplocCascade",
                 "UnpackCascade", "UnpackFlp", "RunDetector", "ReadCascadeDir", "GetLandmarkPoint", "RunCascadeBatch", "RunCascadeBatchSharded",
                 "DetectBatch", "InitDevices", "WireDetections"):
        assert name in funcs, name
    for name in ("CascadeParams", "ImageParams", "Detection", "Pigo", "Puploc", "PuplocCascade", "FlpCascade", "Coord", "DetectionJSON"):
        assert name in types, name
    assert "plc.Seed++" not in go and "atomic.AddUint64(&plc.seed, 1)" in go      # re-entrant like the reference (sync.Pool scratch)
    assert go.count("runtime.LockOSThread()") >= 1                                # thread-local error message fetched on the failing thread


def test_cli_json_wire_format():
    """pigo_b200/wire.py == the `pigo -json` output format (cmd/pigo/main.go:88-100): x/y swap, omitempty, accumulating points, Q > 5."""
    from pigo_b200 import Puploc, wire
    from pigo_b200.pipeline import Face
    f1 = Face((100, 200, 80, 7.5), Puploc(90, 180, 20.9, 0), Puploc(91, 0, 20.0, 0), [Puploc(120, 190, 3.7, 0), Puploc(0, 5, 1.0, 0)])
    f2 = Face((300, 40, 81, 5.0))                                            # Q == 5.0 is NOT > qThresh
    f3 = Face((50, 40, 80, 9.0))                                             # no refinements (e.g. Scale <= 50 path): inherits the points
    got = wire.marshal_wire([f1, f2, f3])
    assert got == ('[{"eyes":[{"x":180,"y":90,"size":20}],"landmark_points":[{"x":190,"y":120,"size":3}],"face":{"x":160,"y":60,"size":80}},'
                   '{"eyes":[{"x":180,"y":90,"size":20}],"landmark_points":[{"x":190,"y":120,"size":3}],"face":{"y":10,"size":80}}]')
    assert wire.marshal_wire([]) == "[]"
