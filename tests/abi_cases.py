"""Argument-error checks shared by the CPU tests of the mixed-size entry points: readers of the C header and the Go shim, one
call builder for the image-table scans and one for the pipeline calls, and the case tables every entry point runs.  Each call
passes NULL cascades unless a case gives one: the handles are validated last, so the message names the first bad argument."""
import ctypes as C
import glob
import os
import re

import numpy as np

import pigo_b200

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PIX = np.zeros(64 * 64, dtype=np.uint8)
ANG = np.array([0.0, 0.25, float("nan"), 1.3], dtype=np.float64)
FAKE = C.c_void_p(16)   # a non-NULL handle that validation never dereferences (it fails on an earlier argument)
PARAMS = (20, 1000, 0.2, 1.1)
HOST = (pigo_b200.MEM_HOST, None)


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


def calls(text: str, prefix: str):
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


def header_protos() -> dict:
    """Argument count of every function include/pigo_b200.h declares."""
    header = open(os.path.join(ROOT, "include", "pigo_b200.h")).read()
    return dict(calls(re.sub(r"/\*.*?\*/", "", header, flags=re.S), ""))


def go_source() -> str:
    """go/pigo/*.go without // comments."""
    go = "\n".join(open(f).read() for f in sorted(glob.glob(os.path.join(ROOT, "go", "pigo", "*.go"))))
    return re.sub(r"//[^\n]*", "", go)


def go_binds(go: str, name: str, protos: dict) -> bool:
    """The Go shim calls `name`, each time with the number of arguments the header declares."""
    n = [k for nm, k in calls(go, "C.") if nm == name]
    return bool(n) and all(k == protos[name] for k in n)


def go_body(go: str, fn: str) -> str:
    """The body of the Go method (pg *Pigo) fn."""
    body = go[go.index("func (pg *Pigo) %s(" % fn):]
    return body[:body.index("\n}\n")]


def descs(*geoms, pixels=PIX.ctypes.data):
    return pigo_b200.image_descs([(pixels, r, c, d) for r, c, d in geoms])


def scan(entry, images, nimages, angles=True, nangles=4, cap=4, with_n_out=True, with_out=True, det_cap=0):
    """One image-table scan entry point (pigo_run_cascade_images[_angles|_sweep|_sharded]).  Returns (status, message)."""
    L = pigo_b200.lib()
    out = np.zeros((4, max(cap, 1)), dtype=pigo_b200.DET_DTYPE)
    tag = np.zeros((4, max(cap, 1)), dtype=np.int32)
    cnt = np.zeros(4, dtype=np.int32)
    ang = ANG.ctypes.data if angles else None
    o, n = out.ctypes.data if with_out else None, cnt.ctypes.data if with_n_out else None
    args = {"pigo_run_cascade_images": (*PARAMS, 0.0, o, cap, n, *HOST),
            "pigo_run_cascade_images_angles": (ang, *PARAMS, o, cap, n, *HOST),
            "pigo_run_cascade_images_sweep": (ang, nangles, *PARAMS, 0.1, det_cap, o, tag.ctypes.data, cap, n, *HOST),
            "pigo_run_cascade_images_sharded": (ang, *PARAMS, o, cap, n),
            "pigo_run_cascade_decoded_sharded": (ang, *PARAMS, o, cap, n)}[entry]
    rc = getattr(L, entry)(None, images, nimages, *args)
    return rc, L.pigo_last_error().decode()


def detect(entry, images, nimages, angles=True, nangles=4, face=None, puploc=None, flp="default", ncalls=2, face_cap=4, prm_kw=None,
           faces=True, n_faces=True, points=True, params=True):
    """One pipeline entry point (pigo_detect_images[_angles|_sweep|_sharded], pigo_detect_decoded_sharded).  Returns (status, message)."""
    L = pigo_b200.lib()
    kw = dict(min_size=20, max_size=1000, shift_factor=0.2, scale_factor=1.1, angle=0.0, iou_threshold=0.1, min_face_scale=50,
              eye_perturbs=50, flp_perturbs=63, det_cap=0)
    kw.update(prm_kw or {})
    prm = pigo_b200.PipelineParams(**kw)
    hs = (C.c_void_p * 2)(None, None) if flp == "default" else flp
    fl = np.zeros(2, dtype=np.uint8)
    out_f = np.zeros(8 * 64, dtype=pigo_b200.DET_DTYPE)
    out_a = np.zeros(8 * 64, dtype=np.int32)
    out_n = np.zeros(8, dtype=np.int32)
    out_p = np.zeros(8 * 64 * 32, dtype=pigo_b200.POINT_DTYPE)
    ang = ANG.ctypes.data if angles else None
    p = C.byref(prm) if params else None
    f, n, pts = (out_f.ctypes.data if faces else None), (out_n.ctypes.data if n_faces else None), (out_p.ctypes.data if points else None)
    args = {"pigo_detect_images": (p, None, 0, f, face_cap, n, pts, *HOST),
            "pigo_detect_images_angles": (ang, p, None, 0, f, face_cap, n, pts, *HOST),
            "pigo_detect_images_sweep": (ang, nangles, p, None, 0, f, out_a.ctypes.data, face_cap, n, pts, *HOST),
            "pigo_detect_images_sharded": (ang, p, None, 0, f, face_cap, n, pts),
            "pigo_detect_decoded_sharded": (ang, p, None, 0, f, face_cap, n, pts)}[entry]
    rc = getattr(L, entry)(face, puploc, hs, fl.ctypes.data, ncalls, images, nimages, *args)
    return rc, L.pigo_last_error().decode()


def cases_for(shared, first=(), own=(), last=()):
    """An entry point's cases: its `first` cases, then the shared ones with each of `own` replacing the shared case of its
    label, the shared cases labelled in `last` at the end.  Cases an entry point gains come after the ones it had, so that
    each older case keeps its parametrized test id."""
    own = {c[0]: c for c in own}
    picked = [own.get(c[0], c) for c in shared]
    return list(first) + [c for c in picked if c[0] not in last] + [c for c in picked if c[0] in last]


# (label, images, nimages, keyword arguments of the builder, part of the expected message)
IMAGE_CASES = [
    ("null images", None, 2, {}, "null images"),
    ("too many images", descs((8, 8, 8)), 65536, {}, "nimages"),
    ("negative count", descs((8, 8, 8)), -1, {}, "nimages"),
    ("negative rows", descs((8, 8, 8), (-1, 8, 8)), 2, {}, "image 1: bad geometry"),
    ("dim < cols", descs((8, 9, 8)), 1, {}, "image 0: bad geometry"),
    ("rows*dim >= 2^31", descs((65536, 32768, 32768)), 1, {}, "image 0: larger than 2^31"),
    ("negative capacity", descs((8, 8, 8)), 1, {"cap": -1}, "negative capacity"),
    ("null n_out", descs((8, 8, 8)), 1, {"with_n_out": False}, "null n_out"),
    ("null pixels", descs((8, 8, 8), pixels=None), 1, {}, "image 0: null pixels"),
    ("null out", descs((8, 8, 8)), 1, {"with_out": False}, "null out"),
]

PIPELINE_CASES = [
    ("too many images", descs((8, 8, 8)), 65536, {}, "nimages"),
    ("negative count", descs((8, 8, 8)), -1, {}, "nimages"),
    ("null images", None, 2, {}, "null images"),
    ("null params", descs((8, 8, 8)), 1, {"params": False}, "null params"),
    ("null faces", descs((8, 8, 8)), 1, {"faces": False}, "null faces"),
    ("null n_faces", descs((8, 8, 8)), 1, {"n_faces": False}, "null n_faces"),
    ("null points", descs((8, 8, 8)), 1, {"points": False}, "null points"),
    ("ncalls > 30", descs((8, 8, 8)), 1, {"ncalls": 31}, "ncalls"),
    ("negative ncalls", descs((8, 8, 8)), 1, {"ncalls": -1}, "ncalls"),
    ("null flp", descs((8, 8, 8)), 1, {"flp": None}, "null flp"),
    ("face_cap 0", descs((8, 8, 8)), 1, {"face_cap": 0}, "face_cap"),
    ("face_cap 4097", descs((8, 8, 8)), 1, {"face_cap": 4097}, "face_cap"),
    ("eye perturbs", descs((8, 8, 8)), 1, {"prm_kw": {"eye_perturbs": 64}}, "Perturbs"),
    ("flp perturbs", descs((8, 8, 8)), 1, {"prm_kw": {"flp_perturbs": -1}}, "Perturbs"),
    ("pupil work > 2^31-1", descs((8, 8, 8)), 65535, {"face_cap": 4096, "ncalls": 30}, "exceeds 2^31-1"),
    ("zero rows", descs((8, 8, 8), (0, 8, 8)), 2, {}, "image 1: bad geometry"),
    ("zero cols", descs((8, 0, 8)), 1, {}, "image 0: bad geometry"),
    ("dim < cols", descs((8, 9, 8)), 1, {}, "image 0: bad geometry"),
    ("rows*dim >= 2^31", descs((65536, 32768, 32768)), 1, {}, "image 0: larger than 2^31"),
    ("null pixels", descs((8, 8, 8), pixels=None), 1, {}, "image 0: null pixels"),
    ("null pupil cascade", descs((8, 8, 8)), 1, {"face": FAKE}, "null pupil cascade"),
    ("null landmark cascade", descs((8, 8, 8)), 1, {"face": FAKE, "puploc": FAKE, "flp": (C.c_void_p * 2)(FAKE, None)}, "null landmark cascade 1"),
]
# the pipeline cases the angle and sweep pipelines run after their older ones
LATER_PIPELINE_CASES = ("negative ncalls", "face_cap 4097", "flp perturbs", "zero cols", "dim < cols", "rows*dim >= 2^31")
