"""Synthetic pupil / landmark cascades, the library's perturbation generator and the launch plan of the RunDetector kernels,
restated on the host: the fixtures of tests/test_puploc_plan_cpu.py and tests/test_puploc_fuzz_gpu.py.

The plan restates `launch_puploc_pairs` (pigo_b200/csrc/puploc.cu): which kernel a launch runs, whether the stage's node codes
are staged in shared memory, the pixel patch's byte cap, and for every stage whether `load_patch` accepts the bounding box of
the perturbations' sample areas.  The per-stage states come from the C oracle run on the cascade's first k stages."""
import struct

import numpy as np

import oracle_lib as O

M64 = (1 << 64) - 1
RNG_MUL = 0xD1342543DE82EF95
SMEM_BUDGET = 110 * 1024      # launch_puploc_pairs: kBudget
LEAF_LIMIT = 100 * 1024       # 63 * trees * 8 bytes of leaves above this: the pair kernel does not run
PATCH_MAX = 48 * 1024
QCOS = [256, 251, 236, 212, 181, 142, 97, 49, 0, -49, -97, -142, -181, -212, -236, -251, -256,
        -251, -236, -212, -181, -142, -97, -49, 0, 49, 97, 142, 181, 212, 236, 251, 256]
QSIN = [0, 49, 97, 142, 181, 212, 236, 251, 256, 251, 236, 212, 181, 142, 97, 49, 0,
        -49, -97, -142, -181, -212, -236, -251, -256, -251, -236, -212, -181, -142, -97, -49, 0]


# ---- cascades -----------------------------------------------------------------------------------------------------------
def puploc_cascade(depth: int, trees: int, stages: int, scales: float, seed: int, pred: float = 0.03, nan_leaves: float = 0.0) -> bytes:
    """A random cascade in the puploc layout (core/puploc.go:38-103): <u32 stages, f32 scales, u32 trees, u32 depth>, then
    per stage and tree 4*2^depth - 4 int8 codes and 2*2^depth float32 predictions.  Codes are uniform int8 with -128 made
    common (its negation wraps under flipV); predictions are uniform in [-pred, pred), small enough that the refined points
    stay near the seed while every tree still moves them; a fraction `nan_leaves` of them is NaN."""
    rng = np.random.default_rng(seed)
    L = 1 << depth
    out = bytearray(struct.pack("<IfII", stages, scales, trees, depth))
    for _ in range(stages * trees):
        codes = rng.integers(-128, 128, size=4 * L - 4, dtype=np.int16)
        codes[rng.random(codes.size) < 0.05] = -128
        preds = rng.uniform(-pred, pred, size=2 * L).astype("<f4")
        if nan_leaves:
            preds[rng.random(preds.size) < nan_leaves] = np.nan
        out += codes.astype(np.int8).tobytes() + preds.tobytes()
    return bytes(out)


def header(packet: bytes):
    """(stages, scales, trees, depth) of a puploc packet."""
    st, sc, tr, dp = struct.unpack_from("<IfII", packet)
    return st, np.float32(sc), tr, dp


def first_stages(packet: bytes, k: int) -> bytes:
    """The cascade made of the first k stages of `packet`: running it gives the state a perturbation enters stage k with."""
    st, sc, tr, dp = struct.unpack_from("<IfII", packet)
    L = 1 << dp
    per = 4 * L - 4 + 8 * L
    return struct.pack("<IfII", k, sc, tr, dp) + packet[16:16 + k * tr * per]


# ---- the library generator ----------------------------------------------------------------------------------------------
def mix64(x: int) -> int:
    """puploc.cu mix64: splitmix64's finaliser, the top 24 bits."""
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    x ^= x >> 31
    return x >> 40


def library_randoms(rng_seed: int, slot: int) -> np.ndarray:
    """[63][3] float32 draws of RunDetector call `slot` when no randoms are given: key = rng_seed * RNG_MUL + slot * 64 + i
    for perturbation i, draw k = mix64(3 * key + k) / 2^24.  `slot` is the seed index of a standalone call (both kernels) and
    slot + slot_base in the pipeline (its slot layout: [image][face_cap][2 + ncalls])."""
    out = np.zeros((63, 3), dtype=np.float32)
    for i in range(63):
        key = (rng_seed * RNG_MUL + slot * 64 + i) & M64
        for k in range(3):
            out[i, k] = np.float32(mix64((key * 3 + k) & M64)) * np.float32(1.0 / 16777216.0)
    return out


# ---- launch plan --------------------------------------------------------------------------------------------------------
def pair_launch(shapes, puploc_stage: int):
    """launch_puploc_pairs for a launch whose positions use cascades of `shapes` [(trees, depth)]: None when the pair kernel
    does not run (63 * trees * 8 B of leaves over 100 KB), else (staged, patch_cap)."""
    trees_max = max(t for t, _ in shapes)
    codes_max = max(t * (4 * (1 << d) + 8) for t, d in shapes)
    leaf = (63 * trees_max * 8 + 15) & ~15
    if leaf > LEAF_LIMIT:
        return None
    codes_max = (codes_max + 15) & ~15
    staged = puploc_stage != 0 and leaf + codes_max <= SMEM_BUDGET
    patch = 0
    if staged and puploc_stage >= 2 and leaf + codes_max + 4096 <= SMEM_BUDGET:
        patch = min(PATCH_MAX, SMEM_BUDGET - leaf - codes_max)
    return staged, patch


def growth(stages: int, scales: float) -> float:
    return max(1.0, abs(float(scales))) ** (stages - 1) if stages > 1 else 1.0


def standalone_kernel(packet: bytes, seed_scales, puploc_mode: int):
    """Which kernel a standalone RunDetector call runs: "warp" (puploc_kernel) when option puploc_mode is 1, when the pair
    kernel cannot hold the cascade's leaves, or when a seed leaves its 32-bit envelope (|Scale| * growth > 16384); else "pair"."""
    st, sc, tr, dp = header(packet)
    g = growth(st, sc)
    if puploc_mode == 1 or pair_launch([(tr, dp)], 1) is None or any(abs(float(np.float32(s))) * g > 16384.0 for s in seed_scales):
        return "warp"
    return "pair"


def _i32(v) -> int:
    """(int) of a float on the device: truncation, saturated, NaN -> 0."""
    v = float(v)
    if v != v:
        return 0
    return int(min(max(v, -2.0 ** 31), 2.0 ** 31 - 1))


def _llround_i32(v) -> int:
    """(int)llround((double)s): half away from zero, then the low 32 bits as a signed int."""
    v = float(v)
    if v != v or abs(v) >= 2.0 ** 63:
        return 0
    t = int(abs(v) + 0.5) if abs(v) - int(abs(v)) >= 0.5 else int(abs(v))
    t = t if v >= 0 else -t
    t &= 0xFFFFFFFF
    return t - (1 << 32) if t >= 1 << 31 else t


def perturbations(seed, randoms):
    """The perturbations' initial (r, c, s) of one seed (core/puploc.go:248-250, float32)."""
    f32 = np.float32
    row, col, scale, P = seed
    out = []
    for i in range(min(P, 63)):
        t1 = f32(f32(scale) * f32(0.15))
        r = f32(f32(row) + f32(t1 * f32(f32(0.5) - randoms[i, 0])))
        c = f32(f32(col) + f32(t1 * f32(f32(0.5) - randoms[i, 1])))
        s = f32(f32(scale) * f32(f32(0.925) + f32(f32(0.15) * randoms[i, 2])))
        out.append((r, c, s))
    return out


def patch_stages(packet: bytes, seed, randoms, image, angle: float, flip: bool, patch_cap: int, aligned: bool, margin: int = 2):
    """(patch, global) stage counts of one pair-kernel call with a pixel patch of `patch_cap` bytes (load_patch): before every
    stage the box of all perturbations' int(r), int(c) +- h, h = |Round(s)|/2 + 2 unrotated and (|iqs| + |iqc|)/512 + 2 rotated
    (iqs, iqc from the initial scale), is clamped to the image, its first column rounded down to 16, and the patch is used
    when rows * pitch (a multiple of 16 >= the width) fits the cap and the image's pitch and base are 16-byte aligned.
    `margin` is the kernel's + 2; a test passes 1 to find boxes whose acceptance depends on it."""
    st, sc, tr, dp = header(packet)
    pixels, rows, cols, dim = image
    P = min(seed[3], 63)
    if patch_cap == 0 or P == 0:
        return 0, st
    slot = int(32.0 * min(angle, 1.0)) if angle > 0 else -1
    init = perturbations(seed, randoms)
    q = [(_i32(np.float32(s * np.float32(QSIN[slot]))), _i32(np.float32(s * np.float32(QCOS[slot])))) if slot >= 0 else (0, 0)
         for _, _, s in init]
    state = init
    patch = 0
    for k in range(st):
        if k > 0:
            pre = O.OraclePuploc(first_stages(packet, k))
            state = [pre.classify(r, c, s, pixels, rows, cols, dim, angle, flip) for r, c, s in init]
        box = [2 ** 31 - 1, -2 ** 31, 2 ** 31 - 1, -2 ** 31]
        for (r, c, s), (iqs, iqc) in zip(state, q):
            ir = max(-(1 << 30), min(1 << 30, _i32(r)))
            ic = max(-(1 << 30), min(1 << 30, _i32(c)))
            h = ((abs(iqs) + abs(iqc)) >> 9) + margin if slot >= 0 else (abs(_llround_i32(s)) >> 1) + margin
            box = [min(box[0], ir - h), max(box[1], ir + h), min(box[2], ic - h), max(box[3], ic + h)]
        r0, r1 = min(max(box[0], 0), rows - 1), min(max(box[1], 0), rows - 1)
        c0, c1 = min(max(box[2], 0), cols - 1) & ~15, min(max(box[3], 0), cols - 1)
        nrows, pitch = r1 - r0 + 1, (c1 - c0 + 16) & ~15
        patch += nrows > 0 and pitch > 0 and nrows * pitch <= patch_cap and aligned and dim % 16 == 0
    return patch, st - patch
