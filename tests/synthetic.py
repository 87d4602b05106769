"""A random cascade in the facefinder binary layout, for tests of tree depths and sizes other than facefinder's."""
import numpy as np


def synthetic_cascade(depth: int, ntrees: int, seed: int) -> bytes:
    """A random cascade in the facefinder binary layout (core/pigo.go:51-110), thresholds loose enough to let windows through."""
    rng = np.random.default_rng(seed)
    L = 1 << depth
    out = bytearray(b"\x03\x00\x00\x00\x81\x7f\x81\x7f")
    out += np.uint32(depth).tobytes() + np.uint32(ntrees).tobytes()
    for t in range(ntrees):
        out += rng.integers(-128, 128, size=4 * L - 4, dtype=np.int8).tobytes()
        out += rng.uniform(-1.0, 1.0, size=L).astype("<f4").tobytes()
        out += np.float32(-0.6 - 0.25 * t).tobytes()
    return bytes(out)
