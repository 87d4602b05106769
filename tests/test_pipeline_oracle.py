"""CPU check of tests/pipeline_oracle.py: the replay accepts outputs that follow the oracle step by step and rejects them when
one field of one landmark point changes."""
import numpy as np
import pytest

import pipeline_oracle as P

TEST_PARAMS = (20, 1000, 0.2, 1.1)   # core/pigo_test.go:44-50


def test_replay_accepts_the_oracle_outputs_and_rejects_one_changed_field(oracle_face, sample_gray):
    oracle = P.oracle_cascades()
    image = (sample_gray, 400, 320, 320)
    cl = P.oracle_clusters(oracle_face, image, TEST_PARAMS, 0.0)
    rnd = np.random.default_rng(3).random((1, len(cl), 17, 63, 3), dtype=np.float32)
    points = P.oracle_points(oracle, image, cl, 0.0, lambda k, slot: rnd[0, k, slot], 50)[None]
    got = (cl[None], np.array([len(cl)]), points)
    cases = [(0, image, cl, 0.0)]
    assert P.replay(oracle, cases, lambda i, k, slot: rnd[i, k, slot], 50, got) == (1, 0)
    k = int(np.flatnonzero(cl["scale"] > 50)[0])
    for field in ("row", "col", "scale"):
        points[field][0, k, 9] += 1
        with pytest.raises(AssertionError):
            P.replay(oracle, cases, lambda i, k, slot: rnd[i, k, slot], 50, got)
        points[field][0, k, 9] -= 1
