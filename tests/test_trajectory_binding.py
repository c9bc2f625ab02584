"""capi.Context.trajectory_enqueue checks the shapes of its arrays before they reach the library, which reads
offsets[-1] points and one knot interval per trajectory: a mismatch raises ValueError and calls nothing."""
import types

import numpy as np
import pytest

import pyoracle_trajectory as tj
from densesurfelmapping_b200 import capi


def test_mismatched_arrays_raise_before_the_call():
    calls = []
    stub = types.SimpleNamespace(h=None, lib=types.SimpleNamespace(dsm_trajectory_enqueue=lambda *a: calls.append(a) or 0),
                                 _ck=lambda rc: None)
    pts = np.zeros((16, 3))
    p = tj.params()
    for points, offsets, dt in ((pts, [0, 8, 16], [1.0]),          # one dt for two trajectories
                                (pts, [0, 8], [1.0, 1.0]),         # two for one
                                (pts[:10], [0, 8, 16], [1.0, 1.0]),  # offsets beyond the points
                                (pts, [0], [])):                   # no trajectory
        with pytest.raises(ValueError):
            capi.Context.trajectory_enqueue(stub, points, offsets, dt, p)
    assert not calls
    capi.Context.trajectory_enqueue(stub, pts, [0, 8, 16], [1.0, 1.0], p)
    assert len(calls) == 1
