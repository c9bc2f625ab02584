"""capi.Context.heading_enqueue checks the shapes of its arrays before they reach the library, which reads
offsets[-1] points and one request per trajectory: a mismatch raises ValueError and calls nothing."""
import types

import numpy as np
import pytest

import pyoracle_heading as H
from densesurfelmapping_b200 import capi
from planner_scenes import rotations


def test_mismatched_arrays_raise_before_the_call():
    calls = []
    stub = types.SimpleNamespace(h=None, lib=types.SimpleNamespace(dsm_heading_enqueue=lambda *a: calls.append(a) or 0),
                                 _ck=lambda rc: None)
    pts = np.zeros((16, 3))
    cam = (10.0, 10.0, 5.0, 5.0, 10, 10, 1.0, 1)
    rot = rotations(8)
    two = H.requests([(0, -1, 1), (1, 2, 1)])
    for points, offsets, req in ((pts, [0, 8, 16], H.requests([(0, -1, 1)])),   # one request for two trajectories
                                 (pts, [0, 8], two),                              # two for one
                                 (pts[:10], [0, 8, 16], two),                     # offsets beyond the points
                                 (pts, [0], H.requests([]))):                     # no trajectory
        with pytest.raises(ValueError):
            capi.Context.heading_enqueue(stub, points, offsets, cam, rot, 4, req, 1, 1)
    assert not calls
    capi.Context.heading_enqueue(stub, pts, [0, 8, 16], cam, rot, 4, two, 1, 1)
    capi.Context.heading_enqueue(stub, pts, [0, 8, 16], cam, rot, 4, [(0, -1, 1), (1, 2, 1)], 1, 1)   # plain rows
    assert len(calls) == 2
    assert capi.HEADING_REQUEST_DTYPE == H.REQUEST_DTYPE and capi.HEADING_DTYPE == H.RECORD_DTYPE
    assert capi.HEADING_SAMPLE_DTYPE == H.SAMPLE_DTYPE and capi.HEADING_COUNT_DTYPE == H.COUNT_DTYPE
    assert capi.HEADING_INFO_DTYPE == H.INFO_DTYPE
