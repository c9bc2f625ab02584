"""The slot order of SurfelMap::fuse_map's post-step (surfel_map.cpp:1077-1109) as the resident pool's k_pool_recycle
computes it in parallel (csrc/dsm_kernels.cu), restated in numpy and pinned to pyoracle.fuse_map_poststep -- the C
restatement that tests/test_refmap.py pins byte for byte to the reference's own fuse_map.

The restatement follows the kernel step by step: the ascending hole list, the fill, then the tail offsets t < q = m - K
(hole d_t reads position N' + t), each either resolved (its own surfel, or a new surfel when it is a filled hole) or a
pointer to the tail offset s of the leftover hole d_s it is; pointer doubling inside segments of `seg` offsets and an
ordered pass over the segments from the top down.  Small segments make the cross-segment path run in small cases."""
import itertools

import numpy as np
import pytest

import pyoracle
from densesurfelmapping_b200.elements import SURFEL_DTYPE


def recycle_sources(dead, K, seg=1024):
    """Source of every slot of the new pool: v < N is old slot v, v >= N is new surfel v - N."""
    dead = np.asarray(dead, bool)
    N = len(dead)
    holes = np.flatnonzero(dead)
    m = len(holes)
    Np = N - m + K
    res = np.arange(max(N, Np), dtype=np.int64)
    k = np.arange(min(K, m))
    h = holes[m - 1 - k]
    res[h[h < Np]] = N + k[h < Np]                       # fill; a filled hole >= N' is read by the tail
    res[N:Np] = N + np.arange(m, K)                      # append (K > m)
    q = m - K
    if q > 0:
        t = np.arange(q)
        p = Np + t
        i = np.searchsorted(holes, p)                    # rank of p among the holes, where p is one
        v = np.where(~dead[p], -1 - p, np.where(i >= q, -1 - (N + m - 1 - i), np.where(i == t, -1 - p, i)))
        src = np.zeros(q, np.int64)
        rounds = int(np.log2(seg))
        assert 1 << rounds == seg
        for sg in range((q + seg - 1) // seg - 1, -1, -1):   # ticket order: the top segment first
            t0, t1 = sg * seg, min(q, sg * seg + seg)
            sv = v[t0:t1].copy()
            for _ in range(rounds):
                inside = (sv >= 0) & (sv < t0 + seg)
                nv = sv.copy()
                nv[inside] = sv[sv[inside] - t0]
                sv = nv
            up = sv >= 0
            assert (sv[up] >= t1).all()                  # what is left points above the segment: already resolved
            sv[up] = src[sv[up]]
            src[t0:t1] = sv
        assert (src < 0).all()
        fin = holes[:q] < Np
        res[holes[:q][fin]] = -1 - src[fin]
    return res[:Np]


def tagged(dead, K, rng=None):
    """A pool whose slot i has last_update = i (update_times 0 where dead) and K new surfels tagged N + k."""
    N = len(dead)
    local = np.zeros(N, SURFEL_DTYPE)
    local["last_update"] = np.arange(N)
    local["update_times"] = np.where(dead, 0, 1 + np.arange(N) % 7)
    new = np.zeros(K, SURFEL_DTYPE)
    new["last_update"] = N + np.arange(K)
    new["update_times"] = 1
    if rng is not None:
        for a in (local, new):
            for f in ("px", "py", "pz", "nx", "ny", "nz", "color", "weight", "size"):
                a[f] = rng.standard_normal(len(a)).astype(np.float32)
    return local, new


def check(dead, K, seg=1024, rng=None):
    local, new = tagged(dead, K, rng)
    want = pyoracle.fuse_map_poststep(local, new)
    src = recycle_sources(dead, K, seg)
    assert np.array_equal(want["last_update"], src), (np.flatnonzero(dead), K, seg)
    assert np.concatenate([local, new])[src].tobytes() == want.tobytes()


def test_every_flag_pattern_up_to_12():
    """Every dead-flag pattern of N <= 12 surfels, K in [0, N + 2], with one-offset and four-offset segments."""
    for N in range(0, 13):
        for bits in range(1 << N):
            dead = np.array([(bits >> i) & 1 for i in range(N)], bool)
            local, _ = tagged(dead, 0)
            for K in range(N + 3):
                _, new = tagged(dead, K)
                want = pyoracle.fuse_map_poststep(local, new)["last_update"]
                for seg in (1, 4, 1024):
                    assert np.array_equal(recycle_sources(dead, K, seg), want), (N, bits, K, seg)


def test_tail_counterexample():
    """N = 5, slots 0-2 dead, K = 0: e4 goes 4 -> 2 -> 0, so the pool is [e4, e3] (pairing the occupied tail positions
    with the holes below N' in descending order would give [e3, e4])."""
    dead = np.array([1, 1, 1, 0, 0], bool)
    assert list(recycle_sources(dead, 0)) == [4, 3]
    check(dead, 0)


@pytest.mark.parametrize("seg", [4, 1024])
def test_longest_chain(seg):
    """One live surfel on top of a run of holes: its chain visits q - 1 leftover holes."""
    for q in (2, 3, 17, 1024, 1025, 5000):
        dead = np.ones(q + 1, bool)
        dead[-1] = False
        src = recycle_sources(dead, 0, seg)
        assert list(src) == [q]
        check(dead, 0, seg)
        for K in (0, 1, q // 2):
            check(np.concatenate([np.zeros(7, bool), dead]), K, seg)


@pytest.mark.parametrize("case", ["none_dead", "all_dead", "tail_only", "m_much_larger", "k_much_larger", "k_zero"])
def test_random_pools(case):
    rng = np.random.default_rng(sum(map(ord, case)))
    for N in (1, 300, 4000, 200_000):
        if case == "none_dead":
            dead, K = np.zeros(N, bool), int(rng.integers(0, 3000))
        elif case == "all_dead":
            dead, K = np.ones(N, bool), int(rng.integers(0, min(N, 3000) + 1))
        elif case == "tail_only":
            dead = np.zeros(N, bool)
            dead[N - int(rng.integers(1, N + 1) * 0.1) - 1:] = True
            K = int(rng.integers(0, dead.sum() + 1))
        elif case == "m_much_larger":   # as after a large retire
            dead, K = rng.random(N) < 0.6, int(rng.integers(0, 20))
        elif case == "k_much_larger":
            dead, K = rng.random(N) < 0.002, int(rng.integers(50, 3000))
        else:
            dead, K = rng.random(N) < rng.random(), 0
        for seg in (64, 1024):
            check(dead, K, seg, rng if N <= 4000 else None)


def test_against_the_reference_node():
    """RefMap.set_local + the node's own fuse_map on a crafted pool: its slots are what the restatement says."""
    if not pyoracle.have_refmap():
        pytest.skip("the reference node library is not built")
    from densesurfelmapping_b200 import synth
    cam = synth.VGA
    rng = np.random.default_rng(5)
    for t, frac in enumerate((0.0, 0.3, 0.9)):
        pose = synth.pose_stream(t)
        gray, depth = synth.make_frame(cam, 700 + t, pose)
        orc = pyoracle.RefSerial(cam) if pyoracle.have_reference() else pyoracle.Restatement(cam)
        local, _ = tagged(rng.random(3000) < frac, 0, rng)
        local["update_times"] = np.where(local["update_times"] == 0, 0, 1000)   # keep them out of the unstable-removal rule
        local["px"], local["py"], local["pz"] = 0.0, 0.0, -5.0                    # behind the camera: not fused
        lo, no = orc.fuse(t, gray, depth, pose, local)
        m = pyoracle.RefMap(cam)
        m.set_local(local)
        m.fuse_map(gray, depth, pose, t)
        got = m.local()
        m.close()
        dead = lo["update_times"] == 0
        src = recycle_sources(dead, len(no))
        assert got.tobytes() == np.concatenate([lo, no])[src].tobytes()
