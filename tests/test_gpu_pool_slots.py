"""The resident pool in the reference's slot order: after dsm_fuse_frame_resident and every frame of
dsm_fuse_stream_resident the pool is, slot for slot, the local_surfels that SurfelMap::fuse_map leaves
(surfel_map.cpp:1077-1109).  Given the same fuse results it is byte-identical: the product's own fuse output
(dsm_fuse_frame, the same kernels) followed by pyoracle.fuse_map_poststep is the expectation."""
import numpy as np
import pytest

import pyoracle
from densesurfelmapping_b200 import synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from util import check_surfels

pytestmark = pytest.mark.gpu

CAM = synth.VGA


def frame(t, seed=800):
    pose = synth.pose_stream(t)
    gray, depth = synth.make_frame(CAM, seed + t, pose)
    return gray, depth, pose


def base_pool(ctx, frames=3):
    """A real pool: `frames` frames of the product's fuse plus the restated post-step."""
    pool = np.zeros(0, SURFEL_DTYPE)
    for t in range(frames):
        gray, depth, pose = frame(t)
        lo, no = ctx.fuse_frame(t, gray, depth, pose, pool)
        pool = pyoracle.fuse_map_poststep(lo, no)
    return pool


def craft(pool, case):
    """Dead-slot patterns (update_times = 0) that force the different shapes of the post-step."""
    p = pool.copy()
    N = len(p)
    i = np.arange(N)
    if case == "holes_low_and_high":      # K < m: holes below N' and inside the tail
        dead = (i < 0.45 * N) | ((i > 0.8 * N) & (i % 3 == 0))
    elif case == "long_chain":            # K < m: one live surfel on top of a long run of holes
        dead = (i >= 0.3 * N) & (i < N - 1)
    elif case == "few_holes":             # K > m: every hole is filled, the rest is appended
        dead = i % 997 == 5
    else:
        raise ValueError(case)
    p["update_times"][dead] = 0
    return p


def expect(ctx, ref, gray, depth, pose, pool):
    lo, no = ctx.fuse_frame(ref, gray, depth, pose, pool)
    return lo, no, pyoracle.fuse_map_poststep(lo, no)


def resident(ctx, pool, ref, gray, depth, pose):
    ctx.pool_upload(pool)
    n_new = ctx.fuse_frame_resident(ref, gray, depth, pose, want_count=True)
    return n_new, ctx.pool_download()


@pytest.fixture(scope="module")
def ctx():
    from densesurfelmapping_b200 import capi
    c = capi.Context(CAM, max_batch=8, max_local_surfels=200000)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pool(ctx):
    return base_pool(ctx)


def test_byte_exact_on_both_frame_slots(ctx, pool):
    for t in range(3, 7):                  # alternating frame slots 0 / 4 (the first slot of each staging half)
        gray, depth, pose = frame(t)
        lo, no, want = expect(ctx, t, gray, depth, pose, pool)
        n_new, got = resident(ctx, pool, t, gray, depth, pose)
        assert n_new == len(no)
        assert got.tobytes() == want.tobytes(), f"frame {t}"
        pool = want


def test_byte_exact_over_a_stream_with_a_reference_jump(ctx):
    pool = np.zeros(0, SURFEL_DTYPE)
    killed = 0
    for t in range(6):
        ref = t // 2 + (9 if t >= 4 else 0)   # the jump kills unstable surfels
        gray, depth, pose = frame(t, 900)
        lo, no, want = expect(ctx, ref, gray, depth, pose, pool)
        killed += int((lo["update_times"] == 0).sum())
        _, got = resident(ctx, pool, ref, gray, depth, pose)
        assert got.tobytes() == want.tobytes(), f"frame {t}"
        pool = want
    assert killed > 0


@pytest.mark.parametrize("case", ["holes_low_and_high", "long_chain", "few_holes"])
def test_byte_exact_on_crafted_holes(ctx, pool, case):
    p = craft(pool, case)
    gray, depth, pose = frame(3)
    lo, no, want = expect(ctx, 3, gray, depth, pose, p)
    m, K = int((lo["update_times"] == 0).sum()), len(no)
    assert (K > m) if case == "few_holes" else (K < m), (K, m)
    if case != "few_holes":
        Np = len(lo) - m + K
        holes = np.flatnonzero(lo["update_times"] == 0)
        assert (holes[:m - K] < Np).any() and (holes >= Np).any()
    _, got = resident(ctx, p, 3, gray, depth, pose)
    assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize("chunk", [1, 3, 4])
def test_stream_chunks_equal_frame_by_frame_on_crafted_pools(ctx, pool, chunk):
    from densesurfelmapping_b200 import capi
    frames = [(3 + t,) + frame(3 + t) for t in range(8)]
    for case in ("holes_low_and_high", "long_chain", "few_holes"):
        p = craft(pool, case)
        ctx.pool_upload(p)
        for r, g, d, ps in frames:
            ctx.fuse_frame_resident(r, g, d, ps)
        want = ctx.pool_download()
        b = capi.Context(CAM, max_batch=8, max_local_surfels=200000)
        b.pool_upload(p)
        for i in range(0, len(frames), chunk):
            part = frames[i:i + chunk]
            b.fuse_stream_resident([f[0] for f in part], np.stack([f[1] for f in part]), np.stack([f[2] for f in part]),
                                   np.stack([f[3] for f in part]))
        got = b.pool_download()
        b.close()
        assert got.tobytes() == want.tobytes(), case


def test_retired_slots_are_recycled_by_the_next_frame(ctx, pool):
    gray, depth, pose = frame(3)
    # pool_retire
    loc, out = pyoracle.retire(pool, 1)
    assert len(out) > 0
    lo, no, want = expect(ctx, 3, gray, depth, pose, loc)
    ctx.pool_upload(pool)
    assert ctx.pool_retire(1).tobytes() == out.tobytes()
    ctx.fuse_frame_resident(3, gray, depth, pose)
    assert ctx.pool_download().tobytes() == want.tobytes()
    # inactive_retire, of two keyframes
    loc1, _ = pyoracle.retire(pool, 1)
    loc0, _ = pyoracle.retire(loc1, 0)
    lo, no, want = expect(ctx, 3, gray, depth, pose, loc0)
    assert (lo["update_times"] == 0).sum() > len(no)
    ctx.pool_upload(pool)
    ctx.inactive_reserve(2 * len(pool))
    assert ctx.inactive_retire(1) > 0 and ctx.inactive_retire(0) > 0
    ctx.fuse_frame_resident(3, gray, depth, pose)
    assert ctx.pool_download().tobytes() == want.tobytes()


def test_against_the_reference_node():
    """On test_refmap's post-step frames the resident pool is RefMap.fuse_map's local_surfels, in order."""
    if not pyoracle.have_refmap():
        pytest.skip("the reference node library is not built")
    from densesurfelmapping_b200 import capi
    from test_refmap import CAM as RCAM, poststep_frames
    m = pyoracle.RefMap(RCAM)
    c = capi.Context(RCAM, max_batch=2, max_local_surfels=100000)
    pool = np.zeros(0, SURFEL_DTYPE)
    for t, (ref, gray, depth, pose) in enumerate(poststep_frames()):
        m.set_local(pool)
        m.fuse_map(gray, depth, pose, ref)
        want = m.local()
        c.pool_upload(pool)             # both start from the reference's pool
        c.fuse_frame_resident(ref, gray, depth, pose)
        got = c.pool_download()
        assert len(got) == len(want), f"frame {t}"
        assert np.array_equal(got["color"].view(np.uint32), want["color"].view(np.uint32)), f"frame {t}"
        check_surfels(got, want, f"frame {t} (in order)")
        pool = want
    m.close()
    c.close()


def test_a_frame_with_more_new_surfels_than_holes_moves_no_survivor(ctx, pool):
    p = craft(pool, "few_holes")
    gray, depth, pose = frame(3)
    lo, no, _ = expect(ctx, 3, gray, depth, pose, p)
    live = lo["update_times"] != 0
    assert len(no) >= (~live).sum()
    _, got = resident(ctx, p, 3, gray, depth, pose)
    assert got[:len(lo)][live].tobytes() == lo[live].tobytes()
    assert len(got) == len(lo) - (~live).sum() + len(no)
