"""GPU tests: k_fuse and k_init_surfels bit for bit against the host model (oracle/pyoracle_fuse.py) on the device's
own seeds, with pools built to reach every branch (tests/fuse_inputs.py), through fuse_frame, a four-slot fuse_batch and
the resident paths; and the device against the reference, each on its own seeds, on the cases that lie clear of every
seed-dependent threshold.  tests/test_fuse_model.py pins the model to the reference and shows the pools catch each
mutation of it."""
import functools

import numpy as np
import pytest

import fuse_inputs as fi
import pyoracle
from densesurfelmapping_b200 import synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from util import canon, check_surfels

pytestmark = pytest.mark.gpu

REF_FRAME = 9
PLANE_FIT_STEPS = 12  # kernels of the schedule through the plane solve: seed init, 3 x (assign, gather, Newton), 2
MARGIN = 1e-3         # relative distance from every seed-dependent threshold for the device-against-reference cases


@pytest.fixture(scope="module")
def capi():
    from densesurfelmapping_b200 import capi as m
    m.load_library()  # raises if the CUDA extension was not built: no fallback
    return m


def _consts(capi, cname):
    return capi.CONSTANTS_RGBD if cname == "rgbd" else capi.CONSTANTS_DRIVE


@functools.lru_cache(maxsize=None)
def _device_seeds(fname, cname):
    """Labels and seeds of the frame after the plane fit, read back from the device; two runs give the same bits."""
    from densesurfelmapping_b200 import capi
    cam, gray, depth = fi.frame(fname)
    ctx = capi.Context(cam, max_batch=1, max_local_surfels=16)
    try:
        ctx.set_constants(_consts(capi, cname))
        ctx.batch_upload([0], gray[None], depth[None], synth.identity_pose()[None], np.zeros(0, SURFEL_DTYPE), [0, 0])
        runs = []
        for _ in range(2):
            ctx.debug_stop_after(PLANE_FIT_STEPS)
            ctx.batch_run()
            ctx.sync()
            runs.append((ctx.labels(), ctx.seeds()))
        ctx.debug_stop_after(0)
    finally:
        ctx.close()
    (l0, s0), (l1, s1) = runs
    assert (l0 == l1).all() and canon(s0) == canon(s1), f"{fname}/{cname}: the tile stages are not deterministic"
    return cam, gray, depth, l0, s0


def _frame(fname, cname, pname, ref=REF_FRAME):
    cam, gray, depth, labels, seeds = _device_seeds(fname, cname)
    return fi.Frame(cam, seeds, labels, depth, fi.POSES[pname], fi.CONSTANTS[cname], ref), gray


def _length(n, phase, over=257):
    """The smallest length >= max(n, over) that is `phase` mod 4."""
    n = max(n, over)
    return n + (phase - n) % 4


def _same(got_pool, got_new, got_fused, want, what):
    assert len(got_new) == len(want["new"]), f"{what}: {len(got_new)} new surfels, the model {len(want['new'])}"
    for name, g, w in (("pool", got_pool, want["pool"]), ("new", got_new, want["new"])):
        if canon(g) != canon(w):
            bad = [i for i in range(len(g)) if canon(g[i:i + 1]) != canon(w[i:i + 1])]
            pytest.fail(f"{what}: {name} differs at {bad[:8]} (outcomes {want['outcome'][bad[:8]] if name == 'pool' else ''})")
    bad = np.nonzero(got_fused != want["fused"])[0]
    assert len(bad) == 0, f"{what}: fused flags differ at {bad[:8]}"


@pytest.mark.parametrize("pname", list(fi.POSES))
@pytest.mark.parametrize("cname", list(fi.CONSTANTS))
@pytest.mark.parametrize("fname", list(fi.FRAMES))
def test_fuse_frame_equals_model(capi, fname, cname, pname):
    """fuse_frame on a crafted pool: updated pool, new surfels, their count and the fused flags equal the model's bit
    for bit.  The identity pose's pool is a multiple of 4 surfels long (bulk staging, full and partial last block),
    the general pose's is not (word staging)."""
    fr, gray = _frame(fname, cname, pname)
    pool, _ = fi.build(fr)
    pool = fi.pad(pool, _length(len(pool) + 300, 0 if pname == "identity" else 2))
    want = fr.run(pool)
    ctx = capi.Context(fr.cam, max_batch=1, max_local_surfels=len(pool) + 16)
    try:
        ctx.set_constants(_consts(capi, cname))
        local, new = ctx.fuse_frame(REF_FRAME, gray, fr.depth, fr.pose, pool)
        fused = ctx.seeds()["fused"]
    finally:
        ctx.close()
    _same(local, new, fused, want, f"{fname}/{cname}/{pname}")


@pytest.mark.parametrize("cname", list(fi.CONSTANTS))
@pytest.mark.parametrize("pattern", fi.INIT_PATTERNS)
def test_init_patterns_equal_model(capi, cname, pattern):
    """k_init_surfels on 15 CTAs, with the emitters following each pattern around the CTA boundaries."""
    fr, gray = _frame("hd", cname, "general")
    pool = fi.init_pool(fr, pattern)
    want = fr.run(pool)
    ctx = capi.Context(fr.cam, max_batch=1, max_local_surfels=len(pool) + 16)
    try:
        ctx.set_constants(_consts(capi, cname))
        local, new = ctx.fuse_frame(REF_FRAME, gray, fr.depth, fr.pose, pool)
        fused = ctx.seeds()["fused"]
    finally:
        ctx.close()
    _same(local, new, fused, want, f"hd/{cname}/{pattern}")


@pytest.mark.parametrize("cname", list(fi.CONSTANTS))
def test_fuse_batch_slots_equal_model(capi, cname):
    """Three different frames in slots 0 - 2 and the first again in slot 3, each with its own pose, pool and reference
    index; the slices start at every 16-byte phase (offsets 0, 1, 2, 3 mod 4)."""
    names = list(fi.BATCH_FRAMES) + [fi.BATCH_FRAMES[0]]
    poses = ["general", "identity", "general", "identity"]
    frames, grays, pools, wants = [], [], [], []
    for b, (fname, pname) in enumerate(zip(names, poses)):
        fr, gray = _frame(fname, cname, pname, ref=REF_FRAME + b)
        if b == 3:  # the same frame as slot 0 under another pose
            fr = fi.Frame(fr.cam, fr.seeds, fr.labels, fr.depth, synth.pose_stream(7), fr.constants, REF_FRAME + b)
        pool, _ = fi.build(fr)
        pool = fi.pad(pool, _length(len(pool), 1), seed=b)
        frames.append(fr), grays.append(gray), pools.append(pool), wants.append(fr.run(pool))
    ofs = np.concatenate([[0], np.cumsum([len(p) for p in pools])]).astype(np.int32)
    assert [int(o) % 4 for o in ofs[:4]] == [0, 1, 2, 3]
    cam = frames[0].cam
    ctx = capi.Context(cam, max_batch=4, max_local_surfels=int(ofs[-1]) + 16)
    try:
        ctx.set_constants(_consts(capi, cname))
        local, news = ctx.fuse_batch([f.ref for f in frames], np.stack(grays), np.stack([f.depth for f in frames]),
                                     np.stack([f.pose for f in frames]), np.concatenate(pools), ofs)
        fused = [ctx.seeds(b)["fused"] for b in range(4)]
    finally:
        ctx.close()
    for b in range(4):
        _same(local[ofs[b]:ofs[b + 1]], news[b], fused[b], wants[b], f"{cname} slot {b} ({names[b]})")


@pytest.mark.parametrize("cname", list(fi.CONSTANTS))
def test_resident_paths_equal_model(capi, cname):
    """fuse_frame_resident, then fuse_stream_resident over two frames: the device pool after each call equals the
    reference's fuse_map post-step of the model's output."""
    fr0, g0 = _frame("vga", cname, "general")
    pool, _ = fi.build(fr0)
    ctx = capi.Context(fr0.cam, max_batch=2, max_local_surfels=1 << 16)
    try:
        ctx.set_constants(_consts(capi, cname))
        ctx.pool_upload(pool)
        ctx.fuse_frame_resident(REF_FRAME, g0, fr0.depth, fr0.pose)
        r = fr0.run(pool)
        want = pyoracle.fuse_map_poststep(r["pool"], r["new"])
        got = ctx.pool_download()
        assert canon(got) == canon(want), "fuse_frame_resident: pool differs from the model's post-step"
        fr1, g1 = _frame("vga2", cname, "general", ref=REF_FRAME + 1)
        fr2, g2 = _frame("near", cname, "identity", ref=REF_FRAME + 2)
        ctx.fuse_stream_resident([fr1.ref, fr2.ref], np.stack([g1, g2]), np.stack([fr1.depth, fr2.depth]),
                                 np.stack([fr1.pose, fr2.pose]))
        for fr in (fr1, fr2):
            r = fr.run(want)
            want = pyoracle.fuse_map_poststep(r["pool"], r["new"])
        got = ctx.pool_download()
        assert canon(got) == canon(want), "fuse_stream_resident: pool differs from the model's post-steps"
    finally:
        ctx.close()


# The near frame has seeds whose view_cos lies within MARGIN of the initialise's 0.1, where the plane fit's 1e-7 may
# decide whether a seed emits: it is held to the model alone, on the device's own seeds.
@pytest.mark.parametrize("pname", list(fi.POSES))
@pytest.mark.parametrize("cname", list(fi.CONSTANTS))
@pytest.mark.parametrize("fname", [f for f in fi.FRAMES if f != "near"])
def test_device_against_reference(capi, fname, cname, pname):
    """Each side on its own seeds: the crafted pool, less the cases the model puts within MARGIN of a seed-dependent
    threshold under either side's seeds, gives the reference's pool and new surfels at the parity contract (geometry
    within 1e-4, update_times, last_update and color exact) and the same fused flags."""
    fr, gray = _frame(fname, cname, pname)
    cam = fr.cam
    orc = pyoracle.RefSerial(cam) if cname == "drive" else pyoracle.RefSerialRGBD(cam)
    labels_r, seeds_r = orc.superpixels(gray, fr.depth)
    fr_r = fi.Frame(cam, seeds_r, labels_r, fr.depth, fr.pose, fr.constants, REF_FRAME)
    assert (labels_r == fr.labels).all(), "labels differ from the reference's"
    for f in (fr, fr_r):  # no seed sits near the view_cos threshold of the initialise
        vc = f.seeds["view_cos"].astype(np.float64)
        assert not (np.abs(vc - 0.1) < MARGIN).any()
    pool, _ = fi.build(fr)
    clear = (fi.margin(fr, pool) >= MARGIN) & (fi.margin(fr_r, pool) >= MARGIN)
    pool = pool[clear]
    assert (fr.run(pool)["outcome"] == fr_r.run(pool)["outcome"]).all()
    ctx = capi.Context(cam, max_batch=1, max_local_surfels=len(pool) + 16)
    try:
        ctx.set_constants(_consts(capi, cname))
        local, new = ctx.fuse_frame(REF_FRAME, gray, fr.depth, fr.pose, pool)
        fused = ctx.seeds()["fused"]
    finally:
        ctx.close()
    want_local, want_new = orc.fuse(REF_FRAME, gray, fr.depth, fr.pose, pool)
    # infinite positions are cut before any seed is read: those surfels stay as they are on both sides
    fin = np.isfinite(pool["px"]) & np.isfinite(pool["py"]) & np.isfinite(pool["pz"])
    assert (~fin).sum() >= 3 and canon(local[~fin]) == canon(want_local[~fin]) == canon(pool[~fin])
    check_surfels(local[fin], want_local[fin], "pool")
    check_surfels(new, want_new, "new")
    assert (fused == orc.seeds()["fused"]).all()
