"""The known-space side of the planner GPU tests: the test's side of the capture-slot table (Views), the small contexts
that load state grids, the byte-for-byte comparison of job results, and the drives the planner jobs share: the known
fields of the windowed drive, a drive with jobs against a twin without them, the rejected frame, and the node drivers'
arguments and twin checks."""
import filecmp
import types

import numpy as np
import pytest

import pyoracle_field_known
import pyoracle_gain as G
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import POINT_DTYPE, SURFEL_DTYPE
from resident_map import STORE, T, camera, frames, map_state, new_ctx, simple_lists, warp, windowed

UNKNOWN, OCCUPIED, FREE = pyoracle_field_known.UNKNOWN, pyoracle_field_known.OCCUPIED, pyoracle_field_known.FREE
MAX_RANGE = 30.0
HALF = 8   # new_ctx's max_batch / 2: a windowed call of n <= 8 frames runs in the staging half of its parity
SMALL_CAM = synth.Camera(64, 48, 60.0, 60.0, 31.5, 23.5, 0.5, 30.0)
K = synth.KITTI


def gcam(cam, max_range, unknown_blocks):
    return G.Camera(cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height, float(np.float32(max_range)), unknown_blocks)


def pose12(p16, W=np.eye(4)):
    """Row-major [R | t] (camera to world) of a column-major pose, after the warp W."""
    T4 = np.asarray(p16, np.float64).reshape(4, 4).T
    return (W @ T4)[:3, :4].reshape(12)


class Views:
    """The test's side of the slot table: per slot, the rays the oracle expects and the view's current pose."""

    def __init__(self, ctx, max_views):
        self.ctx, self.max = ctx, max_views
        ctx.views_enable(max_views, MAX_RANGE)
        self.rays, self.poses, self.n = {}, {}, 0

    def capture_call(self, call, t0, t1):
        """Captures every frame of windowed call number `call` (frames t0..t1-1) into the next slots."""
        for f, t in enumerate(range(t0, t1)):
            slot = self.n % self.max
            self.ctx.views_capture(f, slot)
            self.rays[slot] = pyoracle_field_known.capture(self.ctx.seeds((call % 2) * HALF + f))
            self.poses[slot] = pose12(frames()[t][0])
            self.n += 1

    def warp(self, W):
        for s in self.poses:
            self.poses[s] = pose12(np.eye(4), W @ np.vstack([self.poses[s].reshape(3, 4), [0, 0, 0, 1]]))

    def request(self):
        slots = sorted(self.rays)
        return slots, np.array([self.poses[s] for s in slots]).reshape(-1, 12)

    def oracle_views(self, slots):
        return [(self.rays[s], self.poses[s]) for s in slots]


def small_ctx(shape, voxel):
    """A context of the small camera whose field has grid `shape` (nx, ny, nz) and one view slot: enough to load state
    grids through dsm_debug_field_load_state.  The caller enables its jobs."""
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(voxel, *shape)
    ctx.views_enable(1, 1.0)
    return ctx


def same(got, want, what, names, rounds=True):
    """got equals want byte for byte, part by part; `names` names the parts (a part of got that is None, a host copy the
    request did not make, is skipped).  Without rounds (an exact model has no round count) the header, part 0, must
    say converged, and its rounds and converged are not compared."""
    for k, name in enumerate(names):
        g, w = got[k], np.asarray(want[k])
        if g is None:
            continue
        if not rounds and k == 0:
            assert g["converged"] == 1, f"{what}: not converged in {g['rounds']} rounds"
            g = g.copy()
            g["rounds"], g["converged"] = w["rounds"], w["converged"]
        assert g.tobytes() == w.tobytes(), _difference(g, w, f"{what}: {name}")


def _difference(g, w, what):
    if g.shape != w.shape:
        return f"{what}: shape {g.shape}, want {w.shape}"
    bad = np.flatnonzero((g != w).reshape(-1))
    return f"{what}: {len(bad)} of {g.size} differ, first at {bad[:4]}\n{g.reshape(-1)[bad[:4]]}\nwant\n{w.reshape(-1)[bad[:4]]}"


def known_drive(shape, chunk, voxels, enable, request=True):
    """The windowed drive with loop-closure warps every other call, one context per voxel edge with six view slots and
    enable(ctx) after them, the views warped with the map.  Yields per call the context whose turn it is (voxels[call %
    len(voxels)]) as (call, t0, t1, ctx, voxel, camera, slots, poses, field, state): with `request` the field waited for after a
    host-copy known request at the camera, and its state grid; else None and None.  Closes the contexts at the end."""
    lists = simple_lists()
    ctxs, views = {}, {}
    for v in voxels:
        ctxs[v] = new_ctx(store=STORE)
        ctxs[v].field_enable(v, *shape)
        views[v] = Views(ctxs[v], 6)
        enable(ctxs[v])
    stored = set()
    for call, t0 in enumerate(range(0, T, chunk)):
        t1 = min(T, t0 + chunk)
        for v in voxels:
            windowed(ctxs[v], t0, t1, lists, want_counts=False)
            views[v].capture_call(call, t0, t1)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        if call % 2 == 1 and stored:
            for v in voxels:
                ctxs[v].pool_transform(warp(1))
                ctxs[v].inactive_transform(max(stored), warp(2))
                views[v].warp(warp(1))
        v = voxels[call % len(voxels)]
        ctx = ctxs[v]
        slots, poses = views[v].request()
        cam = camera(t1 - 1)
        field = state = None
        if request:
            ctx.field_enqueue_known(cam, 5, slots, poses)
            field = ctx.field_wait()
            state, _ = ctx.field_state()
        yield call, t0, t1, ctx, v, cam, slots, poses, field, state
    for c in ctxs.values():
        c.close()


def twin_drive(tmp_path, enable_both, enable_a, enqueue, wait, check):
    """A drive with a job on context a, beside publish snapshots and asynchronous checkpoints, leaves everything as on a
    twin b without it.  Both contexts: field, publishing, checkpoints, four view slots, then enable_both(c); then
    enable_a(a).  Per windowed call of two frames, on a then on b: a known request, enqueue(c, c is a, call, t1), a
    snapshot, a checkpoint, a warp on odd calls, then the waits of the field, the state grid, wait(c) (a dict of the
    shared jobs' results by name), the snapshot and the checkpoint.  Then check(a, outs of a, call, t1, what) waits for
    a's job and checks it, and the fields, state grids, shared results, clouds, map and checkpoint files must equal."""
    lists = simple_lists()
    shape, voxel = (64, 64, 32), 0.1
    a, b = new_ctx(store=STORE), new_ctx(store=STORE)
    twins = []
    for c in (a, b):
        c.field_enable(voxel, *shape)
        c.publish_enable()
        c.checkpoint_enable()
        twins.append((c, Views(c, 4)))
        enable_both(c)
    enable_a(a)
    stored = set()
    for call, t0 in enumerate(range(0, T, 2)):
        t1 = t0 + 2
        for c, views in twins:
            windowed(c, t0, t1, lists, want_counts=False)
            views.capture_call(call, t0, t1)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        outs = []
        for c, views in twins:
            slots, poses = views.request()
            c.field_enqueue_known(camera(t1 - 1), 5, slots, poses)
            enqueue(c, c is a, call, t1)
            c.publish_enqueue(5)
            c.checkpoint_enqueue(str(tmp_path / f"{'ab'[c is b]}{call}.dsm"))
            if call % 2 == 1 and stored:
                c.pool_transform(warp(1))
                c.inactive_transform(max(stored), warp(2))
                views.warp(warp(1))
            f = c.field_wait()
            st = c.field_state()
            shared = wait(c)
            p = c.publish_wait()
            assert c.checkpoint_wait(True)
            outs.append(dict(field=f, state=st, clouds=p, shared=shared))
        what = f"after frames {t0}-{t1 - 1}"
        oa, ob = outs
        check(a, oa, call, t1, what)
        assert oa["field"][0].tobytes() == ob["field"][0].tobytes(), f"{what}: field"
        assert oa["state"][0].tobytes() == ob["state"][0].tobytes(), f"{what}: field"
        for name, x in oa["shared"].items():
            y = ob["shared"][name]
            assert all((u is None and w is None) or np.asarray(u).tobytes() == np.asarray(w).tobytes() for u, w in zip(x, y)), \
                f"{what}: {name}"
        pa, pb = oa["clouds"], ob["clouds"]
        assert pa[0].tobytes() == pb[0].tobytes() and pa[1].tobytes() == pb[1].tobytes(), f"{what}: clouds"
        assert map_state(a) == map_state(b), f"{what}: map"
        assert filecmp.cmp(str(tmp_path / f"a{call}.dsm"), str(tmp_path / f"b{call}.dsm"), shallow=False), f"{what}: checkpoint"
    a.close()
    b.close()


def rejected(call):
    """call() raises the rejected frame's DSM_E_CAPACITY (-6); returns the error, which carries the results."""
    with pytest.raises(capi.DsmError) as e:
        call()
    assert e.value.code == -6
    return e.value


def rejected_known(enable, enqueue):
    """The rejected frame: a context whose store takes one surfel, with a field and four view slots, then enable(ctx),
    driven one frame per call (every frame captured) to the second frame after the first one that retires a keyframe;
    a known request at the camera before that retirement, enqueue(ctx, first), and the field's wait raising -6.  Returns
    ctx, field (the error's dist, origin, n_occupied), state and n_free (of field_state), first, shape, voxel, views and
    the requested slots."""
    lists = simple_lists()
    first = next(t for t in range(T) if lists[t][1])
    shape, voxel = (64, 64, 32), 0.1
    ctx = new_ctx(store=1)
    ctx.field_enable(voxel, *shape)
    views = Views(ctx, 4)
    enable(ctx)
    for call, t0 in enumerate(range(0, first + 2)):
        windowed(ctx, t0, t0 + 1, lists, want_counts=False)
        views.capture_call(call, t0, t0 + 1)   # the rejected frame's rays are observations too
    slots, poses = views.request()
    ctx.field_enqueue_known(camera(first - 1), 1, slots, poses)
    enqueue(ctx, first)
    field = rejected(ctx.field_wait).field
    state, n_free = ctx.field_state()
    return types.SimpleNamespace(ctx=ctx, field=field, state=state, n_free=n_free, first=first, shape=shape, voxel=voxel, views=views,
                                 slots=slots)


def assert_error_stays(ctx):
    rejected(ctx.pool_size)   # wait did not clear it


# ---- the node drivers ----
NODE_FIELD = (0.2, 96, 96, 32)
MAX_VIEWS = 5
RELOAD = 12   # the node saves and loads its state after this depth message


def node_args(max_views=MAX_VIEWS):
    """The arguments the known-field node drivers take after the camera: drift_free_poses device max_local max_inactive
    voxel nx ny nz max_views max_range."""
    return [2, 0, 1 << 20, 1 << 21, *NODE_FIELD, max_views, MAX_RANGE]


def twin_clouds(r, q, what):
    """The clouds of one depth message from a driver and its twin: both read, equal; returns the driver's."""
    rr, act, inact = r.i(), r.lst(POINT_DTYPE), r.lst(POINT_DTYPE)
    rq, act_q, inact_q = q.i(), q.lst(POINT_DTYPE), q.lst(POINT_DTYPE)
    assert rr == 0 and rq == 0, f"{what}: clouds {rr} {rq}"
    assert act.tobytes() == act_q.tobytes() and inact.tobytes() == inact_q.tobytes(), f"{what}: clouds"
    return act, inact


def twin_node_tail(r, q, pa, pb):
    """The end of a drive and its twin: local_surfels equal, both outputs read to their end, the PLY and PCD files equal."""
    assert r.lst(SURFEL_DTYPE).tobytes() == q.lst(SURFEL_DTYPE).tobytes()
    assert r.o == len(r.raw) and q.o == len(q.raw)
    for ext in (".ply", ".pcd"):
        assert filecmp.cmp(pa + ext, pb + ext, shallow=False), ext
