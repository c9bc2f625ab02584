"""dsm_frontier_enable / _enqueue / _wait and dsm_debug_field_load_state: exploration frontiers of the latest known field.

The device equals oracle/pyoracle_frontier bit for bit, in the cluster table, the voxel list and the counts: on every
known field of the windowed drive (the model runs on the device's own field_state, which tests/test_gpu_field_known.py
pins to the known-space oracle), a resident request equal to its host-copy twin; on state grids loaded through
dsm_debug_field_load_state (hand cases, random grids over a sweep of densities, a serpentine of about a million voxels,
the checkerboard at 512x512x64; each load's distances, counts and states are held to the known-space oracle first,
through resident_map.load_known), at several min_voxels and both capacity cuts; twice the same request gives the same
bytes; the stream order against later field requests, a publish snapshot and an asynchronous checkpoint; the
rejected-frame and error contracts; and a drive with frontier jobs leaves the map, the clouds and the fields as a twin
without them.  The node is checked through tests/cpp/frontier_main.cpp."""
import filecmp

import numpy as np
import pytest

import pyoracle_frontier
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import POINT_DTYPE, SURFEL_DTYPE
from node_drive import node_script, run_driver
from resident_map import SHAPES, STORE, T, camera, load_known, map_state, new_ctx, simple_lists, warp, windowed
from test_frontier_model import serpentine
from test_gpu_field_known import MAX_RANGE, Views

pytestmark = pytest.mark.gpu

BIG = 1 << 26          # DSM_FRONTIER_MAX_CAPACITY
CAPS = (1 << 14, 1 << 20)   # the loaders' table and list capacities (the result is 5.6 MB)
SMALL_CAM = synth.Camera(64, 48, 60.0, 60.0, 31.5, 23.5, 0.5, 30.0)
UNKNOWN, OCCUPIED, FREE = pyoracle_frontier.UNKNOWN, pyoracle_frontier.OCCUPIED, pyoracle_frontier.FREE


def same(got, want, what):
    gc, gv, gn = got
    wc, wv, wn = want
    assert gn.tobytes() == wn.tobytes(), f"{what}: counts {gn} want {wn}"
    assert gc.tobytes() == wc.tobytes(), f"{what}: {len(gc)} / {len(wc)} clusters, first differing {next((i for i in range(min(len(gc), len(wc))) if gc[i].tobytes() != wc[i].tobytes()), None)}"
    assert gv.tobytes() == wv.tobytes(), f"{what}: voxel list ({len(gv)} / {len(wv)})"


def loader(shape, voxel=0.2, caps=CAPS):
    """A context whose field has grid `shape` (nx, ny, nz), with views and frontiers enabled."""
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    ctx.field_enable(voxel, *shape)
    ctx.views_enable(1, 1.0)
    ctx.frontier_enable(*caps)
    return ctx


def load_and_run(ctx, state, origin, voxel, m):
    load_known(ctx, state, origin, voxel)
    ctx.frontier_enqueue(m)
    return ctx.frontier_wait()


def check_grid(ctx, state, origin, voxel, ms=(1, 2, 50), what=""):
    mc, mv = ctx._frontier_caps
    for m in ms:
        same(load_and_run(ctx, state, origin, voxel, m), pyoracle_frontier.frontiers(state, origin, voxel, m, mc, mv), f"{what} m={m}")


def checkerboard(nz, ny, nx):
    z, y, x = np.indices((nz, ny, nx))
    return np.where((x + y + z) % 2 == 0, FREE, UNKNOWN).astype(np.uint8)


def test_hand_cases():
    cases = []
    st = np.full((3, 3, 3), UNKNOWN, np.uint8)
    for q in [[(0, 0, 0), (0, 1, 1)], [(0, 0, 0), (1, 1, 1)], [(0, 0, 0), (2, 2, 2)]]:   # edge, corner, apart
        s = st.copy()
        for p in q:
            s[p] = FREE
        cases.append(s)
    s = np.full((3, 3, 3), OCCUPIED, np.uint8)
    s[1, 1, 1], s[0, 0, 0] = FREE, UNKNOWN                                            # diagonal only
    cases.append(s.copy())
    s[0, 1, 1] = UNKNOWN                                                              # and a face
    cases.append(s)
    s = np.full((3, 3, 3), FREE, np.uint8)                                            # all free: the box's faces
    cases += [s, np.full((3, 3, 3), UNKNOWN, np.uint8), checkerboard(3, 3, 3)]
    s = np.full((3, 3, 3), FREE, np.uint8)
    s[1, 1, 1] = UNKNOWN
    cases.append(s)
    ctx = loader((3, 3, 3))
    for k, c in enumerate(cases):
        check_grid(ctx, c, (-2, 5, 1), 0.2, ms=(1, 2), what=f"case {k}")
    ctx.close()
    for shape in [(1, 1, 1), (7, 1, 1), (1, 6, 1), (1, 1, 5), (33, 5, 1), (1, 9, 40)]:   # axes of one voxel
        ctx = loader(shape)
        rng = np.random.default_rng(sum(shape))
        for p in [(0.5, 0.0, 0.5), (0.3, 0.2, 0.5)]:
            check_grid(ctx, rng.choice(3, size=shape[::-1], p=p).astype(np.uint8), (0, 0, 0), 0.2, ms=(1, 2), what=f"{shape} {p}")
        for v in (UNKNOWN, FREE):
            check_grid(ctx, np.full(shape[::-1], v, np.uint8), (0, 0, 0), 0.2, ms=(1,), what=f"{shape} all {v}")
        ctx.close()


def test_random_grids_at_a_size_a_user_runs():
    """320x320x40 over a sweep of densities of the three states, min_voxels 1, 2 and 50, and the same request twice."""
    shape, voxel = (320, 320, 40), 0.2
    ctx = loader(shape, voxel, (4096, 1 << 20))
    rng = np.random.default_rng(11)
    for p in [(0.5, 0.0, 0.5), (0.2, 0.1, 0.7), (0.7, 0.1, 0.2), (0.05, 0.05, 0.9), (0.9, 0.0, 0.1), (0.33, 0.33, 0.34)]:
        st = rng.choice(3, size=shape[::-1], p=p).astype(np.uint8)
        check_grid(ctx, st, (-160, -160, -5), voxel, what=f"density {p}")
        a = load_and_run(ctx, st, (-160, -160, -5), voxel, 1)
        b = load_and_run(ctx, st, (-160, -160, -5), voxel, 1)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b)), "the same request twice"
    ctx.close()


def test_serpentine_and_checkerboard():
    """A serpentine of about a million voxels (one path through 320x320x40, the union's longest chains), and the
    checkerboard at 512x512x64 (every free voxel a frontier, all of them one component)."""
    ctx = loader((320, 320, 40), 0.2, (16, 1 << 21))
    st = serpentine(320, 320, 40)
    assert 900_000 < int((st == FREE).sum()) < 1_200_000
    check_grid(ctx, st, (3, -7, 0), 0.2, ms=(1, 50), what="serpentine")
    c, v, n = load_and_run(ctx, st, (3, -7, 0), 0.2, 1)
    assert n["n_components"] == 1 and len(v) == n["n_frontier"]
    ctx.close()
    ctx = loader((512, 512, 64), 0.1, (4, 1 << 24))
    st = checkerboard(64, 512, 512)
    check_grid(ctx, st, (-256, -256, 0), 0.1, ms=(1,), what="checkerboard")
    ctx.close()


def test_capacity_cuts():
    """The voxel cut in the middle of a cluster (offset -1 from that cluster on), the cluster cut, and zero capacities."""
    shape = (64, 48, 16)
    rng = np.random.default_rng(5)
    st = rng.choice(3, size=shape[::-1], p=(0.3, 0.5, 0.2)).astype(np.uint8)
    full = pyoracle_frontier.frontiers(st, (1, 2, 3), 0.2, 1, BIG, BIG)
    big = int(np.argmax(full[0]["n_voxels"] > 3))
    cut = int(full[0]["offset"][big]) + 2
    for caps in [(CAPS[0], cut), (7, CAPS[1]), (7, cut), (0, CAPS[1]), (CAPS[0], 0), (0, 0), (1, 1)]:
        ctx = loader(shape, 0.2, caps)
        check_grid(ctx, st, (1, 2, 3), 0.2, ms=(1, 3), what=f"caps {caps}")
        ctx.close()


def test_stream_order():
    """A job enqueued before the next field request reads the old grid; a job after a plain request is refused."""
    shape = (40, 30, 20)
    ctx = loader(shape, 0.2)
    rng = np.random.default_rng(9)
    a = rng.choice(3, size=shape[::-1], p=(0.4, 0.1, 0.5)).astype(np.uint8)
    b = rng.choice(3, size=shape[::-1], p=(0.6, 0.1, 0.3)).astype(np.uint8)
    ctx.debug_field_load_state(a, (0, 0, 0))
    ctx.frontier_enqueue(1)                 # before the field is waited for
    with pytest.raises(capi.DsmError) as e:
        ctx.frontier_enqueue(1)             # one job in flight
    assert e.value.code == -7
    ctx.field_wait()
    got = ctx.frontier_wait()
    same(got, pyoracle_frontier.frontiers(a, (0, 0, 0), 0.2, 1, *CAPS), "first")
    ctx.frontier_enqueue(1)
    ctx.debug_field_load_state(b, (5, 5, 5))   # the next request, while the job is in flight
    got = ctx.frontier_wait()
    ctx.field_wait()
    same(got, pyoracle_frontier.frontiers(a, (0, 0, 0), 0.2, 1, *CAPS), "the old grid")
    same(load_and_run(ctx, b, (5, 5, 5), 0.2, 1), pyoracle_frontier.frontiers(b, (5, 5, 5), 0.2, 1, *CAPS), "the new grid")
    ctx.field_enqueue((0, 0, 0), 1)         # a plain request
    with pytest.raises(capi.DsmError) as e:
        ctx.frontier_enqueue(1)
    assert e.value.code == -7
    ctx.field_wait()
    ctx.close()


def frontier_of_waited_known(ctx, origin, voxel, m, what):
    """The job on the last waited known field (host copy) against the model on its state grid."""
    state, _ = ctx.field_state()
    mc, mv = ctx._frontier_caps
    ctx.frontier_enqueue(m)
    got = ctx.frontier_wait()
    same(got, pyoracle_frontier.frontiers(state, origin, voxel, m, mc, mv), what)
    return got


@pytest.mark.parametrize("shape", SHAPES[:3], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("chunk", [1, 4])
def test_known_fields_of_the_drive(chunk, shape):
    """The windowed drive with loop-closure warps between calls (views warped with the map); after every call a
    resident known field with a job, then its host-copy twin with a job: both equal the model on the twin's states."""
    lists = simple_lists()
    voxels = (0.125, 0.1, 0.3)
    ctxs, views = {}, {}
    for v in voxels:
        ctxs[v] = new_ctx(store=STORE)
        ctxs[v].field_enable(v, *shape)
        views[v] = Views(ctxs[v], 6)
        ctxs[v].frontier_enable(64, 1 << 16)
    stored, seen = set(), 0
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
        v = voxels[call % 3]
        ctx = ctxs[v]
        slots, poses = views[v].request()
        m = (1, 2, 50)[call % 3]
        ctx.field_enqueue_known(camera(t1 - 1), 5, slots, poses, host_copy=False)
        ctx.frontier_enqueue(m)             # before the field is waited for
        ctx.field_wait()
        resident = ctx.frontier_wait()
        ctx.field_enqueue_known(camera(t1 - 1), 5, slots, poses)
        origin = ctx.field_wait()[1]
        host = frontier_of_waited_known(ctx, origin, v, m, f"frames {t0}-{t1 - 1}, voxel {v}")
        assert all(x.tobytes() == y.tobytes() for x, y in zip(resident, host)), "resident and host-copy requests"
        seen += int(host[2]["n_clusters"]) > 0
    assert seen > 0 or shape == (1, 1, 1)
    for c in ctxs.values():
        c.close()


def test_frontiers_change_nothing_else(tmp_path):
    """A drive with frontier jobs, one beside a publish snapshot and an asynchronous checkpoint, leaves the map, both
    published clouds and the fields byte-identical to a twin without them."""
    lists = simple_lists()
    shape, voxel = (64, 64, 32), 0.1
    a, b = new_ctx(store=STORE), new_ctx(store=STORE)
    va, vb = {}, {}
    for c, d in ((a, va), (b, vb)):
        c.field_enable(voxel, *shape)
        c.publish_enable()
        c.checkpoint_enable()
        d["v"] = Views(c, 4)
    a.frontier_enable(32, 4096)
    stored = set()
    for call, t0 in enumerate(range(0, T, 2)):
        t1 = t0 + 2
        for c, d in ((a, va), (b, vb)):
            windowed(c, t0, t1, lists, want_counts=False)
            d["v"].capture_call(call, t0, t1)
        for t in range(t0, t1):
            stored = (stored | set(lists[t][1])) - set(lists[t][2])
        outs = []
        for c, d in ((a, va), (b, vb)):
            slots, poses = d["v"].request()
            c.field_enqueue_known(camera(t1 - 1), 5, slots, poses)
            if c is a:
                a.frontier_enqueue(1 + call % 3)
            c.publish_enqueue(5)
            c.checkpoint_enqueue(str(tmp_path / f"{'ab'[c is b]}{call}.dsm"))
            if call % 2 == 1 and stored:
                c.pool_transform(warp(1))
                c.inactive_transform(max(stored), warp(2))
                d["v"].warp(warp(1))
            f = c.field_wait()
            st = c.field_state()
            p = c.publish_wait()
            assert c.checkpoint_wait(True)
            outs.append((f, st, p))
        got = a.frontier_wait()
        fa, fb = outs[0][0], outs[1][0]
        what = f"after frames {t0}-{t1 - 1}"
        same(got, pyoracle_frontier.frontiers(outs[0][1][0], fa[1], voxel, 1 + call % 3, 32, 4096), what)
        assert fa[0].tobytes() == fb[0].tobytes() and outs[0][1][0].tobytes() == outs[1][1][0].tobytes(), f"{what}: field"
        assert outs[0][2][0].tobytes() == outs[1][2][0].tobytes() and outs[0][2][1].tobytes() == outs[1][2][1].tobytes(), f"{what}: clouds"
        assert map_state(a) == map_state(b), f"{what}: map"
        assert filecmp.cmp(str(tmp_path / f"a{call}.dsm"), str(tmp_path / f"b{call}.dsm"), shallow=False), f"{what}: checkpoint"
    a.close()
    b.close()


def test_rejected_frame_comes_back_from_wait():
    lists = simple_lists()
    first = next(t for t in range(T) if lists[t][1])
    shape, voxel = (64, 64, 32), 0.1
    b = new_ctx(store=1)
    b.field_enable(voxel, *shape)
    views = Views(b, 4)
    b.frontier_enable(64, 1 << 16)
    for call, t0 in enumerate(range(0, first + 2)):
        windowed(b, t0, t0 + 1, lists, want_counts=False)
        views.capture_call(call, t0, t0 + 1)
    slots, poses = views.request()
    b.field_enqueue_known(camera(first - 1), 1, slots, poses)
    b.frontier_enqueue(1)
    with pytest.raises(capi.DsmError) as e:
        b.field_wait()
    assert e.value.code == -6
    origin = e.value.field[1]
    state, _ = b.field_state()
    with pytest.raises(capi.DsmError) as e:
        b.frontier_wait()
    assert e.value.code == -6
    same(e.value.frontier, pyoracle_frontier.frontiers(state, origin, voxel, 1, 64, 1 << 16), "rejected")
    assert e.value.frontier[2]["n_frontier"] > 0
    with pytest.raises(capi.DsmError) as e:
        b.pool_size()
    assert e.value.code == -6                            # wait did not clear it
    b.close()


def test_error_contract():
    lib = capi.load_library()
    I3 = capi.ctypes.c_int32 * 3
    ctx = capi.Context(SMALL_CAM, max_batch=2, max_local_surfels=1 << 12)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    st = np.full((4, 5, 6), FREE, np.uint8)
    assert lib.dsm_frontier_enable(ctx.h, 1, 1) == -7                      # before dsm_field_enable
    ctx.field_enable(0.2, 6, 5, 4)
    assert lib.dsm_frontier_enable(ctx.h, 1, 1) == -7                      # before dsm_views_enable
    assert lib.dsm_debug_field_load_state(ctx.h, st.ctypes.data, I3(0, 0, 0)) == -7
    ctx.views_enable(1, 1.0)
    assert lib.dsm_frontier_enqueue(ctx.h, 1) == -7                        # before dsm_frontier_enable
    assert lib.dsm_frontier_wait(ctx.h, None, None, None) == -7
    for mc, mv in [(-1, 0), (0, -1), (BIG + 1, 0), (0, BIG + 1)]:
        assert lib.dsm_frontier_enable(ctx.h, mc, mv) == -1, (mc, mv)
    assert lib.dsm_frontier_enable(None, 1, 1) == -1
    ctx.frontier_enable(2, 8)
    assert lib.dsm_frontier_enable(ctx.h, 1, 1) == -7                      # once
    assert lib.dsm_frontier_enqueue(ctx.h, 1) == -7                        # no field request yet
    assert lib.dsm_frontier_wait(ctx.h, None, None, None) == -7            # nothing enqueued
    bad = st.copy()
    bad[3, 4, 5] = 3
    assert lib.dsm_debug_field_load_state(ctx.h, bad.ctypes.data, I3(0, 0, 0)) == -1
    lim = 1 << 24
    for o in [(lim + 1, 0, 0), (0, -lim - 1, 0), (0, 0, lim - 3), (-lim - 1, 0, 0)]:
        assert lib.dsm_debug_field_load_state(ctx.h, st.ctypes.data, I3(*o)) == -1, o
    assert lib.dsm_debug_field_load_state(ctx.h, None, I3(0, 0, 0)) == -1
    assert lib.dsm_debug_field_load_state(ctx.h, st.ctypes.data, None) == -1
    assert lib.dsm_debug_field_load_state(ctx.h, st.ctypes.data, I3(lim - 6, -lim, lim - 4)) == 0   # the bounds themselves
    assert lib.dsm_debug_field_load_state(ctx.h, st.ctypes.data, I3(0, 0, 0)) == -7                 # a field in flight
    assert lib.dsm_frontier_enqueue(ctx.h, 0) == -1
    assert lib.dsm_frontier_enqueue(None, 1) == -1
    assert lib.dsm_frontier_enqueue(ctx.h, 1) == 0
    assert lib.dsm_frontier_enqueue(ctx.h, 1) == -7                        # one job in flight
    ctx.field_wait()
    counts = np.zeros(1, capi.FRONTIER_COUNTS_DTYPE)
    assert lib.dsm_frontier_wait(ctx.h, None, None, counts.ctypes.data) == 0
    assert counts.tolist() == [(0, 0, 0, 0)]                                # all free: no frontier
    assert lib.dsm_frontier_wait(ctx.h, None, None, None) == -7
    state, n_free = ctx.field_state()
    assert state.tobytes() == st.tobytes() and n_free == st.size
    ctx.field_enqueue((0, 0, 0), 1)                                        # a plain request
    ctx.field_wait()
    assert lib.dsm_frontier_enqueue(ctx.h, 1) == -7
    ctx.close()


# ---- the node ----
FIELD = (0.2, 96, 96, 32)
MAX_VIEWS = 5
RELOAD = 12   # the node saves and loads its state after this depth message


def test_node_frontiers_equal_the_model_and_change_nothing(tmp_path):
    """The node drive (keyframes, loop closures): after every fused frame, frontiers() equals the model over the state
    grid the driver dumps; clouds, PLY and PCD files equal a twin without frontiers; after load_state, frontiers()
    returns DSM_E_STATE until the next fused frame."""
    cam, n = synth.KITTI, 24
    sc = node_script(cam, n)
    voxel, nx, ny, nz = FIELD
    pa, pb = str(tmp_path / "mapa"), str(tmp_path / "mapb")
    node = [2, 0, 1 << 20, 1 << 21, *FIELD, MAX_VIEWS, MAX_RANGE]
    r = run_driver("frontier_main", str(tmp_path), cam, sc, node + [64, 1 << 16, RELOAD], tag="a", after=[pa])
    q = run_driver("frontier_main", str(tmp_path), cam, sc, node + [0, 0, RELOAD], tag="b", after=[pb])
    found = 0
    for t in range(n):
        rc, m = r.i(), r.i()
        origin = r.take(np.int32, 3).copy()
        state = r.lst(np.uint8).reshape(nz, ny, nx)
        clusters, vox = r.lst(pyoracle_frontier.CLUSTER_DTYPE), r.lst(np.int32)
        counts = r.take(np.int32, 4).copy()
        after_load = r.i()
        rr, act, inact = r.i(), r.lst(POINT_DTYPE), r.lst(POINT_DTYPE)
        rq, act_q, inact_q = q.i(), q.lst(POINT_DTYPE), q.lst(POINT_DTYPE)
        assert rc == 0 and rr == 0 and rq == 0, f"message {t}: {rc} {rr} {rq}"
        want = pyoracle_frontier.frontiers(state, origin, voxel, m, 64, 1 << 16)
        same((clusters, vox, counts.view(pyoracle_frontier.COUNTS_DTYPE)[0]), want, f"message {t}")
        found += len(clusters) > 0
        assert after_load == (-7 if t == RELOAD - 1 else 1), f"message {t}: frontiers() after load_state"
        assert act.tobytes() == act_q.tobytes() and inact.tobytes() == inact_q.tobytes(), f"message {t}: clouds"
    assert found > n // 2
    assert r.lst(SURFEL_DTYPE).tobytes() == q.lst(SURFEL_DTYPE).tobytes()
    assert r.o == len(r.raw) and q.o == len(q.raw)
    for ext in (".ply", ".pcd"):
        assert filecmp.cmp(pa + ext, pb + ext, shallow=False), ext
