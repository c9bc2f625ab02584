"""oracle/pyoracle_viewpoint, the definition of dsm_viewpoint_enqueue (DESIGN.md §8.15): against a brute force that
scores every candidate and rotation with a whole gain job (oracle/pyoracle_gain) naming the cluster, the offsets, the
samples, the ties, min_seen and top_k, the statuses, reach, the centre voxel, and every limit and refusal."""
import ctypes

import numpy as np
import pytest

import pyoracle_field_known
import pyoracle_frontier
import pyoracle_gain as G
import pyoracle_reach
import pyoracle_viewpoint as V
from densesurfelmapping_b200 import capi
from planner_scenes import open_room, params, rotation, rotations, scene

UNKNOWN, OCCUPIED, FREE = G.UNKNOWN, G.OCCUPIED, G.FREE
INF = V.INF


def job(st, o, voxel, cam, rot, cl, prm, min_voxels=1, max_voxels=1 << 20, reach_cost=None):
    dist = pyoracle_field_known.state_field(st, voxel)[0]
    table, vox, _ = pyoracle_frontier.frontiers(st, o, voxel, min_voxels, 64, max_voxels)
    return V.viewpoints(st, dist, o, voxel, cam, rot, cl, prm, (table, vox), reach_cost), (table, vox), dist


def brute(st, dist, o, voxel, cam, rot, cl, prm, frontier, reach_cost=None):
    """Every candidate by hand, each rotation scored by a gain job on [R_r | t] naming the cluster (every member is a
    sample): the ranked (n_seen, cost, offset index, rotation, voxel) per cluster."""
    p = V.Params(*prm)
    table, vox = frontier
    nz, ny, nx = st.shape
    trav = pyoracle_reach.traversable(st, dist, p.radius)
    out = []
    for c in cl:
        if c >= len(table) or table[c]["offset"] < 0:
            out.append([])
            continue
        g = np.floor(table[c]["centroid"] / np.float64(np.float32(voxel))).astype(np.int64) - np.asarray(o)
        ranked, j = [], -1
        for dz in range(-p.dz_max, p.dz_max + 1):
            for dy in range(-p.r_max, p.r_max + 1):
                for dx in range(-p.r_max, p.r_max + 1):
                    if dx % p.stride or dy % p.stride or dz % p.stride or not p.r_min ** 2 <= dx * dx + dy * dy <= p.r_max ** 2:
                        continue
                    j += 1
                    x, y, z = g + (dx, dy, dz)
                    if not (0 <= x < nx and 0 <= y < ny and 0 <= z < nz) or not trav[z, y, x]:
                        continue
                    cost = INF if not p.with_reach else int(reach_cost[z, y, x])
                    if p.with_reach and cost == INF:
                        continue
                    t = G.centres([(x, y, z)], o, voxel)[0]
                    poses = [np.concatenate([R.reshape(3, 3), t[:, None]], axis=1).reshape(12) for R in np.asarray(rot).reshape(-1, 9)]
                    n = G.gains(st, o, voxel, cam, poses, [c] * len(poses), frontier)[1]["n_cluster"]
                    best = int(np.argmax(n))
                    if n[best] >= max(1, p.min_seen):
                        ranked.append((-int(n[best]), cost, j, best, int((z * ny + y) * nx + x)))
        out.append(sorted(ranked)[:p.top_k])
    return out


def assert_slots(slots, want, what):
    for i, w in enumerate(want):
        got = [(-int(s["n_seen"]), int(s["cost"]), int(s["offset"]), int(s["rotation"]), int(s["voxel"])) for s in slots[i] if s["voxel"] >= 0]
        assert got == w, f"{what}: cluster {i}"
        rest = slots[i][len(w):]
        assert (rest["voxel"] == -1).all() and (rest["n_seen"] == 0).all() and (rest["cost"] == INF).all()


def test_layouts():
    assert V.CLUSTER_DTYPE.itemsize == 32 and V.VIEWPOINT_DTYPE.itemsize == 32 and V.INFO_DTYPE.itemsize == 64
    assert ctypes.sizeof(capi.DsmViewpointParams) == 40
    assert capi.VIEWPOINT_CLUSTER_DTYPE == V.CLUSTER_DTYPE and capi.VIEWPOINT_DTYPE == V.VIEWPOINT_DTYPE
    assert capi.VIEWPOINT_INFO_DTYPE == V.INFO_DTYPE


def test_rotations_are_rotations():
    R = rotations(8, (0.0, 0.4, -0.3)).reshape(-1, 3, 3)
    assert np.allclose(R.transpose(0, 2, 1) @ R, np.eye(3)) and np.allclose(np.linalg.det(R), 1.0)
    # yaw 0 is yaw_pose(0) of the gain tests: forward +x, right -y, down -z
    assert np.allclose(R[0], np.array([(0, -1, 0), (0, 0, -1), (1, 0, 0)], np.float64).T)


def test_offsets_by_hand():
    assert V.offsets(params(0, 1, 0, 1)).tolist() == [[0, -1, 0], [-1, 0, 0], [0, 0, 0], [1, 0, 0], [0, 1, 0]]
    got = V.offsets(params(1, 2, 2, 2))
    ring = [[0, -2], [-2, 0], [2, 0], [0, 2]]
    assert got.tolist() == [[x, y, z] for z in (-2, 0, 2) for x, y in ring]
    assert len(V.offsets(params(2, 3, 0, 1))) == 4 + 8 + 4 + 4      # dx^2 + dy^2 in {4, 5, 8, 9}
    assert len(V.offsets(params(3, 3, 1, 2))) == 0                   # even components never make 9
    assert V.offsets(params(0, 0, 3, 3)).tolist() == [[0, 0, -3], [0, 0, 0], [0, 0, 3]]
    assert V.offsets(params(0, 5, 1, 4)).tolist() == [[x, y, z] for z in (0,) for y in (-4, 0, 4) for x in (-4, 0, 4)
                                                      if x * x + y * y <= 25]
    for prm in [params(0, 7, 3, 1), params(2, 9, 4, 3), params(5, 5, 0, 1), params(0, 64, 16, 8), params(10, 40, 6, 5)]:
        r, s = prm.r_max, prm.stride
        want = sum(1 for dz in range(-prm.dz_max, prm.dz_max + 1) for dy in range(-r, r + 1) for dx in range(-r, r + 1)
                   if dx % s == 0 and dy % s == 0 and dz % s == 0 and prm.r_min ** 2 <= dx * dx + dy * dy <= r * r)
        got = V.offsets(prm)
        assert len(got) == want
        assert [tuple(x) for x in got] == sorted((tuple(x) for x in got), key=lambda q: (q[2], q[1], q[0]))


def test_sample_positions():
    assert V.sample_positions(10, 4).tolist() == [0, 2, 5, 7]
    assert V.sample_positions(3, 5).tolist() == [0, 1, 2]
    assert V.sample_positions(4096, 4096).tolist() == list(range(4096))
    s = V.sample_positions(10007, 4096)
    assert len(s) == 4096 and s[0] == 0 and s[-1] < 10007 and (np.diff(s) >= 2).all()
    s = V.sample_positions((1 << 26) - 1, 4096)      # k n stays in int64
    assert s[-1] == 4095 * ((1 << 26) - 1) // 4096


@pytest.mark.parametrize("unknown_blocks", [0, 1])
def test_model_equals_gain_jobs(unknown_blocks):
    rng = np.random.default_rng(40 + unknown_blocks)
    shape, voxel, o = (16, 14, 8), 0.2, (-5, 2, -3)
    st = scene(rng, shape)
    cam = G.Camera(6.0, 6.0, 7.5, 5.5, 16, 12, 1.3, unknown_blocks)
    rot = np.concatenate([rotations(8), rotations(4, (0.5, -0.5))])
    prm = params(1, 3, 1, 1, top_k=5)
    (info, recs, slots), fr, dist = job(st, o, voxel, cam, rot, [], prm)
    cl = list(range(min(len(fr[0]), 6)))
    (info, recs, slots), fr, dist = job(st, o, voxel, cam, rot, cl, prm)
    assert len(cl) >= 3 and (recs["status"] == 0).all() and (recs["n_viewpoints"] > 0).sum() >= 2
    assert_slots(slots, brute(st, dist, o, voxel, cam, rot, cl, prm, fr), f"ub={unknown_blocks}")
    # seen[r] equals gain's n_cluster on every candidate and rotation
    table, vox = fr
    for i in cl[:3]:
        g = V.centre_voxel(table[i]["centroid"], o, voxel)
        m = vox[table[i]["offset"]:table[i]["offset"] + table[i]["n_voxels"]].astype(np.int64)
        nz, ny, nx = st.shape
        mc = G.centres(np.stack([m % nx, m // nx % ny, m // (nx * ny)], 1), o, voxel)
        for off in V.offsets(prm)[::3]:
            c = g + off
            if not ((c >= 0).all() and (c < shape).all()) or st[c[2], c[1], c[0]] != FREE:
                continue
            t = G.centres([c], o, voxel)[0]
            seen = V.seen_counts(st, o, voxel, cam, rot, t, mc)
            poses = [np.concatenate([R.reshape(3, 3), t[:, None]], axis=1).reshape(12) for R in rot]
            assert seen.tolist() == G.gains(st, o, voxel, cam, poses, [i] * len(rot), fr)[1]["n_cluster"].tolist()
    assert info["n_clusters"] == len(cl) and info["n_offsets"] == len(V.offsets(prm)) and info["n_rotations"] == len(rot)
    assert info["top_k"] == 5 and info["unknown_blocks"] == unknown_blocks and info["with_reach"] == 0
    assert info["n_clusters_table"] == len(table) and info["reserved"].tolist() == [0] * 6
    assert (recs["n_reached"] == recs["n_traversable"]).all() and (slots["cost"] == INF).all()


def test_sampling_cut():
    """With max_samples below a cluster's members, seen[r] counts the sampled members only."""
    rng = np.random.default_rng(8)
    shape, voxel, o = (18, 16, 6), 0.2, (0, 0, 0)
    st = np.full(shape[::-1], FREE, np.uint8)
    st[:, 12:, :] = UNKNOWN                       # one long frontier wall along x at y = 11
    cam = G.Camera(6.0, 6.0, 7.5, 5.5, 16, 12, 2.0, 1)
    rot = rotations(8)
    for ms in (1, 5, 17, 4096):
        prm = params(2, 4, 0, 2, max_samples=ms, top_k=3)
        (info, recs, slots), (table, vox), dist = job(st, o, voxel, cam, rot, [0], prm)
        n = int(table[0]["n_voxels"])
        assert recs[0]["n_samples"] == min(n, ms)
        assert (slots[0]["n_seen"] <= min(n, ms)).all()
        if ms < n:
            m = vox[table[0]["offset"]:][V.sample_positions(n, ms)].astype(np.int64)
            nz, ny, nx = st.shape
            mc = G.centres(np.stack([m % nx, m // nx % ny, m // (nx * ny)], 1), o, voxel)
            s0 = slots[0][0]
            c = np.array([s0["voxel"] % nx, s0["voxel"] // nx % ny, s0["voxel"] // (nx * ny)])
            assert V.seen_counts(st, o, voxel, cam, rot, G.centres([c], o, voxel)[0], mc).max() == s0["n_seen"]
    assert rng is not None


def test_ties():
    voxel, o = 0.25, (0, 0, 0)
    st = open_room()
    cam = G.Camera(4.0, 4.0, 3.5, 3.5, 8, 8, 8.0, 1)
    # between rotations: the same rotation twice goes to the first; from the centre voxel on the cluster's row the best
    # heading looks along the row's longer side (-x: the centre is x = 6 of 0..11)
    looks = [rotation(np.pi / 2), rotation(np.pi), rotation(np.pi), rotation(0.0)]
    prm = params(0, 0, 0, 1, top_k=1)
    (_, recs, slots), (table, vox), _ = job(st, o, voxel, cam, looks, [0], prm)
    g = V.centre_voxel(table[0]["centroid"], o, voxel)
    nz, ny, nx = st.shape
    m = vox.astype(np.int64)
    seen = V.seen_counts(st, o, voxel, cam, looks, G.centres([g], o, voxel)[0],
                         G.centres(np.stack([m % nx, m // nx % ny, m // (nx * ny)], 1), o, voxel))
    assert g.tolist() == [6, 11, 1] and seen[1] == seen[2] > seen[3] > seen[0]
    assert recs[0]["n_reached"] == 1 and slots[0, 0]["rotation"] == 1 and slots[0, 0]["n_seen"] == seen[1]
    # all headings equal (no frustum holds anything but the first): rotation 0
    (_, _, slots), _, _ = job(st, o, voxel, cam, [rotation(np.pi)] * 3, [0], prm)
    assert slots[0, 0]["rotation"] == 0 and slots[0, 0]["n_seen"] == seen[1]
    # between candidates of equal n_seen: the lowest offset index without reach, the lowest cost first with it
    wide = G.Camera(1.0, 1.0, 0.5, 0.5, 1, 1, 8.0, 1)   # a 90-degree cone, looking at the whole wall from afar
    prm = params(0, 1, 0, 1, top_k=5)
    (_, recs, slots), fr, dist = job(st, o, voxel, wide, [rotation(np.pi / 2)], [0], prm)
    n = slots[0]["n_seen"]
    ties = [k for k in range(4) if n[k] == n[k + 1] and n[k] > 0]
    for k in ties:
        assert slots[0, k]["offset"] < slots[0, k + 1]["offset"]
    assert (np.diff(n) <= 0).all()
    cost = np.full(st.shape, INF, np.uint32)
    nz, ny, nx = st.shape
    for s in slots[0]:
        if s["voxel"] >= 0:
            cost.reshape(-1)[s["voxel"]] = 100 - s["offset"]         # reversed costs reverse each tie
    (_, recs2, slots2), _, _ = job(st, o, voxel, wide, [rotation(np.pi / 2)], [0], prm._replace(with_reach=1), reach_cost=cost)
    assert recs2[0]["n_reached"] == (slots[0]["voxel"] >= 0).sum()
    for k in range(4):
        a, b = slots2[0, k], slots2[0, k + 1]
        if b["voxel"] >= 0:
            assert (-a["n_seen"], a["cost"], a["offset"]) < (-b["n_seen"], b["cost"], b["offset"])
            if a["n_seen"] == b["n_seen"]:
                assert a["cost"] < b["cost"] and a["offset"] > b["offset"]
    assert any(slots2[0, k]["n_seen"] == slots2[0, k + 1]["n_seen"] for k in range(4)) or not ties


def test_min_seen_and_top_k_above_the_available():
    voxel, o = 0.25, (0, 0, 0)
    st = open_room()
    cam = G.Camera(4.0, 4.0, 3.5, 3.5, 8, 8, 8.0, 1)
    rot = rotations(4)
    prm = params(0, 2, 1, 1, top_k=16)
    (_, recs, slots), fr, dist = job(st, o, voxel, cam, rot, [0], prm)
    n_all = int(recs[0]["n_viewpoints"])
    assert 0 < n_all < 16 or recs[0]["n_reached"] > 16
    seen = np.sort(slots[0]["n_seen"][slots[0]["voxel"] >= 0])[::-1]
    thresh = int(seen[len(seen) // 2])
    (_, recs2, slots2), _, _ = job(st, o, voxel, cam, rot, [0], prm._replace(min_seen=thresh))
    assert recs2[0]["n_viewpoints"] == min(16, (seen >= thresh).sum()) or recs[0]["n_viewpoints"] == 16
    assert (slots2[0]["n_seen"][slots2[0]["voxel"] >= 0] >= thresh).all()
    (_, recs3, slots3), _, _ = job(st, o, voxel, cam, rot, [0], prm._replace(min_seen=10 ** 6))
    assert recs3[0]["n_viewpoints"] == 0 and (slots3["voxel"] == -1).all() and (slots3["offset"] == -1).all()
    assert (slots3["rotation"] == -1).all() and (slots3["cost"] == INF).all() and (slots3["reserved"] == 0).all()
    # a camera facing away sees nothing: no viewpoints even with min_seen 0
    (_, recs4, _), _, _ = job(st, o, voxel, cam, [rotation(-np.pi / 2)], [0], params(0, 0, 0, 1, top_k=3))
    assert recs4[0]["n_reached"] == 1 and recs4[0]["n_viewpoints"] == 0


def test_statuses():
    rng = np.random.default_rng(23)
    shape, voxel, o = (12, 10, 6), 0.2, (0, 0, 0)
    st = rng.choice(3, size=shape[::-1], p=(0.6, 0.1, 0.3)).astype(np.uint8)
    dist = pyoracle_field_known.state_field(st, voxel)[0]
    table, _, _ = pyoracle_frontier.frontiers(st, o, voxel, 1, 64, 1 << 20)
    table, vox, _ = pyoracle_frontier.frontiers(st, o, voxel, 1, 64, int(table["n_voxels"][:len(table) // 2].sum()))
    listed, unlisted = np.flatnonzero(table["offset"] >= 0), np.flatnonzero(table["offset"] < 0)
    cl = [int(listed[0]), int(unlisted[0]), len(table), len(table) + 9, int(listed[-1])]
    cam = G.Camera(6.0, 6.0, 7.5, 5.5, 16, 12, 1.0, 0)
    info, recs, slots = V.viewpoints(st, dist, o, voxel, cam, rotations(4), cl, params(), (table, vox))
    assert recs["status"].tolist() == [0, 2, 3, 3, 0] and recs["cluster"].tolist() == cl
    for k in (1, 2, 3):
        r = recs[k]
        assert (r["n_samples"], r["n_inside"], r["n_traversable"], r["n_reached"], r["n_viewpoints"]) == (0, 0, 0, 0, 0)
        assert (slots[k]["voxel"] == -1).all()
    assert info["n_clusters_table"] == len(table)


def test_reach_walls_off_a_traversable_candidate():
    """A free room whose +y wall is unknown holds a sealed pocket of free voxels near the cluster; the robot stands
    outside it: the pocket's candidates are traversable but not reached, and each reported cost is the Dijkstra cost."""
    voxel, o = 0.25, (0, 0, 0)
    st = np.full((3, 13, 13), FREE, np.uint8)
    st[:, 12, :] = UNKNOWN
    st[:, 4:10, 0:5] = OCCUPIED
    st[:, 5:9, 1:4] = FREE
    dist = pyoracle_field_known.state_field(st, voxel)[0]
    trav = pyoracle_reach.traversable(st, dist, 0.0)
    nz, ny, nx = st.shape
    cost = pyoracle_reach.dijkstra(trav, (1 * ny + 2) * nx + 10)
    table, vox, _ = pyoracle_frontier.frontiers(st, o, voxel, 1, 8, 1 << 10)
    cam = G.Camera(4.0, 4.0, 3.5, 3.5, 8, 8, 8.0, 1)
    prm = params(0, 6, 1, 1, top_k=16)
    a = V.viewpoints(st, dist, o, voxel, cam, rotations(8), [0], prm, (table, vox))
    b = V.viewpoints(st, dist, o, voxel, cam, rotations(8), [0], prm._replace(with_reach=1), (table, vox), cost)
    ra, rb = a[1][0], b[1][0]
    assert ra["n_reached"] == ra["n_traversable"] and rb["n_traversable"] == ra["n_traversable"]
    assert 0 < rb["n_reached"] < rb["n_traversable"]
    g = V.centre_voxel(table[0]["centroid"], o, voxel)
    walled = [j for j, off in enumerate(V.offsets(prm)) if 1 <= (g + off)[0] <= 3 and 5 <= (g + off)[1] <= 8 and
              0 <= (g + off)[2] < nz]
    assert all(cost[(g + off)[2], (g + off)[1], (g + off)[0]] == INF for off in V.offsets(prm)[walled])
    assert walled
    for s in b[2][0]:
        if s["voxel"] >= 0:
            assert s["offset"] not in walled and s["cost"] == cost.reshape(-1)[s["voxel"]]
    assert b[0]["with_reach"] == 1
    assert_slots(b[2], brute(st, dist, o, voxel, cam, rotations(8), [0], prm._replace(with_reach=1), (table, vox), cost), "reach")


def test_centre_voxel_lies_within_the_bounds():
    rng = np.random.default_rng(5)
    for voxel, o in [(0.2, (0, 0, 0)), (0.1, (-300, 77, -12)), (0.3, (1 << 20, -(1 << 20), 5)), (0.125, (3, 3, 3))]:
        for p in [(0.3, 0.1, 0.6), (0.6, 0.1, 0.3), (0.1, 0.0, 0.9)]:
            st = rng.choice(3, size=(10, 14, 18), p=p).astype(np.uint8)
            table, _, _ = pyoracle_frontier.frontiers(st, o, voxel, 1, 1 << 12, 1 << 20)
            for rec in table:
                g = V.centre_voxel(rec["centroid"], o, voxel)
                assert (g >= rec["lo"]).all() and (g <= rec["hi"]).all(), (rec, g)


def test_refusals():
    ok = G.Camera(10.0, 10.0, 5.0, 5.0, 10, 10, 1.0, 1)
    rot = rotations(4)
    prm = params()
    V.check_request(ok, 0.1, rot, [0, 3], prm, 4, 1000)
    V.check_request(ok, 0.1, rot, [], prm, 4, 1000)
    nan, inf = float("nan"), float("inf")
    for cam in [ok._replace(fx=0.0), ok._replace(fy=nan), ok._replace(cx=inf), ok._replace(width=0), ok._replace(height=65537),
                ok._replace(max_range=0.0), ok._replace(max_range=12.9), ok._replace(max_range=nan), ok._replace(unknown_blocks=2)]:
        with pytest.raises(ValueError):
            V.check_request(cam, 0.1, rot, [0], prm, 4, 1000)
    bad_rot = rot.copy()
    bad_rot[1, 4] = nan
    for r in (np.zeros((0, 9)), np.tile(rot, (17, 1)), bad_rot):
        with pytest.raises(ValueError):
            V.check_request(ok, 0.1, r, [0], prm, 4, 1000)
    V.check_request(ok, 0.1, np.tile(rot, (16, 1)), [0], prm, 4, 1000)
    for cl in ([-1], [0] * 5):
        with pytest.raises(ValueError):
            V.check_request(ok, 0.1, rot, cl, prm, 4, 1000)
    for bad in [prm._replace(r_min=-1), prm._replace(r_min=4), prm._replace(r_max=65), prm._replace(dz_max=-1),
                prm._replace(dz_max=17), prm._replace(stride=0), prm._replace(stride=9), prm._replace(max_samples=0),
                prm._replace(max_samples=4097), prm._replace(min_seen=-1), prm._replace(top_k=0), prm._replace(top_k=17),
                prm._replace(with_reach=2), prm._replace(radius=nan), prm._replace(radius=-0.1), prm._replace(radius=inf),
                params(3, 3, 1, 2), params(0, 64, 16, 1)]:
        with pytest.raises(ValueError):
            V.check_request(ok, 0.1, rot, [0], bad, 4, 1 << 22)
    V.check_request(ok, 0.1, rot, [0], params(0, 64, 16, 8, top_k=16, min_seen=7, with_reach=1, radius=0.3), 4, 1 << 22)
    # n_offsets at its limit: the largest r_max at dz_max 1 and stride 1 whose 3 layers fit
    r = max(r for r in range(1, 40) if len(V.offsets(params(0, r, 1, 1))) <= V.MAX_OFFSETS)
    n18 = len(V.offsets(params(0, r, 1, 1)))
    V.check_request(ok, 0.1, rot, [0], params(0, r, 1, 1), 4, 1 << 22)
    with pytest.raises(ValueError):
        V.check_request(ok, 0.1, rot, [0], params(0, r + 1, 1, 1), 4, 1 << 22)
    # max_candidates and the work bound
    n = len(V.offsets(prm))
    V.check_request(ok, 0.1, rot, [0, 1], prm, 4, 2 * n)
    with pytest.raises(ValueError):
        V.check_request(ok, 0.1, rot, [0, 1], prm, 4, 2 * n - 1)
    big = params(0, r, 1, 1, max_samples=4096)
    k = V.MAX_WORK // (n18 * 4096)
    V.check_request(ok, 0.1, rot, [0] * k, big, V.MAX_CLUSTERS, V.MAX_CANDIDATES)
    with pytest.raises(ValueError):
        V.check_request(ok, 0.1, rot, [0] * (k + 1), big, V.MAX_CLUSTERS, V.MAX_CANDIDATES)
    for a, b in [(0, 1), (V.MAX_CLUSTERS + 1, 1), (1, 0), (1, V.MAX_CANDIDATES + 1)]:
        with pytest.raises(ValueError):
            V.check_enable(a, b)
    V.check_enable(1, 1)
    V.check_enable(V.MAX_CLUSTERS, V.MAX_CANDIDATES)
