"""oracle/pyoracle_viewpoint_terrain, the definition of dsm_viewpoint_enqueue_terrain (DESIGN.md §8.23): against a brute
force that scores every traversable ring cell and rotation with a whole gain job at the camera pose, for all six up axes
and both blocking rules; the camera voxel, the centre cell, reach's costs and a walled-off pocket, the ties, the hand
scenes whose answer is known, and every refusal."""
import numpy as np
import pytest

import pyoracle_frontier
import pyoracle_gain as G
import pyoracle_reach_terrain as RT
import pyoracle_terrain as TR
import pyoracle_viewpoint as V
import pyoracle_viewpoint_terrain as VT
from ground_views import WIDE, pit_behind_wall, rotations, scene, shelf_behind_wall
from planner_scenes import params
from pyoracle_field_known import FREE, OCCUPIED, UNKNOWN

INF = V.INF


def frontier(st, o, voxel):
    table, vox, _ = pyoracle_frontier.frontiers(st, o, voxel, 1, 64, 1 << 20)
    return table, vox


def brute(st, o, voxel, tr, cam, rot, cl, prm, eye, fr, reach_cost=None):
    """Every ring cell by hand, each rotation scored by a gain job on [R_r | t] naming the cluster, with the camera eye
    voxels above the cell's level: the ranked (n_seen, cost, offset index, rotation, cell) per cluster."""
    p = V.Params(*prm)
    tinfo, level, status, _, clearance = tr
    up = int(tinfo["up"])
    a, (h0, h1) = abs(up) - 1, RT.plane_axes(up)
    P, Q = int(tinfo["m"][h0]), int(tinfo["m"][h1])
    lev, sta, cle = level.reshape(Q, P), status.reshape(Q, P), clearance.reshape(Q, P)
    table, _ = fr
    v = np.float64(np.float32(voxel))
    out = []
    for c in cl:
        if c >= len(table) or table[c]["offset"] < 0:
            out.append([])
            continue
        g = np.floor(table[c]["centroid"] / v).astype(np.int64) - np.asarray(o)
        ranked, j = [], -1
        for dy in range(-p.r_max, p.r_max + 1):
            for dx in range(-p.r_max, p.r_max + 1):
                if dx % p.stride or dy % p.stride or not p.r_min ** 2 <= dx * dx + dy * dy <= p.r_max ** 2:
                    continue
                j += 1
                x, y = g[h0] + dx, g[h1] + dy
                if not (0 <= x < P and 0 <= y < Q) or not (sta[y, x] == FREE and cle[y, x] >= np.float32(p.radius)):
                    continue
                cost = INF if not p.with_reach else int(reach_cost.reshape(Q, P)[y, x])
                if p.with_reach and cost == INF:
                    continue
                k = [0, 0, 0]
                k[h0], k[h1], k[a] = x, y, int(lev[y, x]) + (eye if up > 0 else -eye)
                t = G.centres([k], o, voxel)[0]
                poses = [np.concatenate([Rm.reshape(3, 3), t[:, None]], axis=1).reshape(12) for Rm in np.asarray(rot).reshape(-1, 9)]
                n = G.gains(st, o, voxel, cam, poses, [c] * len(poses), fr)[1]["n_cluster"]
                best = int(np.argmax(n))
                if n[best] >= max(1, p.min_seen):
                    ranked.append((-int(n[best]), cost, j, best, int(y * P + x)))
        out.append(sorted(ranked)[:p.top_k])
    return out


def assert_slots(slots, want, what):
    for i, w in enumerate(want):
        got = [(-int(s["n_seen"]), int(s["cost"]), int(s["offset"]), int(s["rotation"]), int(s["voxel"])) for s in slots[i] if s["voxel"] >= 0]
        assert got == w, f"{what}: cluster {i}"
        rest = slots[i][len(w):]
        assert (rest["voxel"] == -1).all() and (rest["n_seen"] == 0).all() and (rest["cost"] == INF).all()


@pytest.mark.parametrize("unknown_blocks", [0, 1])
@pytest.mark.parametrize("up", TR.UPS)
def test_model_equals_gain_jobs(up, unknown_blocks):
    rng = np.random.default_rng(70 + 3 * up + unknown_blocks)
    shape = [15, 13, 12]
    shape[abs(up) - 1] = 9
    voxel, o = 0.2, tuple(int(x) for x in rng.integers(-20, 20, 3))
    st = scene(rng, shape, up, p_box=0.08, p_hole=0.05)
    tr = TR.job(st, o, voxel, up, 3, 1)
    fr = frontier(st, o, voxel)
    cam = G.Camera(1.5, 1.5, 2.0, 1.5, 4, 3, 1.2, unknown_blocks)
    rot = rotations(up, 6, (0.0, -0.4))
    cl = list(range(min(len(fr[0]), 4))) + [len(fr[0])]
    for eye in (1, 3):
        prm = params(1, 3, 0, 1, max_samples=4096, top_k=4)
        info, recs, slots = VT.viewpoints(st, voxel, tr, cam, rot, cl, prm, eye, fr)
        assert_slots(slots, brute(st, o, voxel, tr, cam, rot, cl, prm, eye, fr), f"up {up}, eye {eye}")
        assert recs["status"][-1] == 3 and (recs["status"][:-1] == 0).all()
        assert info["origin"].tolist() == list(o) and info["n_offsets"] == len(V.offsets(prm)) and info["n_rotations"] == len(rot)
        assert info["unknown_blocks"] == unknown_blocks and info["n_clusters_table"] == len(fr[0])
        assert (recs["n_reached"] == recs["n_traversable"]).all()
    assert len(cl) >= 2 and (recs["n_viewpoints"] > 0).sum() >= 1


@pytest.mark.parametrize("up", TR.UPS)
def test_camera_voxel_is_free_and_eye_above_the_level(up):
    rng = np.random.default_rng(10 + up)
    for trial in range(3):
        shape = [int(x) for x in rng.integers(6, 14, 3)]
        shape[abs(up) - 1] = int(rng.integers(8, 16))
        st = scene(rng, shape, up, p_box=0.15, p_hole=0.1)
        headroom = int(rng.integers(1, shape[abs(up) - 1] // 2))
        o = tuple(int(x) for x in rng.integers(-1000, 1000, 3))
        tinfo, level, status, _, _ = TR.job(st, o, 0.1, up, headroom, int(rng.integers(0, 3)))
        a, (h0, h1) = abs(up) - 1, RT.plane_axes(up)
        P, Q = shape[h0], shape[h1]
        lev = level.reshape(Q, P)
        for q, p in np.argwhere(status.reshape(Q, P) == FREE):
            for eye in range(1, headroom + 1):
                k = VT.camera_voxel(p, q, lev, up, eye)
                assert (k >= 0).all() and (k < shape).all(), (trial, p, q, eye)
                assert st[k[2], k[1], k[0]] == FREE and k[h0] == p and k[h1] == q
                assert (k[a] - lev[q, p]) * np.sign(up) == eye
                t = VT.camera_point(q * P + p, (tinfo, level), 0.1, eye)
                assert t.tolist() == G.centres([k], o, 0.1)[0].tolist()


def test_centre_cell_is_the_centroids_column():
    rng = np.random.default_rng(5)
    for up in TR.UPS:
        for voxel, o in [(0.2, (0, 0, 0)), (0.1, (-300, 77, -12)), (0.3, (1 << 20, -(1 << 20), 5))]:
            st = rng.choice(3, size=(10, 14, 18), p=(0.3, 0.1, 0.6)).astype(np.uint8)
            table, _ = frontier(st, o, voxel)
            h0, h1 = RT.plane_axes(up)
            for rec in table:
                g = VT.centre_cell(rec["centroid"], o, voxel, up)
                g3 = V.centre_voxel(rec["centroid"], o, voxel)
                assert g.tolist() == [g3[h0], g3[h1], 0]
                assert rec["lo"][h0] <= g[0] <= rec["hi"][h0] and rec["lo"][h1] <= g[1] <= rec["hi"][h1]


def test_reach_costs_and_a_walled_off_pocket():
    """A floor whose pocket of traversable cells is ringed by unsupported columns: without reach its cells are
    candidates; with the terrain reach job's costs from outside they are never reached, and every cost is the job's."""
    nx, ny, nz = 16, 14, 6
    st = np.full((nz, ny, nx), FREE, np.uint8)
    st[0] = OCCUPIED
    st[:, 3:10, 1:8] = UNKNOWN                   # a ring of columns without support ...
    st[:, 4:9, 2:7] = FREE                        # ... around a pocket with a floor
    st[0, 4:9, 2:7] = OCCUPIED
    st[1:, 13, :] = UNKNOWN                       # the frontier: the far wall's free border
    voxel, o = 0.2, (3, -4, 0)
    tr = TR.job(st, o, voxel, 3, 3, 1)
    fr = frontier(st, o, voxel)
    start = ((o[0] + 13 + 0.5) * 0.2, (o[1] + 2 + 0.5) * 0.2, 0.5)
    cost = RT.job(tr, (nx, ny, nz), voxel, start, 0.0, 1, exact=True)[3]
    assert cost.reshape(ny, nx)[6, 4] == INF and cost.reshape(ny, nx)[1, 1] != INF
    rot = rotations(3, 8)
    prm = params(0, 9, 0, 1, top_k=16)
    cl = list(range(len(fr[0])))
    a = VT.viewpoints(st, voxel, tr, WIDE, rot, cl, prm, 2, fr)
    b = VT.viewpoints(st, voxel, tr, WIDE, rot, cl, prm._replace(with_reach=1), 2, fr, cost)
    assert (a[1]["n_reached"] == a[1]["n_traversable"]).all() and (b[1]["n_traversable"] == a[1]["n_traversable"]).all()
    assert (b[1]["n_reached"] < b[1]["n_traversable"]).any() and b[0]["with_reach"] == 1
    pocket = {y * nx + x for y in range(4, 9) for x in range(2, 7)}
    assert any(s["voxel"] in pocket for s in a[2].reshape(-1)), "the pocket holds candidates without reach"
    for s in b[2].reshape(-1):
        if s["voxel"] >= 0:
            assert s["voxel"] not in pocket and s["cost"] == cost.reshape(-1)[s["voxel"]]
    assert_slots(b[2], brute(st, o, voxel, tr, WIDE, rot, cl, prm._replace(with_reach=1), 2, fr, cost), "reach")


def test_ties():
    st = pit_behind_wall(11, 3)
    voxel, o = 0.2, (0, 0, 0)
    tr = TR.job(st, o, voxel, 3, 7, 1)
    fr = frontier(st, o, voxel)
    looks = rotations(3, 4)                                     # +x, +y, -x, -y
    # between rotations: a repeated rotation goes to its first copy
    prm = params(0, 9, 0, 1, top_k=16)
    _, _, s1 = VT.viewpoints(st, voxel, tr, WIDE, looks[[1, 0, 0]], [0], prm, 1, fr)
    assert (s1[0]["rotation"][s1[0]["voxel"] >= 0] != 2).all() and (s1[0]["rotation"] == 1).any()
    # between candidates of equal n_seen: the lowest offset index without reach, the lowest cost first with it
    _, recs, s = VT.viewpoints(st, voxel, tr, WIDE, looks, [0], prm, 1, fr)
    n = s[0]["n_seen"]
    ties = [k for k in range(15) if n[k] == n[k + 1] and n[k] > 0]
    assert ties and all(s[0, k]["offset"] < s[0, k + 1]["offset"] for k in ties)
    cost = np.full(tr[2].shape, INF, np.uint32)
    for x in s[0]:
        if x["voxel"] >= 0:
            cost.reshape(-1)[x["voxel"]] = 1000 - x["offset"]       # reversed costs reverse each tie
    _, _, s2 = VT.viewpoints(st, voxel, tr, WIDE, looks, [0], prm._replace(with_reach=1), 1, fr, cost)
    for k in range(15):
        a, b = s2[0, k], s2[0, k + 1]
        if b["voxel"] >= 0:
            assert (-a["n_seen"], a["cost"], a["offset"]) < (-b["n_seen"], b["cost"], b["offset"])
            if a["n_seen"] == b["n_seen"]:
                assert a["cost"] < b["cost"] and a["offset"] > b["offset"]


def test_shelf_seen_only_from_a_high_eye():
    """The frontier is the free layer z = 6 on a shelf of unknown space behind a wall up to z = 6: from the floor a
    camera at eye <= 6 sees it only through the wall, so no viewpoint; at eye 7 and 8 the cells before the wall see it."""
    st = shelf_behind_wall()
    voxel, o = 0.2, (0, 0, 0)
    tr = TR.job(st, o, voxel, 3, 8, 1)
    fr = frontier(st, o, voxel)
    assert len(fr[0]) == 1
    rot = rotations(3, 8)
    prm = params(0, 9, 0, 1, top_k=4)
    for eye in range(1, 9):
        _, recs, slots = VT.viewpoints(st, voxel, tr, WIDE, rot, [0], prm, eye, fr)
        assert recs[0]["n_traversable"] > 0
        assert (recs[0]["n_viewpoints"] > 0) == (eye >= 7), eye
        if eye >= 7:
            assert (slots[0]["voxel"][slots[0]["voxel"] >= 0] % 14 <= 5).all()   # from the floor before the wall
            assert_slots(slots, brute(st, o, voxel, tr, WIDE, rot, [0], prm, eye, fr), f"eye {eye}")


def test_wall_seen_around_its_end():
    """The frontier is the free layer over a pit behind a full-height wall: with a gap at the wall's end the floor before
    the wall sees it around that end, at eye 1; without the gap nothing sees it."""
    voxel, o = 0.2, (0, 0, 0)
    rot = rotations(3, 8)
    prm = params(0, 9, 0, 1, top_k=4)
    for gap in (0, 2):
        st = pit_behind_wall(11, gap)
        tr = TR.job(st, o, voxel, 3, 7, 1)
        fr = frontier(st, o, voxel)
        _, recs, slots = VT.viewpoints(st, voxel, tr, WIDE, rot, [0], prm, 1, fr)
        assert (recs[0]["n_viewpoints"] > 0) == (gap > 0), gap
        assert_slots(slots, brute(st, o, voxel, tr, WIDE, rot, [0], prm, 1, fr), f"gap {gap}")
    # the best cells stand before the wall (x <= 6); through the gap they look across the pit at +x headings
    best = slots[0][slots[0]["voxel"] >= 0]
    assert (best["voxel"] % 14 <= 6).all() and best[0]["n_seen"] > 0


def test_refusals():
    ok = G.Camera(10.0, 10.0, 5.0, 5.0, 10, 10, 1.0, 1)
    rot = rotations(3, 4)
    prm = params(dz_max=0)
    VT.check_request(ok, 0.1, rot, [0, 3], prm, 1, 4, 4, 1000)
    VT.check_request(ok, 0.1, rot, [0], prm, 4, 4, 4, 1000)
    for bad in [dict(params=params(dz_max=1)), dict(params=params(dz_max=16)), dict(eye=0), dict(eye=5), dict(eye=-1),
                dict(camera=ok._replace(fx=0.0)), dict(rotations=np.zeros((0, 9))), dict(clusters=[-1]),
                dict(params=prm._replace(top_k=17)), dict(params=prm._replace(radius=float("nan")))]:
        kw = dict(camera=ok, voxel=0.1, rotations=rot, clusters=[0], params=prm, eye=2, headroom=4, max_clusters=4, max_candidates=1000)
        kw.update(bad)
        with pytest.raises(ValueError):
            VT.check_request(**kw)
    # the job itself refuses what the device refuses
    st = pit_behind_wall(11, 2)
    tr = TR.job(st, (0, 0, 0), 0.2, 3, 7, 1)
    with pytest.raises(ValueError):
        VT.viewpoints(st, 0.2, tr, WIDE, rot, [0], params(dz_max=1), 2, frontier(st, (0, 0, 0), 0.2))
    with pytest.raises(ValueError):
        VT.viewpoints(st, 0.2, tr, WIDE, rot, [0], prm, 8, frontier(st, (0, 0, 0), 0.2))
