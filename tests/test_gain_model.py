"""The view-gain model (oracle/pyoracle_gain.py, DESIGN.md §8.12) on the host: against a plain per-voxel loop over
pyoracle_field_known.walk, against exact rational geometry, on hand cases, under a 90-degree yaw symmetry, with cluster
statuses, the host box against the padded cube of the range sphere, and the refusals of dsm_gain_enqueue."""
import ctypes
from fractions import Fraction

import numpy as np
import pytest

import pyoracle_field_known as K
import pyoracle_frontier
import pyoracle_gain as G
from densesurfelmapping_b200 import capi

UNKNOWN, OCCUPIED, FREE = G.UNKNOWN, G.OCCUPIED, G.FREE


def yaw_pose(k, t, pitch_down=False):
    """A camera looking along the k-th horizontal axis direction (+x, +y, -x, -y) from t; R a signed permutation."""
    f = [(1, 0, 0), (0, 1, 0), (-1, 0, 0), (0, -1, 0)][k]
    r = [(0, -1, 0), (1, 0, 0), (0, 1, 0), (-1, 0, 0)][k]
    dn = (0, 0, -1)
    R = np.array([r, dn, f], np.float64).T
    if pitch_down:   # looking straight down (z forward = world -z)
        R = np.array([r, f, dn], np.float64).T * np.array([1, -1, 1])
    return np.concatenate([R, np.asarray(t, np.float64)[:, None]], axis=1).reshape(12)


def random_pose(rng, centre, spread):
    q = rng.normal(size=4)
    a, b, c, d = q / np.linalg.norm(q)
    R = np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                  [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                  [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])
    t = np.asarray(centre, np.float64) + rng.uniform(-spread, spread, 3)
    return np.concatenate([R, t[:, None]], axis=1).reshape(12)


def plain(state, origin, voxel, camera, pose):
    """One view's counts by a per-voxel Python loop: the frustum test in Python floats, one walk per voxel through
    pyoracle_field_known.walk, the blocking rule over its visits before the end voxel, and the frontier predicate by
    hand."""
    cam = G.Camera(*camera)
    nz, ny, nx = state.shape
    v = float(np.float32(voxel))
    P = [float(p) for p in pose]
    t = [P[3], P[7], P[11]]
    R = float(np.float32(cam.max_range))
    out = dict(n_frustum=0, n_free=0, n_unknown=0, n_occupied=0, n_frontier=0)
    for z in range(nz):
        for y in range(ny):
            for x in range(nx):
                c = [(float(origin[0] + x) + 0.5) * v, (float(origin[1] + y) + 0.5) * v, (float(origin[2] + z) + 0.5) * v]
                d = [c[k] - t[k] for k in range(3)]
                if not ((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2] <= R * R):
                    continue
                q = [(P[m] * d[0] + P[4 + m] * d[1]) + P[8 + m] * d[2] for m in range(3)]
                if not q[2] > 0:
                    continue
                u = cam.fx * (q[0] / q[2]) + cam.cx
                w = cam.fy * (q[1] / q[2]) + cam.cy
                if not (0 <= u < cam.width and 0 <= w < cam.height):
                    continue
                out["n_frustum"] += 1
                _, vis, end = K.walk(np.array([t]), np.array([c]), voxel)
                assert end[-1] and (vis[-1] == np.array([origin[0] + x, origin[1] + y, origin[2] + z])).all() or not end.any()
                if not end.any():
                    continue
                ok = True
                for i in vis[:-1]:
                    qx, qy, qz = int(i[0]) - origin[0], int(i[1]) - origin[1], int(i[2]) - origin[2]
                    if not (0 <= qx < nx and 0 <= qy < ny and 0 <= qz < nz):
                        ok = False
                        break
                    s = state[qz, qy, qx]
                    if (s != FREE) if cam.unknown_blocks else (s == OCCUPIED):
                        ok = False
                        break
                if not ok:
                    continue
                s = state[z, y, x]
                out[["n_unknown", "n_occupied", "n_free"][s]] += 1
                if s == FREE:
                    for dx, dy, dz in [(-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1)]:
                        a, b, cc = x + dx, y + dy, z + dz
                        if 0 <= a < nx and 0 <= b < ny and 0 <= cc < nz and state[cc, b, a] == UNKNOWN:
                            out["n_frontier"] += 1
                            break
    return out


def test_layouts():
    assert G.GAIN_DTYPE.itemsize == 32 and G.INFO_DTYPE.itemsize == 32 and ctypes.sizeof(capi.DsmGainCamera) == 48
    assert capi.VIEW_GAIN_DTYPE == G.GAIN_DTYPE and capi.GAIN_INFO_DTYPE == G.INFO_DTYPE


def test_end_voxel_is_the_voxel_itself():
    rng = np.random.default_rng(3)
    for voxel in (0.1, 0.2, 0.125, 0.3, 0.05):
        o = rng.integers(-(1 << 24), (1 << 24) - 1024, size=3)
        xyz = rng.integers(0, 1024, size=(4096, 3))
        c = G.centres(xyz, o, voxel)
        assert (np.floor(c / np.float64(np.float32(voxel))) == (o + xyz)).all()


@pytest.mark.parametrize("unknown_blocks", [0, 1])
def test_model_equals_a_plain_loop(unknown_blocks):
    rng = np.random.default_rng(11 + unknown_blocks)
    shape, voxel, o = (9, 7, 6), 0.2, (-4, 3, -2)
    st = rng.choice(3, size=shape[::-1], p=(0.3, 0.1, 0.6)).astype(np.uint8)
    cam = G.Camera(20.0, 24.0, 15.5, 11.5, 32, 24, 1.1, unknown_blocks)
    centre = G.centres([(4, 3, 3)], o, voxel)[0]
    poses = [random_pose(rng, centre, 0.6) for _ in range(12)] + [yaw_pose(k, centre) for k in range(4)]
    _, recs = G.gains(st, o, voxel, cam, poses)
    for j, p in enumerate(poses):
        want = plain(st, o, voxel, cam, p)
        got = {k: int(recs[j][k]) for k in want}
        assert got == want, f"view {j}"
    assert recs["n_free"].sum() > 0 and recs["n_unknown"].sum() + recs["n_occupied"].sum() > 0


def exact_crossings(t, c, v):
    """(voxels, tie): the voxels the segment t -> c crosses for a positive length, in exact rationals and in order, and
    whether two of its plane crossings on different axes lie within 1e-9 voxel edges of each other (a tie)."""
    ft = [Fraction(float(x)) / Fraction(float(v)) for x in t]
    fc = [Fraction(float(x)) / Fraction(float(v)) for x in c]
    d = [fc[k] - ft[k] for k in range(3)]
    L = float(sum(x * x for x in d)) ** 0.5
    cuts = []
    for k in range(3):
        if d[k] != 0:
            lo, hi = sorted((ft[k], fc[k]))
            for m in range(lo.numerator // lo.denominator, hi.numerator // hi.denominator + 2):
                s_ = (m - ft[k]) / d[k]
                if 0 < s_ < 1:
                    cuts.append((s_, k))
    cuts.sort()
    tie = any(a[1] != b[1] and float(b[0] - a[0]) * L <= 1e-9 for a, b in zip(cuts[:-1], cuts[1:]))
    bounds = sorted({Fraction(0), Fraction(1)} | {s_ for s_, _ in cuts})
    out = []
    for a, b in zip(bounds[:-1], bounds[1:]):
        mid = (a + b) / 2
        p = [ft[k] + mid * d[k] for k in range(3)]
        out.append(tuple(x.numerator // x.denominator for x in p))
    return out, tie


@pytest.mark.parametrize("unknown_blocks", [0, 1])
def test_seen_against_exact_geometry(unknown_blocks):
    """A voxel counted as seen has a segment from the camera to its centre that crosses only passing voxels for more
    than 1e-9 voxel edges; the model and the exact geometry disagree only where a crossing is shorter than that."""
    rng = np.random.default_rng(5 + unknown_blocks)
    shape, voxel, o = (8, 8, 6), 0.3, (2, -5, 1)
    st = rng.choice(3, size=shape[::-1], p=(0.2, 0.1, 0.7)).astype(np.uint8)
    nz, ny, nx = st.shape
    v = np.float64(np.float32(voxel))
    centre = G.centres([(4, 4, 3)], o, voxel)[0]
    checked = disagree = 0
    for _ in range(6):
        pose = random_pose(rng, centre, 0.5)
        t = pose.reshape(3, 4)[:, 3]
        xyz = np.stack(np.meshgrid(np.arange(nx), np.arange(ny), np.arange(nz), indexing="ij"), -1).reshape(-1, 3)
        c = G.centres(xyz, o, voxel)
        s = G.seen(st, o, voxel, t, c, unknown_blocks)
        for (x, y, z), cc, got in zip(xyz, c, s):
            cross, tie = exact_crossings(t, cc, v)
            assert cross[-1] == (o[0] + x, o[1] + y, o[2] + z)
            ok = True
            for vox in cross[:-1]:
                q = (vox[0] - o[0], vox[1] - o[1], vox[2] - o[2])
                inside = 0 <= q[0] < nx and 0 <= q[1] < ny and 0 <= q[2] < nz
                st_q = st[q[2], q[1], q[0]] if inside else None
                ok = ok and inside and ((st_q == FREE) if unknown_blocks else (st_q != OCCUPIED))
            checked += 1
            if got != ok:
                disagree += 1
                assert tie, f"voxel {(x, y, z)}: model {got}, exact {ok} without a tie"
    assert checked > 1000 and disagree <= checked // 100


def wall_scene(kind):
    st = np.full((5, 5, 12), FREE, np.uint8)
    st[:, :, 6] = kind
    return st


def test_hand_cases():
    voxel, o = 0.5, (0, 0, 0)
    cam = G.Camera(4.0, 4.0, 3.5, 3.5, 8, 8, 5.5, 1)
    t = G.centres([(1, 2, 2)], o, voxel)[0]
    pose = yaw_pose(0, t)
    # an occupied wall: its first layer is seen, nothing behind it
    st = wall_scene(OCCUPIED)
    _, r = G.gains(st, o, voxel, cam, [pose])
    _, rf = G.gains(np.full_like(st, FREE), o, voxel, cam, [pose])
    assert r[0]["n_occupied"] > 0 and r[0]["n_frustum"] == rf[0]["n_frustum"]
    seen_free_behind = rf[0]["n_free"] - r[0]["n_free"]
    assert seen_free_behind > 0 and r[0]["n_free"] + r[0]["n_occupied"] < rf[0]["n_free"]
    # an unknown slab blocks with unknown_blocks = 1 and passes with 0
    st = wall_scene(UNKNOWN)
    _, r1 = G.gains(st, o, voxel, cam, [pose])
    _, r0 = G.gains(st, o, voxel, cam._replace(unknown_blocks=0), [pose])
    assert r1[0]["n_unknown"] == r[0]["n_occupied"] and r1[0]["n_free"] == r[0]["n_free"]
    assert r0[0]["n_free"] + r0[0]["n_unknown"] == rf[0]["n_free"] and r0[0]["n_unknown"] == r1[0]["n_unknown"]
    # the frontier voxels are the free layer in front of the slab
    assert r1[0]["n_frontier"] > 0 and r1[0]["n_frontier"] <= r1[0]["n_free"]


def test_image_edges_behind_and_range():
    """v = 1 and a camera at a voxel centre make every quantity exact: u = 0 counts and u = width does not, a centre at
    q_z <= 0 never counts and a centre exactly at max_range does."""
    voxel, o = 1.0, (0, 0, 0)
    st = np.full((5, 1, 5), FREE, np.uint8)   # [z][y][x]
    t = np.array([0.5, 0.5, 0.5])
    pose = np.concatenate([np.eye(3), t[:, None]], axis=1).reshape(12)   # z forward = world z, x right = world x
    cam = G.Camera(1.0, 1.0, 0.0, 0.5, 1, 1, 2.5, 1)
    c = G.centres([(0, 0, 2), (1, 0, 2), (2, 0, 2), (0, 0, 0), (1, 0, 0), (0, 0, 3)], o, voxel)
    f = G.frustum(c, pose, cam)
    assert f.tolist() == [True, True, False, False, False, False]   # u = 0, 0.5 in; u = 1 out; q_z = 0, 0 out; range 3 > 2.5
    c2 = G.centres([(0, 0, 2)], o, voxel)                            # |d| = 2
    assert G.frustum(c2, pose, cam._replace(max_range=2.0)).tolist() == [True]
    assert G.frustum(c2, pose, cam._replace(max_range=np.nextafter(np.float32(2.0), np.float32(0)))).tolist() == [False]
    _, r = G.gains(st, o, voxel, cam, [pose])
    assert r[0]["n_frustum"] == 3 and r[0]["n_free"] == 3     # (0,0,1) at u = 0, w = 0.5; (0,0,2) and (1,0,2)


def test_camera_outside_or_in_unknown_and_clipped_boxes():
    voxel, o = 0.25, (3, 3, 3)
    rng = np.random.default_rng(2)
    st = rng.choice(3, size=(6, 7, 8), p=(0.1, 0.1, 0.8)).astype(np.uint8)
    st[2, 3, 3:] = FREE
    cam = G.Camera(10.0, 10.0, 7.5, 5.5, 16, 12, 2.0, 1)
    inside_t = G.centres([(3, 3, 2)], o, voxel)[0]
    outside_t = G.centres([(-2, 3, 2)], o, voxel)[0]
    _, r = G.gains(st, o, voxel, cam, [yaw_pose(0, outside_t), yaw_pose(0, inside_t)])
    assert r[0]["status"] == 1 and r[0]["n_frustum"] > 0
    assert r[0]["n_free"] == r[0]["n_unknown"] == r[0]["n_occupied"] == r[0]["n_frontier"] == 0
    assert r[1]["status"] == 0 and r[1]["n_free"] > 0
    st2 = st.copy()
    st2[2, 3, 3] = UNKNOWN
    _, r1 = G.gains(st2, o, voxel, cam, [yaw_pose(0, inside_t)])
    _, r0 = G.gains(st2, o, voxel, cam._replace(unknown_blocks=0), [yaw_pose(0, inside_t)])
    assert r1[0]["n_free"] + r1[0]["n_unknown"] + r1[0]["n_occupied"] == 0 and r0[0]["n_free"] > 0
    # the box of a camera in a corner is clipped by the grid; the padded cube gives the same counts
    nz, ny, nx = st.shape
    corner = G.centres([(0, 0, 0)], o, voxel)[0]
    pose = yaw_pose(1, corner)
    lo, size = G.box(pose, cam, voxel, o, (nx, ny, nz))
    assert (lo == 0).all() and (size < 2 * 8 + 3).all()
    assert G.gains(st, o, voxel, cam, [pose])[1].tobytes() == G.gains(st, o, voxel, cam, [pose], pyramid=False)[1].tobytes()


@pytest.mark.parametrize("shape", [(1, 1, 1), (5, 1, 1), (1, 6, 1), (1, 1, 7)])
def test_axes_of_one_voxel(shape):
    rng = np.random.default_rng(sum(shape))
    voxel, o = 0.5, (0, 0, 0)
    st = rng.choice([FREE, UNKNOWN], size=shape[::-1], p=(0.8, 0.2)).astype(np.uint8)
    cam = G.Camera(3.0, 3.0, 2.0, 2.0, 4, 4, 4.0, 0)
    t = G.centres([(0, 0, 0)], o, voxel)[0]
    poses = [yaw_pose(k, t + 0.1) for k in range(4)] + [random_pose(rng, t, 0.2) for _ in range(4)]
    _, r = G.gains(st, o, voxel, cam, poses)
    for j, p in enumerate(poses):
        want = plain(st, o, voxel, cam, p)
        assert {k: int(r[j][k]) for k in want} == want


def symmetric_scene(n, nz, rng):
    """A state grid [nz][n][n] (n odd) that depends only on z and on |dx| + |dy| from the centre column: symmetric
    under 90-degree yaw about the centre voxel, and every tie of the walk between two horizontal axes lands on voxels of
    one state, so the lowest-axis rule cannot break the symmetry."""
    h = n // 2
    table = rng.choice(3, size=(nz, 2 * h + 1), p=(0.25, 0.15, 0.6)).astype(np.uint8)
    table[:, :3] = FREE
    y, x = np.mgrid[0:n, 0:n]
    l1 = np.abs(x - h) + np.abs(y - h)
    st = table[:, l1]
    st[:, h, h] = FREE
    return st


def symmetric_views(n, nz, voxel):
    h = n // 2
    t = G.centres([(h, h, nz // 2)], (0, 0, 0), voxel)[0]
    return t, [yaw_pose(k, t) for k in range(4)]


def test_yaw_symmetry():
    rng = np.random.default_rng(17)
    n, nz, voxel = 15, 7, 0.5
    st = symmetric_scene(n, nz, rng)
    t, poses = symmetric_views(n, nz, voxel)
    for ub in (0, 1):
        cam = G.Camera(6.0, 6.0, 7.5, 5.5, 16, 12, 3.5, ub)
        _, r = G.gains(st, (0, 0, 0), voxel, cam, poses)
        assert all(r[k].tobytes() == r[0].tobytes() for k in range(4)), r
        assert r[0]["n_free"] > 0 and r[0]["n_frustum"] > r[0]["n_free"]


def test_cluster_coverage_and_statuses():
    rng = np.random.default_rng(23)
    shape, voxel, o = (12, 10, 6), 0.2, (0, 0, 0)
    st = rng.choice(3, size=shape[::-1], p=(0.6, 0.1, 0.3)).astype(np.uint8)
    st[3, 5, 6] = FREE
    table, _, _ = pyoracle_frontier.frontiers(st, o, voxel, 1, 64, 1 << 20)
    table, vox, _ = pyoracle_frontier.frontiers(st, o, voxel, 1, 64, int(table["n_voxels"][:len(table) // 2].sum()))
    listed = np.flatnonzero(table["offset"] >= 0)
    unlisted = np.flatnonzero(table["offset"] < 0)
    assert len(listed) > 0 and len(unlisted) > 0
    cam = G.Camera(8.0, 8.0, 7.5, 5.5, 16, 12, 2.0, 0)
    t = G.centres([(6, 5, 3)], o, voxel)[0]
    poses = [yaw_pose(k % 4, t) for k in range(6)] + [yaw_pose(0, G.centres([(-3, 0, 0)], o, voxel)[0])]
    cl = [int(listed[0]), int(unlisted[0]), len(table), -1, int(listed[-1]), len(table) + 7, int(listed[0])]
    info, r = G.gains(st, o, voxel, cam, poses, cl, (table, vox))
    assert info["n_clusters_table"] == len(table) and info["n_views"] == len(poses)
    assert r["status"].tolist() == [0, 2, 3, 0, 0, 3, 1]
    assert r["n_cluster"].tolist()[1:4] == [-1, -1, -1] and r["n_cluster"][5] == -1 and r["n_cluster"][6] == 0
    slot = G.cluster_slots(st.shape, table, vox)
    assert (slot.reshape(-1)[vox] >= 0).all() and (slot >= 0).sum() == len(vox)
    for j in (0, 4):   # by hand: the seen members of the cluster
        want = 0
        nz, ny, nx = st.shape
        xyz = np.stack(np.meshgrid(np.arange(nx), np.arange(ny), np.arange(nz), indexing="ij"), -1).reshape(-1, 3)
        c = G.centres(xyz, o, voxel)
        f = G.frustum(c, poses[j], cam)
        s = G.seen(st, o, voxel, t, c[f], 0)
        g = xyz[f][s]
        want = int((slot[g[:, 2], g[:, 1], g[:, 0]] == cl[j]).sum())
        assert r[j]["n_cluster"] == want
    info0, _ = G.gains(st, o, voxel, cam, poses)
    assert info0["n_clusters_table"] == 0


def test_box_holds_every_counted_voxel():
    """The host's box never misses a voxel the padded cube of the range sphere counts, on random poses and cameras,
    near the grid's faces too."""
    rng = np.random.default_rng(31)
    shape, voxel, o = (20, 16, 10), 0.2, (-7, 4, 0)
    st = rng.choice(3, size=shape[::-1], p=(0.1, 0.05, 0.85)).astype(np.uint8)
    nz, ny, nx = st.shape
    cams = [G.Camera(60.0, 60.0, 31.5, 23.5, 64, 48, 1.6, 0), G.Camera(20.0, 30.0, -5.0, 40.0, 40, 30, 2.4, 0),
            G.Camera(1226 / 2.2, 370 / 2.2, 613.0, 185.0, 1226, 370, 2.0, 1)]
    centre = G.centres([(10, 8, 5)], o, voxel)[0]
    for cam in cams:
        poses = [random_pose(rng, centre, 2.5) for _ in range(10)]
        a = G.gains(st, o, voxel, cam, poses)[1]
        b = G.gains(st, o, voxel, cam, poses, pyramid=False)[1]
        assert a.tobytes() == b.tobytes()
        for p in poses:
            lo, size = G.box(p, cam, voxel, o, (nx, ny, nz))
            clo, csize = G.box(p, cam, voxel, o, (nx, ny, nz), pyramid=False)
            assert ((lo >= clo) & (lo + size <= clo + csize)).all() or (size == 0).any()
    # a pose that is no rotation uses the cube alone
    skew = np.array([[2.0, 0, 0, 0.5], [0, 1, 0, 0.5], [0, 0, 1, 0.5]]).reshape(12)
    assert [x.tolist() for x in G.box(skew, cams[0], voxel, o, (nx, ny, nz))] == \
        [x.tolist() for x in G.box(skew, cams[0], voxel, o, (nx, ny, nz), pyramid=False)]


def test_refusals():
    ok = G.Camera(10.0, 10.0, 5.0, 5.0, 10, 10, 1.0, 1)
    pose = np.eye(3, 4).reshape(12)
    G.check_request(ok, 0.1, [pose], None, 4)
    G.check_request(ok, 0.1, np.zeros((0, 12)), None, 4)
    nan, inf = float("nan"), float("inf")
    bad = [ok._replace(fx=0.0), ok._replace(fx=-1.0), ok._replace(fx=nan), ok._replace(fy=inf), ok._replace(cx=nan),
           ok._replace(cy=inf), ok._replace(width=0), ok._replace(height=65537), ok._replace(max_range=0.0),
           ok._replace(max_range=-1.0), ok._replace(max_range=nan), ok._replace(max_range=inf),
           ok._replace(max_range=12.9), ok._replace(unknown_blocks=2), ok._replace(unknown_blocks=-1)]
    for cam in bad:
        with pytest.raises(ValueError):
            G.check_request(cam, 0.1, [pose], None, 4)
    G.check_request(ok._replace(max_range=float(np.float32(12.8))), 0.1, [pose], None, 4)
    with pytest.raises(ValueError):
        G.check_request(ok, 0.1, [pose] * 5, None, 4)
    p2 = pose.copy()
    p2[5] = nan
    with pytest.raises(ValueError):
        G.check_request(ok, 0.1, [p2], None, 4)
    with pytest.raises(ValueError):
        G.check_request(ok, 0.1, [pose], [-2], 4)
    G.check_request(ok, 0.1, [pose], [-1], 4)
    # the work bound: (2 ceil(R / v) + 3)^3 per view
    m = 2 * 128 + 3
    n_max = G.MAX_WORK // m ** 3
    big = ok._replace(max_range=12.8)
    G.check_request(big, 0.1, np.tile(pose, (n_max, 1)), None, G.MAX_VIEWS)
    with pytest.raises(ValueError):
        G.check_request(big, 0.1, np.tile(pose, (n_max + 1, 1)), None, G.MAX_VIEWS)
    for n in (0, G.MAX_VIEWS + 1):
        with pytest.raises(ValueError):
            G.check_enable(n)
    G.check_enable(1)
    G.check_enable(G.MAX_VIEWS)
