"""oracle/pyoracle_frontier, the definition of dsm_frontier_enqueue's exploration frontiers: against a plain-Python
breadth-first search on random grids, and on hand cases at the edges of the definition (edge- and corner-only joins,
diagonal-only unknown, the grid boundary, one-voxel axes, uniform grids, the 3-D checkerboard, a serpentine), the
centroid, the open and face sums, the order, and both capacity cuts.  tests/test_gpu_frontier.py holds the device to
this model bit for bit."""
from collections import deque

import numpy as np
import pytest

from pyoracle_frontier import CLUSTER_DTYPE, FREE, OCCUPIED, UNKNOWN, frontier_mask, frontiers

BIG = 1 << 26


def bfs_model(state, origin, voxel, min_voxels, max_clusters, max_voxels):
    """The definition of include/dsm.h read literally, one voxel at a time."""
    nz, ny, nx = state.shape
    lin = lambda x, y, z: (z * ny + y) * nx + x
    inside = lambda x, y, z: 0 <= x < nx and 0 <= y < ny and 0 <= z < nz
    faces = [(-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1)]
    front = {}
    for z in range(nz):
        for y in range(ny):
            for x in range(nx):
                if state[z, y, x] != FREE:
                    continue
                unk = [d for d in faces if inside(x + d[0], y + d[1], z + d[2]) and state[z + d[2], y + d[1], x + d[0]] == UNKNOWN]
                if unk:
                    front[(x, y, z)] = unk
    seen, comps = set(), []
    for p in sorted(front, key=lambda q: lin(*q)):
        if p in seen:
            continue
        seen.add(p)
        todo, members = deque([p]), []
        while todo:
            q = todo.popleft()
            members.append(q)
            for dz in (-1, 0, 1):
                for dy in (-1, 0, 1):
                    for dx in (-1, 0, 1):
                        r = (q[0] + dx, q[1] + dy, q[2] + dz)
                        if r in front and r not in seen:
                            seen.add(r)
                            todo.append(r)
        comps.append(sorted(members, key=lambda q: lin(*q)))
    clusters = [c for c in comps if len(c) >= min_voxels]
    recs, vox, at = [], [], 0
    v = float(np.float32(voxel))
    for c in clusters[:max_clusters]:
        n = len(c)
        pairs = [d for q in c for d in front[q]]
        sums = [sum(q[k] for q in c) for k in range(3)]
        off = at if at + n <= max_voxels else -1
        if off >= 0:
            vox += [lin(*q) for q in c]
        at += n
        recs.append((n, lin(*c[0]), off, [min(q[k] for q in c) for k in range(3)], [max(q[k] for q in c) for k in range(3)],
                     0, len(pairs), [sum(d[k] for d in pairs) for k in range(3)],
                     [(sums[k] / n + (origin[k] + 0.5)) * v for k in range(3)]))
    counts = (len(front), len(comps), len(clusters), len(vox))
    return np.array(recs, CLUSTER_DTYPE), np.array(vox, np.int32), counts


def same(got, want):
    assert got[0].tobytes() == want[0].tobytes(), (got[0], want[0])
    assert got[1].tobytes() == want[1].tobytes()
    assert tuple(int(got[2][k]) for k in ("n_frontier", "n_components", "n_clusters", "n_listed")) == tuple(want[2])


def run(state, origin=(0, 0, 0), voxel=0.2, m=1, mc=BIG, mv=BIG):
    return frontiers(np.asarray(state, np.uint8), origin, voxel, m, mc, mv)


@pytest.mark.parametrize("p", [(0.2, 0.1, 0.7), (0.5, 0.0, 0.5), (0.7, 0.1, 0.2), (0.05, 0.05, 0.9), (0.33, 0.33, 0.34)])
def test_model_equals_a_plain_search(p):
    rng = np.random.default_rng(int(p[0] * 1000))
    for shape in [(4, 5, 6), (3, 7, 9), (1, 8, 8), (6, 1, 5), (5, 6, 1), (2, 2, 2)]:
        st = rng.choice(3, size=shape, p=p).astype(np.uint8)
        for m, mc, mv in [(1, BIG, BIG), (2, 3, 10), (3, 1, 0), (1, 0, BIG)]:
            same(run(st, (-3, 5, 7), 0.3, m, mc, mv), bfs_model(st, (-3, 5, 7), 0.3, m, mc, mv))


def test_edge_and_corner_joins_make_one_cluster():
    st = np.full((3, 3, 3), UNKNOWN, np.uint8)
    for edge in ([(0, 0, 0), (0, 1, 1)], [(0, 0, 0), (1, 1, 1)]):   # (z, y, x): shares an edge / only a corner
        s = st.copy()
        for q in edge:
            s[q] = FREE
        c, vox, n = run(s)
        assert (n["n_frontier"], n["n_components"]) == (2, 1) and c["n_voxels"].tolist() == [2]
    s = st.copy()
    s[0, 0, 0] = s[2, 2, 2] = FREE                                     # two apart: two clusters
    assert run(s)[2]["n_components"] == 2


def test_only_a_face_neighbour_makes_a_frontier():
    st = np.full((3, 3, 3), OCCUPIED, np.uint8)
    st[1, 1, 1] = FREE
    st[0, 0, 0] = UNKNOWN                                              # diagonal only
    assert run(st)[2]["n_frontier"] == 0
    st[0, 1, 1] = UNKNOWN                                              # below (z - 1): a face
    c, vox, n = run(st)
    assert n["n_frontier"] == 1 and c["n_faces"].tolist() == [1] and c["open"].tolist() == [[0, 0, -1]]


def test_the_grid_boundary_does_not_count():
    st = np.full((4, 4, 4), FREE, np.uint8)
    assert run(st)[2]["n_frontier"] == 0                               # all free: no frontier at the box's faces
    st[1:3, 1:3, 1:3] = UNKNOWN
    c, vox, n = run(st)
    assert n["n_frontier"] == 24 and n["n_components"] == 1 and c["n_faces"].tolist() == [24]
    assert c["open"].tolist() == [[0, 0, 0]] and c["lo"].tolist() == [[0, 0, 0]] and c["hi"].tolist() == [[3, 3, 3]]


def test_uniform_grids_and_one_voxel_axes():
    for shape in [(1, 1, 1), (1, 1, 7), (1, 5, 1), (6, 1, 1), (4, 4, 4)]:
        for v in (UNKNOWN, OCCUPIED, FREE):
            c, vox, n = run(np.full(shape, v, np.uint8))
            assert len(c) == 0 and len(vox) == 0 and n.tolist() == (0, 0, 0, 0)
    row = np.array([[[FREE, UNKNOWN, FREE, FREE, UNKNOWN]]], np.uint8)   # a 5 x 1 x 1 grid
    c, vox, n = run(row)
    assert c["first"].tolist() == [0, 2] and c["n_voxels"].tolist() == [1, 2] and vox.tolist() == [0, 2, 3]
    assert c["open"][:, 0].tolist() == [1, 0] and c["n_faces"].tolist() == [1, 2]


def test_checkerboard_is_one_component():
    z, y, x = np.indices((6, 7, 8))
    st = np.where((x + y + z) % 2 == 0, FREE, UNKNOWN).astype(np.uint8)
    c, vox, n = run(st)
    assert n["n_frontier"] == int((st == FREE).sum()) and n["n_components"] == 1
    assert c["first"].tolist() == [0] and vox.tolist() == np.flatnonzero(st.reshape(-1) == FREE).tolist()
    same(run(st, m=2, mc=1, mv=10), bfs_model(st, (0, 0, 0), 0.2, 2, 1, 10))


def serpentine(nx, ny, nz):
    """Free rows along x on every other (y, z) line, joined at alternating ends into one path through the whole grid;
    everything else unknown."""
    st = np.full((nz, ny, nx), UNKNOWN, np.uint8)
    lines = [(y, z) for z in range(0, nz, 2) for y in (range(0, ny, 2) if z // 2 % 2 == 0 else range(ny - 1 - (ny - 1) % 2, -1, -2))]
    for k, (y, z) in enumerate(lines):
        st[z, y, :] = FREE
        if k + 1 < len(lines):
            y2, z2 = lines[k + 1]
            x = nx - 1 if k % 2 == 0 else 0
            if z2 == z:
                st[z, y + 1 if y2 > y else y - 1, x] = FREE
            else:
                st[z + 1, y, x] = FREE
    return st


def test_serpentine_fills_the_grid():
    st = serpentine(9, 7, 5)
    c, vox, n = run(st)
    assert n["n_components"] == 1 and n["n_frontier"] == int((st == FREE).sum())
    same(run(st, (2, -4, 1), 0.1), bfs_model(st, (2, -4, 1), 0.1, 1, BIG, BIG))


def test_centroid_sums_order_and_capacity_cuts():
    rng = np.random.default_rng(3)
    st = rng.choice(3, size=(8, 9, 10), p=(0.3, 0.5, 0.2)).astype(np.uint8)
    c, vox, n = run(st, (-7, 11, 3), 0.15)
    assert n["n_clusters"] > 5 and (np.diff(c["first"]) > 0).all()
    v = np.float64(np.float32(0.15))
    for r in c:
        mem = vox[r["offset"]:r["offset"] + r["n_voxels"]]
        xyz = np.stack([mem % 10, mem // 10 % 9, mem // 90], axis=1)
        assert (np.diff(mem) > 0).all() and mem[0] == r["first"]
        want = (xyz.sum(axis=0).astype(np.float64) / np.float64(len(mem)) + (np.array([-7, 11, 3], np.float64) + 0.5)) * v
        assert r["centroid"].tobytes() == want.tobytes()
    # the voxel cut in the middle of a cluster: offset -1 from that cluster on, the list a prefix of whole clusters
    big = int(np.argmax(c["n_voxels"] > 1))
    cut = int(c["offset"][big]) + 1
    cc, vv, nn = run(st, (-7, 11, 3), 0.15, mv=cut)
    assert cc["offset"][:big].tolist() == c["offset"][:big].tolist() and (cc["offset"][big:] == -1).all()
    assert vv.tolist() == vox[:c["offset"][big]].tolist() and nn["n_listed"] == c["offset"][big]
    # the cluster cut: the table holds the first clusters, the counts report all of them
    cc, vv, nn = run(st, (-7, 11, 3), 0.15, mc=3)
    assert cc.tobytes() == c[:3].tobytes() and nn["n_clusters"] == n["n_clusters"] and len(vv) == c["n_voxels"][:3].sum()
    # min_voxels filters after the components are counted
    cc, vv, nn = run(st, m=3)
    assert nn["n_components"] == n["n_components"] and nn["n_clusters"] == int((c["n_voxels"] >= 3).sum())
    assert frontier_mask(st).sum() == n["n_frontier"]
