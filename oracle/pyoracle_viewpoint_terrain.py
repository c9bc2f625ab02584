"""The terrain viewpoint job of dsm_viewpoint_enqueue_terrain (DESIGN.md §8.23) restated by composing pyoracle_terrain's
planes, pyoracle_reach_terrain's column snap and cost plane, and pyoracle_viewpoint's offsets, samples and seen counts:
the viewpoint job of §8.15 on the plane (P, Q, 1) of a terrain job, each candidate cell's camera standing eye voxels
above its support, scored through the 3-D state grid the terrain job read."""
import numpy as np

import pyoracle_gain as G
import pyoracle_reach as R
import pyoracle_reach_terrain as RT
import pyoracle_viewpoint as V


def check_request(camera, voxel, rotations, clusters, params, eye, headroom, max_clusters, max_candidates):
    """Raises ValueError where dsm_viewpoint_enqueue_terrain returns DSM_E_INVALID: dsm_viewpoint_enqueue's checks, then
    dz_max != 0 and eye outside [1, headroom] of the terrain job."""
    V.check_request(camera, voxel, rotations, clusters, params, max_clusters, max_candidates)
    if V.Params(*params).dz_max != 0:
        raise ValueError("dz_max must be 0 on the terrain plane")
    if not 1 <= eye <= headroom:
        raise ValueError("eye outside [1, headroom]")


def centre_cell(centroid, origin, voxel, up):
    """int64 (p, q, 0): the centroid's column, reach's start snap floor(centroid_h / v) - o_h on the two in-plane axes."""
    h0, h1 = RT.plane_axes(up)
    return V.centre_voxel(RT.column_point(centroid, up, voxel), (origin[h0], origin[h1], 0), voxel)


def camera_voxel(p, q, level, up, eye):
    """int64 (3,): the field voxel of the camera over cell (p, q) of the level plane [Q][P]: (p, q) on the in-plane axes
    and level + eye (up > 0) or level - eye (up < 0) on the up axis."""
    h0, h1 = RT.plane_axes(up)
    out = np.zeros(3, np.int64)
    out[h0], out[h1] = p, q
    out[abs(up) - 1] = int(level[q, p]) + (eye if up > 0 else -eye)
    return out


def viewpoints(state, voxel, terrain, camera, rotations, clusters, params, eye, frontier, reach_cost=None):
    """(info INFO_DTYPE record, records CLUSTER_DTYPE (n,), slots VIEWPOINT_DTYPE (n, top_k)) of the job, as
    dsm_viewpoint_wait returns them after dsm_viewpoint_enqueue_terrain.  state: the known field's state grid [nz][ny][nx]
    the terrain job read; terrain: the (info, level, status, step, clearance) of pyoracle_terrain.job (or of the device);
    frontier: (table, voxel list) of a frontier job on that field; reach_cost: the terrain reach job's uint32 cost plane
    [m2][m1][m0] (needed with with_reach)."""
    p = V.Params(*params)
    st = np.asarray(state, np.uint8)
    nz, ny, nx = st.shape
    tinfo, level, status, _, clearance = terrain
    up, origin = int(tinfo["up"]), [int(x) for x in tinfo["origin"]]
    h0, h1 = RT.plane_axes(up)
    m = [int(x) for x in tinfo["m"]]
    P, Q = m[h0], m[h1]
    check_request(camera, voxel, rotations, clusters, params, eye, int(tinfo["headroom"]), V.MAX_CLUSTERS, V.MAX_CANDIDATES)
    lev = np.asarray(level, np.int64).reshape(Q, P)
    trav = R.traversable(np.asarray(status, np.uint8).reshape(1, Q, P), np.asarray(clearance, np.float32).reshape(1, Q, P), p.radius)[0]
    cost_plane = None if reach_cost is None else np.asarray(reach_cost, np.uint32).reshape(Q, P)
    table, vox = frontier
    rot = np.asarray(rotations, np.float64).reshape(-1, 9)
    cl = np.asarray(clusters, np.int64).reshape(-1)
    off = V.offsets(p)[:, :2]
    recs = np.zeros(len(cl), V.CLUSTER_DTYPE)
    slots = np.zeros((len(cl), p.top_k), V.VIEWPOINT_DTYPE)
    slots["voxel"], slots["offset"], slots["rotation"], slots["cost"] = -1, -1, -1, V.INF
    for i, c in enumerate(cl):
        r = recs[i]
        r["cluster"] = c
        r["status"] = 3 if c >= len(table) else 2 if table[c]["offset"] < 0 else 0
        if r["status"]:
            continue
        T = table[c]
        g = centre_cell(T["centroid"], origin, voxel, up)[:2]
        members = vox[T["offset"]:T["offset"] + T["n_voxels"]].astype(np.int64)
        mm = members[V.sample_positions(len(members), p.max_samples)]
        r["n_samples"] = len(mm)
        mc = G.centres(np.stack([mm % nx, mm // nx % ny, mm // (nx * ny)], 1), origin, voxel)
        cand = g + off
        inside = (cand[:, 0] >= 0) & (cand[:, 0] < P) & (cand[:, 1] >= 0) & (cand[:, 1] < Q)
        r["n_inside"] = inside.sum()
        ranked = []
        for j in np.flatnonzero(inside):
            x, y = (int(k) for k in cand[j])
            if not trav[y, x]:
                continue
            r["n_traversable"] += 1
            cost = V.INF
            if p.with_reach:
                cost = int(cost_plane[y, x])
                if cost == V.INF:
                    continue
            r["n_reached"] += 1
            t = G.centres([camera_voxel(x, y, lev, up, eye)], origin, voxel)[0]
            seen = V.seen_counts(st, origin, voxel, camera, rot, t, mc)
            best = int(np.argmax(seen))      # the first maximum: the lowest rotation on ties
            n_seen = int(seen[best])
            if n_seen >= max(1, p.min_seen):
                ranked.append((-n_seen, cost, int(j), best, y * P + x))
        ranked.sort()
        for k, (neg, cost, j, best, lin) in enumerate(ranked[:p.top_k]):
            slots[i, k] = (lin, j, best, -neg, cost, (0, 0, 0))
        r["n_viewpoints"] = min(len(ranked), p.top_k)
    info = np.zeros((), V.INFO_DTYPE)
    info["origin"] = np.asarray(origin, np.int32)
    info["n_clusters"], info["n_offsets"], info["n_rotations"], info["top_k"] = len(cl), len(off), len(rot), p.top_k
    info["unknown_blocks"], info["with_reach"], info["n_clusters_table"] = G.Camera(*camera).unknown_blocks, p.with_reach, len(table)
    return info, recs, slots


def camera_point(cell, terrain, voxel, eye):
    """fp64 (3,): the world point of a slot's camera, ((o_k + voxel_k) + 0.5) v of camera_voxel for cell q P + p."""
    tinfo, level = terrain[0], terrain[1]
    up = int(tinfo["up"])
    h0, h1 = RT.plane_axes(up)
    P, Q = int(tinfo["m"][h0]), int(tinfo["m"][h1])
    lev = np.asarray(level, np.int64).reshape(Q, P)
    return G.centres([camera_voxel(cell % P, cell // P, lev, up, eye)], [int(x) for x in tinfo["origin"]], voxel)[0]
