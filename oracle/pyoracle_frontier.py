"""The exploration frontiers of dsm_frontier_enqueue (DESIGN.md §8.10) restated in numpy and scipy: the frontier voxels of
a three-state grid, their 26-connected components (scipy.ndimage.label), the cluster records, the voxel list and the
counts, in the layout dsm_frontier_wait hands out."""
import numpy as np
from scipy import ndimage

UNKNOWN, OCCUPIED, FREE = 0, 1, 2
MAX_CAPACITY = 1 << 26   # DSM_FRONTIER_MAX_CAPACITY

CLUSTER_DTYPE = np.dtype([("n_voxels", "<i4"), ("first", "<i4"), ("offset", "<i4"), ("lo", "<i4", 3), ("hi", "<i4", 3),
                          ("reserved", "<i4"), ("n_faces", "<i8"), ("open", "<i8", 3), ("centroid", "<f8", 3)])
COUNTS_DTYPE = np.dtype([("n_frontier", "<i4"), ("n_components", "<i4"), ("n_clusters", "<i4"), ("n_listed", "<i4")])

# the six face neighbours as (axis of the [z][y][x] array, step) and the unit step's (x, y, z) component it adds to open
FACES = [(2, -1), (2, 1), (1, -1), (1, 1), (0, -1), (0, 1)]


def unknown_faces(state):
    """bool [6][nz][ny][nx]: the face neighbour of FACES[f] lies inside the grid and is unknown."""
    st = np.asarray(state)
    out = np.zeros((6,) + st.shape, bool)
    unk = st == UNKNOWN
    for f, (ax, step) in enumerate(FACES):
        n = st.shape[ax]
        src = [slice(None)] * 3
        dst = [slice(None)] * 3
        if step < 0:   # the neighbour at index - 1: voxels 1 .. n-1 see unk[0 .. n-2]
            dst[ax], src[ax] = slice(1, n), slice(0, n - 1)
        else:
            dst[ax], src[ax] = slice(0, n - 1), slice(1, n)
        out[f][tuple(dst)] = unk[tuple(src)]
    return out


def frontier_mask(state):
    """Free voxels with an unknown face neighbour inside the grid."""
    return (np.asarray(state) == FREE) & unknown_faces(state).any(axis=0)


def components(mask):
    """(label grid, count): 26-connected components numbered 1.. in ascending order of their lowest linear index."""
    return ndimage.label(mask, structure=np.ones((3, 3, 3), bool))


def frontiers(state, origin, voxel, min_voxels, max_clusters, max_voxels):
    """(clusters CLUSTER_DTYPE [min(n_clusters, max_clusters)], voxels int32 [n_listed], counts COUNTS_DTYPE record) of
    the state grid [nz][ny][nx] at integer origin (x, y, z) and voxel edge `voxel` (float32)."""
    st = np.asarray(state, np.uint8)
    nz, ny, nx = st.shape
    mask = frontier_mask(st)
    lab, n_comp = components(mask)
    flat = lab.reshape(-1)
    idx = np.flatnonzero(flat)                    # ascending linear indices of the frontier voxels
    comp = flat[idx].astype(np.int64) - 1
    count = np.bincount(comp, minlength=n_comp)
    keep = np.flatnonzero(count >= min_voxels)    # the clusters, in component order
    tab = keep[:max_clusters]
    out = np.zeros(len(tab), CLUSTER_DTYPE)
    slot = np.full(n_comp, -1, np.int64)
    slot[tab] = np.arange(len(tab))
    x, y, z = idx % nx, idx // nx % ny, idx // (nx * ny)
    xyz = np.stack([x, y, z], axis=1).astype(np.int64)
    faces = unknown_faces(st).reshape(6, -1)[:, idx]                   # [6][frontier voxel]
    n_faces = faces.sum(axis=0).astype(np.int64)
    opn = np.stack([faces[1].astype(np.int64) - faces[0], faces[3].astype(np.int64) - faces[2],
                    faces[5].astype(np.int64) - faces[4]], axis=1)
    s = slot[comp]
    m = s >= 0
    sm = s[m]
    n = count[tab].astype(np.int64)
    first = np.full(len(tab), np.iinfo(np.int64).max, np.int64)
    np.minimum.at(first, sm, idx[m])
    lo = np.full((len(tab), 3), np.iinfo(np.int64).max, np.int64)
    hi = np.full((len(tab), 3), -1, np.int64)
    sums = np.zeros((len(tab), 3), np.int64)
    opens = np.zeros((len(tab), 3), np.int64)
    nf = np.zeros(len(tab), np.int64)
    np.minimum.at(lo, sm, xyz[m])
    np.maximum.at(hi, sm, xyz[m])
    np.add.at(sums, sm, xyz[m])
    np.add.at(opens, sm, opn[m])
    np.add.at(nf, sm, n_faces[m])
    pre = np.concatenate([[0], np.cumsum(n)[:-1]]).astype(np.int64)
    listed = pre + n <= max_voxels
    out["n_voxels"] = n
    out["first"] = first
    out["offset"] = np.where(listed, pre, -1)
    out["lo"], out["hi"] = lo, hi
    out["n_faces"], out["open"] = nf, opens
    o = np.asarray(origin, np.int64).astype(np.float64)
    v = np.float64(np.float32(voxel))
    with np.errstate(invalid="ignore", divide="ignore"):
        out["centroid"] = (sums.astype(np.float64) / n[:, None].astype(np.float64) + (o + 0.5)) * v
    n_lc = int(listed.sum())                      # the listed clusters are a prefix of the table
    order = np.argsort(s[m], kind="stable")       # members grouped by slot, ascending within one
    members = idx[m][order]
    n_listed = int(n[:n_lc].sum())
    vox = members[:n_listed].astype(np.int32)
    counts = np.zeros((), COUNTS_DTYPE)
    counts["n_frontier"], counts["n_components"] = int(mask.sum()), n_comp
    counts["n_clusters"], counts["n_listed"] = len(keep), n_listed
    return out, vox, counts

