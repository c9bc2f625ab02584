"""The grids, poses, rotations and matrices that more than one planner test builds: the model tests on the CPU and the
GPU tests that hold the device to those models.  CPU only; every scene is a pure function of its arguments."""
import numpy as np

import pyoracle_gain as G
import pyoracle_tour as TM
import pyoracle_viewpoint as V
from pyoracle_field_known import FREE, OCCUPIED, UNKNOWN


# ---- state grids [nz][ny][nx] ----
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


def maze(n, seed):
    """A perfect maze on an n x n lattice of cells, two voxels per cell, two voxels tall: one path between any two cells."""
    rng = np.random.default_rng(seed)
    st = np.full((2, 2 * n + 1, 2 * n + 1), OCCUPIED, np.uint8)
    seen = np.zeros((n, n), bool)
    stack = [(0, 0)]
    seen[0, 0] = True
    st[:, 1, 1] = FREE
    while stack:
        x, y = stack[-1]
        nb = [(x + dx, y + dy) for dx, dy in ((1, 0), (-1, 0), (0, 1), (0, -1)) if 0 <= x + dx < n and 0 <= y + dy < n and not seen[y + dy, x + dx]]
        if not nb:
            stack.pop()
            continue
        a, b = nb[rng.integers(len(nb))]
        seen[b, a] = True
        st[:, 2 * b + 1, 2 * a + 1] = FREE
        st[:, y + b + 1, x + a + 1] = FREE
        stack.append((a, b))
    return st


def wall_scene(kind):
    st = np.full((5, 5, 12), FREE, np.uint8)
    st[:, :, 6] = kind
    return st


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


def scene(rng, shape, n_blobs=6, p_occupied=0.04):
    """A state grid [nz][ny][nx]: free space with scattered occupied voxels and n_blobs unknown boxes, each bordered by
    its own frontier clusters."""
    nx, ny, nz = shape
    st = np.where(rng.random((nz, ny, nx)) < p_occupied, OCCUPIED, FREE).astype(np.uint8)
    for _ in range(n_blobs):
        a = [int(rng.integers(0, n)) for n in (nx, ny, nz)]
        b = [min(n, x + int(rng.integers(1, 4))) for x, n in zip(a, (nx, ny, nz))]
        st[a[2]:b[2], a[1]:b[1], a[0]:b[0]] = UNKNOWN
    return st


def open_room():
    """A free room 12x12x3 whose +y wall is unknown: one flat cluster along the wall."""
    st = np.full((3, 13, 12), FREE, np.uint8)
    st[:, 12, :] = UNKNOWN
    return st


# ---- camera poses (12 doubles, row-major [R | t]) and rotations (9 doubles, row-major) ----
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


def symmetric_views(n, nz, voxel):
    h = n // 2
    t = G.centres([(h, h, nz // 2)], (0, 0, 0), voxel)[0]
    return t, [yaw_pose(k, t) for k in range(4)]


def rotation(yaw, pitch=0.0):
    """The row-major camera-to-world 3x3 of a camera looking along yaw (from +x toward +y) and pitch (up), x right, y
    down, z forward."""
    f = np.array([np.cos(pitch) * np.cos(yaw), np.cos(pitch) * np.sin(yaw), np.sin(pitch)])
    r = np.array([np.sin(yaw), -np.cos(yaw), 0.0])
    return np.stack([r, np.cross(f, r), f], axis=1).reshape(9)


def rotations(n_yaw, pitches=(0.0,)):
    """A yaw sweep of n_yaw headings at each pitch, (n_yaw len(pitches), 9)."""
    return np.stack([rotation(2 * np.pi * k / n_yaw, p) for p in pitches for k in range(n_yaw)])


def params(r_min=1, r_max=3, dz_max=1, stride=1, max_samples=4096, min_seen=0, top_k=4, with_reach=0, radius=0.0):
    return V.Params(r_min, r_max, dz_max, stride, max_samples, min_seen, top_k, with_reach, radius)


# ---- travel-cost matrices ----
def random_matrix(n, rng, p_inf=0.0, symmetric=False, hi=1000):
    M = rng.integers(0, hi, (n, n)).astype(np.uint32)
    if symmetric:
        M = np.minimum(M, M.T)
    if p_inf:
        M[rng.random((n, n)) < p_inf] = TM.INF
    np.fill_diagonal(M, 0)
    return M


def metric_matrix(n, rng, stretch=1.3):
    """Euclidean distances between random points, each entry stretched by a factor in [1, stretch]: asymmetric, close
    to metric, as travel costs through free space are."""
    p = rng.uniform(0, 100, (n, 2))
    d = np.linalg.norm(p[:, None] - p[None], axis=-1)
    return np.round(d * rng.uniform(1.0, stretch, (n, n)) * 10).astype(np.uint32)
