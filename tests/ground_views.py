"""Scenes and camera rotations for the ground viewpoint tests (DESIGN.md §8.23): ground planes on any up axis with boxes
and unsupported holes whose borders are frontiers, rotations that keep the camera upright along that axis, and the
hand scenes whose answer is known (a frontier over a pit behind a low wall, seen only from a high eye; a frontier behind
a full-height wall, seen around its end)."""
import numpy as np

import pyoracle_gain as G
import pyoracle_reach_terrain as RT
from pyoracle_field_known import FREE, OCCUPIED, UNKNOWN


def scene(rng, shape, up, p_box=0.06, p_hole=0.03):
    """A state grid [nz][ny][nx] of grid `shape` (nx, ny, nz): a flat ground a third of the way up the up axis, boxes
    three voxels high and holes without support (unknown columns)."""
    a = abs(up) - 1
    h0, h1 = RT.plane_axes(up)
    n_a = shape[a]
    g = np.full((shape[h1], shape[h0]), n_a // 3)
    g[rng.random(g.shape) < p_box] += 3
    k = np.arange(n_a)
    up_k = (k if up > 0 else n_a - 1 - k)[None, None, :]
    col = np.where(up_k < g[..., None], UNKNOWN, np.where(up_k == g[..., None], OCCUPIED, FREE)).astype(np.uint8)
    col[rng.random(g.shape) < p_hole] = UNKNOWN
    pos = {h1: 0, h0: 1, a: 2}
    return np.ascontiguousarray(np.transpose(col, (pos[2], pos[1], pos[0])))


def rotations(up, n_yaw, pitches=(0.0,)):
    """(n, 9) row-major camera-to-world rotations of an upright camera (x right, y down, z forward) on up axis `up`:
    n_yaw headings in the ground plane, yaw 0 along the lower in-plane axis, at each pitch (radians, up positive)."""
    a = abs(up) - 1
    h0, h1 = RT.plane_axes(up)
    U = np.zeros(3)
    U[a] = np.sign(up)
    out = []
    for p in pitches:
        for k in range(n_yaw):
            yaw = 2.0 * np.pi * k / n_yaw
            fh = np.zeros(3)
            fh[h0], fh[h1] = np.cos(yaw), np.sin(yaw)
            f = np.cos(p) * fh + np.sin(p) * U
            r = np.cross(-U, fh)
            d = np.cross(f, r)
            out.append(np.stack([r, d, f], axis=1).reshape(9))
    return np.array(out)


WIDE = G.Camera(1.0, 1.0, 1.0, 1.0, 2, 2, 3.0, 1)   # a 90-degree square cone out to 3 m (15 voxels of 0.2 m)


def pit_behind_wall(wall_top, gap, shape=(14, 8, 12)):
    """A z-up scene (up = +3) [nz][ny][nx]: an occupied floor at z = 0 under free space for x <= 5; a wall at x = 6 from
    z = 1 to wall_top for y below ny - gap (the floor runs through the gap); behind it, x >= 7, a pit of unknown space up
    to z = 0 under free space, so the free layer z = 1 over it is one frontier cluster.  With headroom 7 only the floor
    (and the gap) has support."""
    nx, ny, nz = shape
    st = np.full((nz, ny, nx), FREE, np.uint8)
    st[0, :, :7] = OCCUPIED
    st[0, :, 7:] = UNKNOWN
    st[1:wall_top + 1, :ny - gap, 6] = OCCUPIED
    return st


def shelf_behind_wall(shape=(14, 6, 12)):
    """A z-up scene: the floor at z = 0 for x <= 5, a wall at x = 6 up to z = 6, and behind it a shelf of unknown space up
    to z = 5, so the frontier is the free layer z = 6 on the shelf: a camera at z <= 6 sees it only through the wall, one
    at z >= 7 over it.  With headroom 8 the wall has no support (5 free voxels above it)."""
    nx, ny, nz = shape
    st = np.full((nz, ny, nx), FREE, np.uint8)
    st[0, :, :6] = OCCUPIED
    st[0:7, :, 6] = OCCUPIED
    st[0:6, :, 7:] = UNKNOWN
    return st
