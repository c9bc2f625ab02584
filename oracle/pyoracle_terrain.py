"""The terrain job of dsm_terrain_* (DESIGN.md §8.20) restated in numpy: per column of a known field's state grid along
the up axis, the uppermost occupied voxel with `headroom` observed free voxels above it, the largest level difference to
its supported 8-neighbours, the status in the field's state codes and the clearance to the nearest cell that is not
traversable, on the field grid with the up axis collapsed."""
import numpy as np

import pyoracle_field_known
from pyoracle_field_known import FREE, OCCUPIED, UNKNOWN

MAX_STEP = 1023
UPS = (1, -1, 2, -2, 3, -3)
INFO_DTYPE = np.dtype([("origin", "<i4", 3), ("m", "<i4", 3), ("up", "<i4"), ("headroom", "<i4"), ("max_step", "<i4"),
                       ("n_support", "<i4"), ("n_blocked", "<i4"), ("n_traversable", "<i4"), ("reserved", "<i4", 4)])
NO_SUPPORT, BLOCKED, TRAVERSABLE = UNKNOWN, OCCUPIED, FREE


def check_enable(up):
    """Raises ValueError where dsm_terrain_enable returns DSM_E_INVALID."""
    if up not in UPS:
        raise ValueError("up outside {+-1, +-2, +-3}")


def check_request(shape, up, headroom, max_step):
    """Raises ValueError where dsm_terrain_enqueue returns DSM_E_INVALID; shape is the field's (nx, ny, nz)."""
    check_enable(up)
    n_a = shape[abs(up) - 1]
    if not 1 <= headroom <= n_a - 1:
        raise ValueError("headroom outside [1, n_a - 1]")
    if not 0 <= max_step <= MAX_STEP:
        raise ValueError("max_step outside [0, 1023]")


def _columns(state, up):
    """state [nz][ny][nx] as [cells of the terrain grid, in its linear order][walk order from the top down], and the map
    from walk position to the coordinate k along the up axis."""
    a = abs(up) - 1
    axis = 2 - a                          # numpy axis of grid axis a
    cols = np.moveaxis(state, axis, -1)   # [..][k], the other axes in their order: the terrain grid's linear order
    n_a = cols.shape[-1]
    ks = np.arange(n_a)[::-1] if up > 0 else np.arange(n_a)
    return cols.reshape(-1, n_a)[:, ks], ks


def terrain_shape(shape, up):
    """m (m0, m1, m2) of a field grid (nx, ny, nz)."""
    m = list(shape)
    m[abs(up) - 1] = 1
    return tuple(m)


def levels(state, up, headroom):
    """int16 level per cell [m2][m1][m0]: the uppermost k with state[k] == OCCUPIED whose `headroom` voxels above lie
    in the grid and are all FREE, or -1."""
    nz, ny, nx = state.shape
    cols, ks = _columns(np.asarray(state, np.uint8), up)
    n_a = cols.shape[1]
    free = cols == FREE
    # run[j]: the consecutive free voxels directly above walk position j (those at walk positions < j)
    run = np.zeros(cols.shape, np.int64)
    for j in range(1, n_a):
        run[:, j] = np.where(free[:, j - 1], run[:, j - 1] + 1, 0)
    ok = (cols == OCCUPIED) & (run >= headroom)
    first = np.argmax(ok, axis=1)
    lev = np.where(ok.any(axis=1), ks[first], -1).astype(np.int16)
    m = terrain_shape((nx, ny, nz), up)
    return lev.reshape(m[2], m[1], m[0])


def steps(level, up):
    """(step, full) per cell: full the largest |level - level(n)| over the in-grid 8-neighbours in the two horizontal
    axes that have support (0 without any, and 0 on a cell without support); step = min(full, 255) as uint8."""
    a = abs(up) - 1
    lev = np.asarray(level, np.int64)
    plane = np.squeeze(lev, axis=2 - a)            # [h1][h0]
    H1, H0 = plane.shape
    pad = np.full((H1 + 2, H0 + 2), -1, np.int64)
    pad[1:-1, 1:-1] = plane
    full = np.zeros_like(plane)
    for d1 in (-1, 0, 1):
        for d0 in (-1, 0, 1):
            if d1 == 0 and d0 == 0:
                continue
            nb = pad[1 + d1:1 + d1 + H1, 1 + d0:1 + d0 + H0]
            full = np.maximum(full, np.where(nb >= 0, np.abs(plane - nb), 0))
    full = np.where(plane >= 0, full, 0)
    full = np.expand_dims(full, 2 - a).reshape(lev.shape)
    return np.minimum(full, 255).astype(np.uint8), full


def job(state, origin, voxel, up, headroom, max_step):
    """(info, level, status, step, clearance) of a terrain job on the state grid [nz][ny][nx] at `origin`, as
    dsm_terrain_wait returns them: a INFO_DTYPE record and the four planes [m2][m1][m0]."""
    state = np.asarray(state, np.uint8)
    nz, ny, nx = state.shape
    check_request((nx, ny, nz), up, headroom, max_step)
    lev = levels(state, up, headroom)
    step, full = steps(lev, up)
    status = np.where(lev < 0, NO_SUPPORT, np.where(full > max_step, BLOCKED, TRAVERSABLE)).astype(np.uint8)
    clearance, n_blocked, n_trav = pyoracle_field_known.state_field(status, voxel)
    info = np.zeros(1, INFO_DTYPE)[0]
    info["origin"] = origin
    info["m"] = terrain_shape((nx, ny, nz), up)
    info["up"], info["headroom"], info["max_step"] = up, headroom, max_step
    info["n_blocked"], info["n_traversable"] = n_blocked, n_trav
    info["n_support"] = n_blocked + n_trav
    return info, lev, status, step, clearance


def height(level, origin, voxel, up):
    """The supporting surface's height in metres along the up direction (float64, NaN without support):
    (o_a + k + 1) v for a positive up and -(o_a + k) v for a negative one."""
    a = abs(up) - 1
    k = np.asarray(level, np.float64)
    v = float(np.float32(voxel))
    h = (origin[a] + k + 1) * v if up > 0 else -(origin[a] + k) * v
    return np.where(k >= 0, h, np.nan)
