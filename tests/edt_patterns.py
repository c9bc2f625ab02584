"""Crafted site grids for the exact distance transform of csrc/dsm_field.cu (DESIGN.md §8.7), shared by the CPU proof of
the envelope's branches (tests/test_field_edt_model.py) and the device tests (tests/test_gpu_field_edt.py), so the
device gets exactly the inputs the CPU test proved.

A plane pattern is a bool site mask [L][L] indexed [b][a]: `a` is the earlier of the plane's two axes in pass order
(x, then y, then z) and `b` the later one, so the envelope pass along `b` sees f(a, b) = (a - nearest site of row b)^2
on its line at `a`.  `grid` lays a plane into a 3-D grid with one short axis, the plane repeated along it; the short
axis's own pass then leaves every value alone."""
import numpy as np

L = 1024   # the longest line dsm_field_enable accepts
WIDE = [(L, L, 2), (L, 2, L), (2, L, L)]   # the wide planes: (nx, ny, nz), one short axis


def column(n=L):
    """Sites at a = 0 in every row: f = a^2 is constant along every line, (n - 1)^2 on the far one, and no entry ever
    leaves the envelope (a full envelope of n entries)."""
    m = np.zeros((n, n), bool)
    m[:, 0] = True
    return m


def fan(n=L, k=37):
    """The site of row b at a = k b mod n: drops (a separator at or beyond the line's end), pops that leave entries
    behind, and exact separators."""
    m = np.zeros((n, n), bool)
    b = np.arange(n)
    m[b, (k * b) % n] = True
    return m


def staircase(n=L):
    """The site of row b at a = n - 1 - b: on the line at a = 0, f = (n - 1 - b)^2 falls along the line, and each new
    site of its first half pops the envelope down to empty."""
    m = np.zeros((n, n), bool)
    b = np.arange(n)
    m[b, n - 1 - b] = True
    return m


def tie(n=L):
    """Row 0's site two voxels off the line at a = 0 (f(0) = 4) and row 2's on it (f(2) = 0): at t_top = 0 the new
    parabola equals the top entry, which stays (the pop test is strict), and the separator is exact."""
    m = np.zeros((n, n), bool)
    m[0, 2] = True
    m[2, 0] = True
    return m


def corner(n=L):
    """One site at a = b = 0: d2 = 2 (n - 1)^2 at the plane's far corner, and every row but row 0 is an empty line.  In
    (L, L, 2) the z pass's packed word carries f = 2 (n - 1)^2."""
    m = np.zeros((n, n), bool)
    m[0, 0] = True
    return m


PLANES = {"column": column, "fan": fan, "staircase": staircase, "tie": tie, "corner": corner}


def long_axes(shape):
    """(a, b): the plane's axes (0 x, 1 y, 2 z) of a shape with one short axis, a before b in pass order."""
    a, b = [k for k in range(3) if shape[k] > 2]
    return a, b


def grid(plane, shape):
    """The site mask [nz][ny][nx] of a plane pattern (a mask [L][L] indexed [b][a]) on a shape of WIDE."""
    a, b = long_axes(shape)
    nx, ny, nz = shape
    out = np.zeros((nz, ny, nx), bool)
    idx = np.indices((nz, ny, nx))        # idx[2 - k] is the coordinate along axis k
    out[...] = plane[idx[2 - b], idx[2 - a]]
    return out


def corners_and_centre(shape):
    """The nine single-site masks [nz][ny][nx]: each of the eight corners, then the centre."""
    nx, ny, nz = shape
    out = []
    for z in (0, nz - 1):
        for y in (0, ny - 1):
            for x in (0, nx - 1):
                out.append((x, y, z))
    out.append((nx // 2, ny // 2, nz // 2))
    masks = []
    for x, y, z in out:
        m = np.zeros((nz, ny, nx), bool)
        m[z, y, x] = True
        masks.append(m)
    return masks


def line_ends(shape):
    """Sites at both ends of every line along the shape's longest axis."""
    nx, ny, nz = shape
    m = np.zeros((nz, ny, nx), bool)
    k = int(np.argmax(shape))
    sl = [slice(None)] * 3
    for end in (0, shape[k] - 1):
        sl[2 - k] = end
        m[tuple(sl)] = True
    return m


def random_sites(shape, density, rng):
    """Sites at `density` (at least one)."""
    nx, ny, nz = shape
    m = rng.random((nz, ny, nx)) < density
    if not m.any():
        m[tuple(rng.integers(0, n) for n in (nz, ny, nx))] = True
    return m
