"""The exact distance transform of csrc/dsm_field.cu restated literally, one branch at a time: k_field_rows (the nearest
site to the left and to the right of every voxel, squared) and k_field_lines' lower envelope, with the packed word
f << 10 | u, the strict pop test, the recomputed t_top, the push or drop at w < len and the final walk.  The restatement
equals oracle/pyoracle_field.squared_distances and a brute-force minimum on random grids and lines, and every crafted
pattern of tests/edt_patterns.py reaches the branch it is built for on the lines it is built for.  tests/test_gpu_field_edt.py
feeds the device exactly these grids.

The floor correction of env_sep for a negative numerator never fires: after the pop loop the top entry is at least as
close as the new site at t_top >= 0, so the parabolas meet at or after t_top.  The counter `neg_floor` stays 0 here."""
from collections import Counter

import numpy as np
import pytest

import edt_patterns as P
import pyoracle_field

INF = 2 ** 31 - 1   # FIELD_INF
BRANCHES = ("full", "pop_empty", "pop_nonempty", "drop", "exact_sep", "tie", "empty")


def rows(sites):
    """k_field_rows on the bool sites [..., n] along the last axis: int64 squared distance to the nearest site at or left
    of x and at or right of x, INF when the row has none."""
    n = sites.shape[-1]
    x = np.arange(n)
    left = np.maximum.accumulate(np.where(sites, x, -1), axis=-1)
    right = np.flip(np.minimum.accumulate(np.flip(np.where(sites, x, INF), -1), axis=-1), -1)
    d = np.minimum(np.where(left >= 0, x - left, INF), np.where(right != INF, right - x, INF))
    return np.where(d == INF, INF, d * d).astype(np.int64)


def env_at(e, x):
    d = x - (e & 1023)
    return (e >> 10) + d * d


def env_sep(e, u, fu, c):
    s, fs = e & 1023, e >> 10
    num, den = u * u - s * s + fu - fs, 2 * (u - s)
    q = abs(num) // den * (1 if num >= 0 else -1)   # C's division truncates toward zero
    r = num - q * den
    c["exact_sep"] += r == 0
    if r != 0 and num < 0:
        c["neg_floor"] += 1
        return q - 1
    return q


def line(f, c):
    """k_field_lines on one line of f (ints, INF for none): the minimum of f(u) + (x - u)^2 at every x."""
    n = len(f)
    env = [0] * n
    top, t_top = -1, 0
    for u in range(n):
        fu = int(f[u])
        if fu == INF:
            continue
        popped = False
        while top >= 0:
            have, new = env_at(env[top], t_top), fu + (t_top - u) * (t_top - u)
            if not have > new:
                c["tie"] += have == new
                break
            top -= 1
            popped = True
            t_top = 1 + env_sep(env[top - 1], env[top] & 1023, env[top] >> 10, c) if top >= 1 else 0
        if popped:
            c["pop_empty" if top < 0 else "pop_nonempty"] += 1
        if top < 0:
            top, t_top = 0, 0
            env[0] = fu << 10 | u
        else:
            w = 1 + env_sep(env[top], u, fu, c)
            if w < n:
                top += 1
                t_top = w
                env[top] = fu << 10 | u
            else:
                c["drop"] += 1
    if top < 0:
        c["empty"] += 1
        return [INF] * n
    c["full"] += top + 1 == n
    out, k, cur = [], 0, env[0]
    for u in range(n):
        d = env_at(cur, u)
        while k < top:
            nxt = env[k + 1]
            dn = env_at(nxt, u)
            if dn > d:
                break
            k += 1
            cur, d = nxt, dn
        out.append(d)
    return out


def edt(sites, c):
    """The three passes on the sites [nz][ny][nx]: int64 d2, INF where the grid has no site."""
    d = rows(sites)
    nz, ny, nx = sites.shape
    for z in range(nz):
        for x in range(nx):
            d[z, :, x] = line(d[z, :, x], c)
    for y in range(ny):
        for x in range(nx):
            d[:, y, x] = line(d[:, y, x], c)
    return d


def oracle(sites):
    d2 = pyoracle_field.squared_distances(sites)
    return np.full(sites.shape, INF, np.int64) if d2 is None else d2


def brute_line(f):
    f = np.asarray(f, np.int64)
    u = np.flatnonzero(f != INF)
    if not len(u):
        return np.full(len(f), INF, np.int64)
    x = np.arange(len(f))
    return (f[u][None, :] + (x[:, None] - u[None, :]) ** 2).min(1)


@pytest.mark.parametrize("seed", range(30))
def test_random_grids_equal_the_oracle_and_the_brute_force_minimum(seed):
    rng = np.random.default_rng(seed)
    shape = tuple(int(s) for s in rng.integers(1, 14, 3))
    sites = rng.random(shape) < rng.choice([0.0, 0.005, 0.05, 0.3, 0.9])
    c = Counter()
    got = edt(sites, c)
    assert got.tolist() == oracle(sites).tolist()
    if sites.any():
        s = np.argwhere(sites)
        g = np.indices(shape).reshape(3, -1).T
        want = ((g[:, None, :] - s[None]) ** 2).sum(-1).min(1).reshape(shape)
        assert got.tolist() == want.tolist()
    assert c["neg_floor"] == 0


@pytest.mark.parametrize("n", [1, 2, 3, 31, 32, 33, 385, 1023, 1024])
def test_random_lines_equal_the_brute_force_minimum(n):
    """Lines of any f, up to the z pass's 2 * 1023^2, sparse and dense."""
    rng = np.random.default_rng(n)
    c = Counter()
    for density in (0.0, 0.01, 0.3, 1.0):
        for top in (4, 1023 ** 2, 2 * 1023 ** 2):
            f = np.where(rng.random(n) < density, rng.integers(0, top + 1, n), INF)
            assert line(f, c) == brute_line(f).tolist(), (density, top)
    assert c["neg_floor"] == 0
    if n >= 31:
        assert all(c[b] for b in ("pop_empty", "pop_nonempty", "drop", "exact_sep", "empty")), c


# the lines along b each plane pattern is built for, and the branches they must reach
BUILT_FOR = {
    "column": ([P.L - 1], ("full",)),
    "fan": ([0, 1, 500, P.L - 1], ("drop", "pop_nonempty", "exact_sep")),
    "staircase": ([0], ("pop_empty",)),
    "tie": ([0], ("tie", "exact_sep")),
    "corner": ([P.L - 1], ()),
}


@pytest.mark.parametrize("name", list(P.PLANES))
def test_each_pattern_reaches_its_branch(name):
    plane = P.PLANES[name]()
    f = rows(plane)                            # [b][a]: the values the pass along b reads
    want = oracle(plane)
    on, branches = BUILT_FOR[name]
    c = Counter()
    for a in on:
        assert line(f[:, a], c) == want[:, a].tolist(), a
    assert c["neg_floor"] == 0
    for b in branches:
        assert c[b] > 0, (name, b, c)
    if name == "column":
        assert c["full"] == 1 and (f[:, P.L - 1] == (P.L - 1) ** 2).all()
    if name == "staircase":
        assert c["pop_empty"] >= P.L // 2 - 1   # every site of the first half empties the envelope
    if name == "tie":
        assert f[0, 0] == 4 and f[2, 0] == 0 and c["tie"] == 1 and c["pop_empty"] == c["pop_nonempty"] == 0
    if name == "corner":
        assert want[P.L - 1, P.L - 1] == 2 * (P.L - 1) ** 2 and line(f[:, P.L - 1], c)[-1] == 2 * (P.L - 1) ** 2
    # a row with no site (every row but row 0 of the corner) is an empty line for an envelope pass along a
    empty = np.flatnonzero(~plane.any(1))
    if len(empty):
        e = Counter()
        assert line(f[empty[0]], e) == [INF] * P.L and e["empty"] == 1


def test_every_branch_is_reached():
    """Over all patterns: the branches the device tests rely on, each at least once."""
    c = Counter()
    for name, fn in P.PLANES.items():
        f = rows(fn())
        for a in BUILT_FOR[name][0]:
            line(f[:, a], c)
    line([INF] * 8, c)
    assert all(c[b] > 0 for b in BRANCHES), c
    assert c["neg_floor"] == 0


@pytest.mark.parametrize("shape", [(40, 40, 2), (40, 2, 40), (2, 40, 40)], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("name", list(P.PLANES))
def test_a_plane_laid_into_a_grid_keeps_its_distances(shape, name):
    """grid() repeats the plane along the short axis, whose own pass changes nothing: the 3-D transform is the plane's,
    repeated (shown at n = 40 through the literal passes)."""
    plane = P.PLANES[name](40)
    sites = P.grid(plane, shape)
    c = Counter()
    got = edt(sites, c)
    a, b = P.long_axes(shape)
    flat = oracle(plane)                         # [b][a]
    idx = np.indices(sites.shape)
    assert got.tolist() == flat[idx[2 - b], idx[2 - a]].tolist()
    assert got.tolist() == oracle(sites).tolist()


def test_crafted_sweep_patterns():
    """The axis sweep's patterns: nine single sites, line ends and random sites; each against the oracle."""
    rng = np.random.default_rng(7)
    for shape in [(33, 3, 5), (5, 33, 3), (3, 5, 33), (2, 1, 1), (1, 1, 1)]:
        masks = P.corners_and_centre(shape) + [P.line_ends(shape)]
        masks += [P.random_sites(shape, d, rng) for d in (1e-4, 1e-2, 0.3)]
        for m in masks:
            assert m.shape == shape[::-1] and m.any()
            assert edt(m, Counter()).tolist() == oracle(m).tolist()
    assert P.line_ends((5, 3, 1024))[[0, -1]].all() and not P.line_ends((5, 3, 1024))[1:-1].any()
