"""The tour model of oracle/pyoracle_tour (DESIGN.md §8.14) on the CPU: the order is a permutation of the included sites
from site 0 and its cost an independent recomputation; every converged start is a local optimum, checked by applying
every 2-opt and Or-opt move and recomputing the whole tour (which also checks the O(1) deltas); no start beats the
Held-Karp optimum, and for m <= 4 a converged start equals it; hand cases; the bounds."""
import numpy as np
import pytest

import pyoracle_reach as R
import pyoracle_reach_matrix as RM
import pyoracle_tour as T
from densesurfelmapping_b200 import capi
from planner_scenes import metric_matrix, random_matrix

INF = T.INF


def recost(M, open_, order):
    """The tour's cost and legs priced P, leg by leg from the definition."""
    c = k = 0
    m = len(order)
    for a, b in zip(order, list(order[1:]) + [order[0]]):
        if a == b or (open_ and b == 0):
            continue
        x = int(M[a][b])
        c += T.P if x == INF else x
        k += x == INF
    return c, k


def every_move(m):
    for i in range(1, m - 1):
        for j in range(i + 1, m):
            yield T.code_2opt(i, j)
    for i in range(1, m):
        for L in (1, 2, 3):
            if i + L - 1 > m - 1:
                continue
            for q in range(m):
                if not i - 1 <= q <= i + L - 1:
                    yield T.code_or(i, L, q)


def held_karp(W, inc):
    """The least cost of a tour over the included sites from site 0 (W already holds the open rule)."""
    rest = [int(j) for j in inc if j != 0]
    k = len(rest)
    if k == 0:
        return 0
    Wr = W[np.ix_(rest, rest)]
    dp = np.full((1 << k, k), np.iinfo(np.int64).max // 4, np.int64)
    for j in range(k):
        dp[1 << j, j] = W[0, rest[j]]
    for mask in range(1, 1 << k):
        ends = [j for j in range(k) if mask >> j & 1]
        if len(ends) < 2:
            continue
        for j in ends:
            prev = mask ^ (1 << j)
            ks = [x for x in ends if x != j]
            dp[mask, j] = min(dp[prev, x] + Wr[x, j] for x in ks)
    return int(min(dp[(1 << k) - 1, j] + W[rest[j], 0] for j in range(k)))


def check(M, open_, n_starts, max_passes, seed, optimum=False):
    info, starts, order = T.tour(M, open_, n_starts, max_passes, seed)
    inc = T.included(M)
    m = len(inc)
    W = T.weights(M, open_)
    o = order[:m]
    assert o[0] == 0 and sorted(o.tolist()) == inc.tolist() and (order[m:] == -1).all()
    c, k = recost(M, open_, o.tolist())
    assert (info["best_cost"], info["n_infinite"], info["n_included"]) == (c, k, m)
    s = int(np.lexsort((np.arange(n_starts), starts["cost"]))[0])
    assert info["best_start"] == s and starts["cost"][s] == c
    assert ((starts["passes"] < max_passes) == (starts["converged"] == 1)).all()
    for si in range(n_starts):
        t, cs, p, conv = T.search(W, inc, si, seed, max_passes)
        assert (cs, p, conv) == tuple(starts[si].tolist()) and recost(M, open_, t.tolist())[0] == cs
        if conv:
            for code in every_move(m):
                assert T.cost(W, T.apply(t, code)) >= cs, (si, T.decode(code))
    if optimum:
        hk = held_karp(W, inc)
        assert (starts["cost"] >= hk).all()
        if m <= 4:
            assert all(x >= hk and (not conv or x == hk) for x, conv in zip(starts["cost"], starts["converged"]))
    return info, starts, order


@pytest.mark.parametrize("seed", range(6))
def test_random_against_held_karp(seed):
    rng = np.random.default_rng(seed)
    for n in (1, 2, 3, 4, 5, 7, 9, 12):
        for open_ in (0, 1):
            for p_inf in (0.0, 0.2):
                M = random_matrix(n, rng, p_inf)
                check(M, open_, 6, 64, seed * 100 + n, optimum=True)
            check(metric_matrix(n, rng), open_, 4, 64, seed, optimum=True)


def test_larger_instances_are_local_optima():
    rng = np.random.default_rng(11)
    for n, p_inf, sym in [(17, 0.0, False), (24, 0.1, False), (33, 0.0, True), (40, 0.02, False)]:
        for open_ in (0, 1):
            check(random_matrix(n, rng, p_inf, sym), open_, 3, 1000, n)
    check(metric_matrix(48, rng), 1, 2, 1000, 5)


def test_deltas_equal_recomputed_costs():
    """moves() prices every move of a tour by its O(1) formulas; each equals the recomputed cost difference."""
    rng = np.random.default_rng(3)
    for n in range(1, 11):
        for open_ in (0, 1):
            M = random_matrix(n, rng, 0.15)
            W = T.weights(M, open_)
            inc = T.included(M)
            t = T.construct(W, inc, 1, 9)
            d, c = T.moves(W, t)
            assert sorted(c.tolist()) == sorted(every_move(len(t)))
            for dd, cc in zip(d.tolist(), c.tolist()):
                t2 = T.apply(t, cc)
                assert t2[0] == 0 and sorted(t2.tolist()) == sorted(t.tolist())
                assert T.cost(W, t2) - T.cost(W, t) == dd, T.decode(cc)


def test_a_line_open_and_closed():
    """Sites on a line at 0, 3, 1, 2 (site order): the open path walks outward once, the closed tour comes back."""
    x = np.array([0, 3, 1, 2])
    M = np.abs(x[:, None] - x[None]).astype(np.uint32)
    info, starts, order = check(M, 1, 4, 16, 1, optimum=True)
    assert order.tolist() == [0, 2, 3, 1] and info["best_cost"] == 3
    info, starts, order = check(M, 0, 4, 16, 1, optimum=True)
    assert order.tolist() == [0, 2, 3, 1] and info["best_cost"] == 6
    assert (starts["converged"] == 1).all()


def test_excluded_sites_and_the_smallest_tours():
    rng = np.random.default_rng(4)
    M = random_matrix(6, rng)
    M[0, 2] = M[0, 5] = INF                                    # sites 2 and 5 unreachable from the robot
    info, _, order = check(M, 0, 3, 16, 2, optimum=True)
    assert info["n_included"] == 4 and order.tolist()[4:] == [-1, -1] and not {2, 5} & set(order[:4].tolist())
    M0 = np.full((5, 5), INF, np.uint32)                       # site 0 of status != 0 in a matrix job: m = 1
    info, starts, order = check(M0, 1, 2, 8, 0)
    assert info["n_included"] == 1 and order.tolist() == [0, -1, -1, -1, -1] and info["best_cost"] == 0
    assert (starts["passes"] == 0).all() and (starts["converged"] == 1).all()
    info, starts, order = check(np.array([[0, 7], [5, 0]], np.uint32), 0, 2, 8, 0, optimum=True)   # m = 2
    assert order.tolist() == [0, 1] and info["best_cost"] == 12 and (starts["passes"] == 0).all()
    info, _, _ = check(np.array([[0, 7], [INF, 0]], np.uint32), 1, 1, 8, 0)                        # the way back is free
    assert info["best_cost"] == 7 and info["n_infinite"] == 0
    info, _, _ = check(np.zeros((1, 1), np.uint32), 0, 1, 0, 0)                                     # n = 1
    assert info["n_included"] == 1 and info["best_cost"] == 0


def test_legs_without_a_path_are_priced_and_counted():
    """Two groups reachable from the robot but not from each other: every tour crosses between them once, without a path."""
    M = np.full((5, 5), INF, np.uint32)
    M[0, :] = [0, 1, 2, 1, 2]
    for g in ([1, 2], [3, 4]):
        for a in g:
            for b in g:
                M[a, b] = 0 if a == b else 1
    M[1:, 0] = 1
    info, starts, order = check(M, 0, 4, 16, 7, optimum=True)
    assert info["n_infinite"] == 1 and info["best_cost"] == T.P + 1 + 1 + 1 + 1
    info, _, _ = check(M, 1, 4, 16, 7, optimum=True)
    assert info["n_infinite"] == 1 and info["best_cost"] == T.P + 1 + 1 + 1


def test_an_all_equal_matrix():
    """Ties go to the lowest index: start 0 is 0, 1, 2, ... and no move improves it."""
    M = np.full((9, 9), 5, np.uint32)
    np.fill_diagonal(M, 0)
    info, starts, order = check(M, 0, 5, 16, 3)
    assert order.tolist() == list(range(9)) and info["best_start"] == 0 and info["best_cost"] == 45
    assert (starts["passes"] == 0).all() and (starts["converged"] == 1).all() and (starts["cost"] == 45).all()


def test_passes_zero_and_a_pass_cut():
    rng = np.random.default_rng(5)
    M = random_matrix(30, rng)
    W = T.weights(M, 0)
    inc = T.included(M)
    _, full, _ = check(M, 0, 3, 1000, 1)
    assert (full["converged"] == 1).all() and (full["passes"] > 2).all()
    _, none, _ = check(M, 0, 3, 0, 1)
    assert (none["passes"] == 0).all() and (none["converged"] == 0).all()
    assert [T.cost(W, T.construct(W, inc, s, 1)) for s in range(3)] == none["cost"].tolist()
    _, cut, _ = check(M, 0, 3, 2, 1)
    assert (cut["passes"] == 2).all() and (cut["converged"] == 0).all()
    assert (cut["cost"] < none["cost"]).all() and (cut["cost"] >= full["cost"]).all()


def test_seeds():
    """Start 0 does not depend on the seed; the other starts do, and the splitmix64 draw is the published one."""
    assert T.splitmix64(0) == 0xE220A8397B1DCDAF and T.splitmix64(1) == 0x910A2DEC89025CC1
    rng = np.random.default_rng(6)
    M = random_matrix(40, rng)
    a = T.tour(M, 1, 8, 0, 1)[1]
    b = T.tour(M, 1, 8, 0, 2)[1]
    assert a["cost"][0] == b["cost"][0] and (a["cost"][1:] != b["cost"][1:]).any()
    W, inc = T.weights(M, 1), T.included(M)
    assert (T.construct(W, inc, 0, 1) == T.construct(W, inc, 0, 1 << 63)).all()


def test_a_matrix_job_output_as_it_stands():
    """The matrix model's output on a grid with a wall, an unreachable site and one outside the grid, handed over
    unchanged: sites of status != 0 and sites without a path from the robot fall out."""
    st = np.full((3, 10, 12), R.FREE, np.uint8)
    st[:, :, 6] = R.OCCUPIED
    st[:, 9, 6] = R.FREE
    st[:, 4, 9:] = R.OCCUPIED
    st[:, 0:4, 10] = R.OCCUPIED
    v = 0.5
    pts = [((c[0] + 0.5) * v, (c[1] + 0.5) * v, (c[2] + 0.5) * v)
           for c in [(1, 1, 1), (3, 8, 0), (9, 2, 1), (8, 8, 2), (11, 1, 1), (40, 0, 0), (5, 0, 0)]]
    info, sites, M = RM.matrix(st, np.full(st.shape, np.inf, np.float32), (0, 0, 0), v, pts, 0.0, 0, 1000)
    assert info["status"] == 0 and sites["status"][5] == 1 and M[0, 4] == INF
    for open_ in (0, 1):
        ti, _, order = check(M, open_, 4, 64, 0, optimum=True)
        assert ti["n_included"] == 5 and set(order[:5].tolist()) == {0, 1, 2, 3, 6} and ti["n_infinite"] == 0


def test_bounds():
    assert T.valid(1, 0, 1, 0) and T.valid(1024, 1, 1024, 0) and T.valid(1024, 0, 1, 4096) and T.valid(64, 0, 1024, 1024)
    for n, o, k, p in [(0, 0, 1, 1), (1025, 0, 1, 1), (4, 2, 1, 1), (4, -1, 1, 1), (4, 0, 0, 1), (4, 0, 1025, 1),
                       (4, 0, 1, -1), (4, 0, 1, 65537), (1024, 0, 1, 4097), (1024, 0, 2, 2049), (64, 0, 1024, 1025)]:
        assert not T.valid(n, o, k, p), (n, o, k, p)
    assert not T.valid(9, 0, 1, 1, max_sites=8) and not T.valid(1, 0, 5, 1, max_starts=4)
    assert 1024 * 1024 * 4096 == T.MAX_WORK and T.P > 1024 * (INF - 1)    # P exceeds any sum of 1024 finite legs
    lib = capi.load_library()                                  # the refusals the library makes without a device
    m = np.zeros((1, 1), np.uint32)
    assert lib.dsm_tour_enable(None, 1, 1) == -1
    assert lib.dsm_tour_enqueue(None, m.ctypes.data, 1, 0, 1, 0, 0) == -1
    assert lib.dsm_tour_wait(None, None, None, None) == -1

