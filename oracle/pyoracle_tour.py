"""The tour job of dsm_tour_enqueue (DESIGN.md §8.14): a deterministic multi-start local search for the asymmetric TSP
over a travel-cost matrix, all in int64, in the layout dsm_tour_wait hands out.

Site 0 is the robot.  The included sites are site 0 and every j >= 1 with M[0][j] != UINT32_MAX.  A leg i -> j weighs
0 when i == j or (open and j == 0), else M[i][j], or P = 2^42 for UINT32_MAX.  Start s builds a tour greedily (start 0:
nearest neighbour; start s >= 1: one of the three nearest unvisited sites, drawn by splitmix64), then each pass applies
the least (delta, code) 2-opt or Or-opt move while its delta is negative."""
import numpy as np

MAX_SITES = 1024          # DSM_TOUR_MAX_SITES
MAX_STARTS = 1024         # DSM_TOUR_MAX_STARTS
MAX_PASSES = 65536        # DSM_TOUR_MAX_PASSES
MAX_WORK = 1 << 32        # DSM_TOUR_MAX_WORK: n_starts x max_passes x n^2
INF = 0xFFFFFFFF
P = 1 << 42               # DSM_TOUR_P: the weight of a leg without a path
M64 = (1 << 64) - 1
INFO_DTYPE = np.dtype([("n_sites", "<i4"), ("n_included", "<i4"), ("open", "<i4"), ("n_starts", "<i4"), ("max_passes", "<i4"),
                       ("best_start", "<i4"), ("best_cost", "<i8"), ("seed", "<u8"), ("n_infinite", "<i4"), ("reserved", "<i4", 5)])
START_DTYPE = np.dtype([("cost", "<i8"), ("passes", "<i4"), ("converged", "<i4")])


def splitmix64(x):
    """The splitmix64 generator's output for state x: the golden-ratio increment, then its finaliser."""
    z = (int(x) + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def valid(n, open_, n_starts, max_passes, max_sites=MAX_SITES, max_starts=MAX_STARTS):
    """The bounds of dsm_tour_enqueue: False where it returns DSM_E_INVALID."""
    return (1 <= n <= max_sites and 1 <= n_starts <= max_starts and open_ in (0, 1) and 0 <= max_passes <= MAX_PASSES
            and n_starts * max_passes * n * n <= MAX_WORK)


def included(M):
    """The included sites in index order: 0 and every j >= 1 with M[0][j] finite."""
    M = np.asarray(M, np.uint32)
    inc = M[0] != INF
    inc[0] = True
    return np.flatnonzero(inc)


def weights(M, open_):
    """w as an int64 [n][n] matrix."""
    M = np.asarray(M, np.uint32)
    W = np.where(M == INF, np.int64(P), M.astype(np.int64))
    np.fill_diagonal(W, 0)
    if open_:
        W[:, 0] = 0
    return W


def legs(W, t):
    """The leg weights w(t_k, t_{k+1}), k < m, with t_m = t_0."""
    t = np.asarray(t)
    return W[t, np.roll(t, -1)]


def cost(W, t):
    return int(legs(W, t).sum())


def construct(W, inc, s, seed):
    """Start s's tour: positions 1..m-1 filled in turn from the c = min(3, unvisited) unvisited sites of least
    (w(t_{k-1}, j), j); start 0 takes the first, start s >= 1 candidate splitmix64(seed ^ (s << 32) ^ k) % c."""
    m = len(inc)
    t = [0]
    left = np.ones(W.shape[0], bool)
    left[0] = False
    rest = np.zeros(W.shape[0], bool)
    rest[inc] = True
    left &= rest
    for k in range(1, m):
        js = np.flatnonzero(left)
        key = (W[t[-1], js] << 10) | js
        c = min(3, len(js))
        pick = 0 if s == 0 else splitmix64((int(seed) ^ (s << 32) ^ k) & M64) % c
        j = int(js[np.argsort(key, kind="stable")[pick]])
        t.append(j)
        left[j] = False
    return np.array(t, np.int64)


def code_2opt(i, j):
    return (i << 12) | j


def code_or(i, L, q):
    return (1 << 22) | (i << 12) | (L << 10) | q


def decode(code):
    return code >> 22, (code >> 12) & 1023, (code >> 10) & 3, code & 1023


def apply(t, code):
    """The tour after move `code`: 2-opt reverses positions [i, j]; Or-opt moves [i, i+L-1] into gap q."""
    typ, i, L, x = decode(code)
    t = list(t)
    if typ == 0:
        return np.array(t[:i] + t[i:x + 1][::-1] + t[x + 1:], np.int64)
    e = i + L - 1
    seg, rest = t[i:e + 1], t[:i] + t[e + 1:]
    at = x + 1 if x < i else x + 1 - L       # gap q's place in the tour without the segment
    return np.array(rest[:at] + seg + rest[at:], np.int64)


def moves(W, t):
    """Every move of tour t as (deltas, codes), by the O(1) formulas of the prefix sums."""
    t = np.asarray(t, np.int64)
    m = len(t)
    T = np.append(t, t[0])
    WT = W[np.ix_(T, T)]                     # WT[a][b] = w(t_a, t_b), positions 0..m
    f = WT[np.arange(m), np.arange(1, m + 1)]
    b = WT[np.arange(1, m + 1), np.arange(m)]
    F = np.concatenate([[0], np.cumsum(f)])
    B = np.concatenate([[0], np.cumsum(b)])
    ds, cs = [], []
    if m >= 3:                               # 2-opt: rows i in [1, m-2], columns j in [1, m-1], j > i
        i = np.arange(1, m)[:, None]
        j = np.arange(1, m)[None, :]
        d = WT[0:m - 1, 1:m] + WT[1:m, 2:m + 1] - f[i - 1] - f[j] + (B[j] - B[i]) - (F[j] - F[i])
        ok = j > i
        ds.append(d[ok])
        cs.append(code_2opt(np.broadcast_to(i, ok.shape)[ok], np.broadcast_to(j, ok.shape)[ok]))
    for L in (1, 2, 3):                      # Or-opt: rows i in [1, m-L], columns q in [0, m-1] outside [i-1, i+L-1]
        if m - L < 1:
            continue
        i = np.arange(1, m - L + 1)[:, None]
        q = np.arange(m)[None, :]
        e = i + L - 1
        d = (WT[i - 1, e + 1] - f[i - 1] - f[e]) + WT[0:m, 1:m - L + 1].T + WT[L:m, 1:m + 1] - f[q]
        ok = (q < i - 1) | (q > e)
        ds.append(d[ok])
        cs.append(code_or(np.broadcast_to(i, ok.shape)[ok], L, np.broadcast_to(q, ok.shape)[ok]))
    if not ds:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(ds), np.concatenate(cs)


def best_move(W, t):
    """(delta, code) of the least (delta, code) move, or None when the tour has no move."""
    d, c = moves(W, t)
    if len(d) == 0:
        return None
    dmin = d.min()
    return int(dmin), int(c[d == dmin].min())


def search(W, inc, s, seed, max_passes):
    """(tour, cost, passes, converged) of start s: up to max_passes passes, each applying its least move while that
    move's delta is negative; converged when a pass found none, so passes < max_passes exactly when converged."""
    t = construct(W, inc, s, seed)
    passes, converged = 0, 0
    for _ in range(max_passes):
        bm = best_move(W, t)
        if bm is None or bm[0] >= 0:
            converged = 1
            break
        t = apply(t, bm[1])
        passes += 1
    return t, cost(W, t), passes, converged


def tour(M, open_, n_starts, max_passes, seed):
    """(info INFO_DTYPE record, starts START_DTYPE [n_starts], order int32 [n]) of a tour job on the uint32 matrix
    M [n][n]: the best start is the least (cost, s); order holds its tour, -1 past n_included."""
    M = np.asarray(M, np.uint32)
    n = M.shape[0]
    inc = included(M)
    W = weights(M, open_)
    starts = np.zeros(n_starts, START_DTYPE)
    best = None
    for s in range(n_starts):
        t, c, p, conv = search(W, inc, s, seed, max_passes)
        starts[s] = (c, p, conv)
        if best is None or c < best[1]:
            best = (s, c, t)
    s, c, t = best
    order = np.full(n, -1, np.int32)
    order[:len(t)] = t
    info = np.zeros((), INFO_DTYPE)
    info["n_sites"], info["n_included"], info["open"] = n, len(inc), open_
    info["n_starts"], info["max_passes"], info["best_start"], info["best_cost"] = n_starts, max_passes, s, c
    info["seed"], info["n_infinite"] = np.uint64(seed), int((legs(W, t) == P).sum())
    return info, starts, order
