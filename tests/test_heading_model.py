"""oracle/pyoracle_heading, the definition of dsm_heading_enqueue (DESIGN.md §8.19): the plan against brute-force
enumeration of every step sequence, the counts against whole gain jobs (oracle/pyoracle_gain) on the poses [R_r | p_s],
the sample positions against pyoracle_trajectory.curve_samples, hand cases (an unknown slab to one side, a held heading,
an unreachable end, a turn through rotation 0, samples outside the grid) and every refusal."""
import itertools

import numpy as np
import pytest

import pyoracle_gain as G
import pyoracle_heading as H
import pyoracle_trajectory as tj
from planner_scenes import rotations, scene

UNKNOWN, OCCUPIED, FREE = G.UNKNOWN, G.OCCUPIED, G.FREE


def cam(max_range, unknown_blocks=1):
    return G.Camera(60.0, 60.0, 31.5, 23.5, 64, 48, float(np.float32(max_range)), unknown_blocks)


def brute(score, start, end, max_step):
    """Every step sequence in the tie order (itertools.product is lexicographic in it): the first with the highest
    score, then the fewest steps."""
    S, n_rot = score.shape
    order = np.array(H.step_order(max_step), np.int64)
    seq = np.array(list(itertools.product(range(len(order)), repeat=S - 1)), np.int64).reshape(-1, S - 1)
    d = order[seq]
    turns = np.concatenate([np.zeros((len(d), 1), np.int64), np.cumsum(d, axis=1)], axis=1)
    rots = (start + turns) % n_rot
    ok = np.ones(len(d), bool) if end < 0 else rots[:, -1] == end
    if not ok.any():
        return 1, np.full(S, -1), np.zeros(S), 0, 0
    tot = score[np.arange(S)[None, :], rots].sum(axis=1)
    steps = np.abs(d).sum(axis=1)
    best = tot[ok].max()
    cand = ok & (tot == best)
    fewest = steps[cand].min()
    k = int(np.flatnonzero(cand & (steps == fewest))[0])
    return 0, rots[k], turns[k], int(tot[k]), int(steps[k])


@pytest.mark.parametrize("n_rot", [1, 2, 3, 4, 5])
def test_plan_equals_brute_force(n_rot):
    rng = np.random.default_rng(n_rot)
    half = -(-n_rot // 2)
    for S in range(2, 7):
        for max_step in sorted({0, 1, half, n_rot} if S <= 4 else {0, 1, half}):
            for end in [-1] + list(range(n_rot)):
                for trial in range(3):
                    hi = [1, 2, 4][trial]   # few distinct values: many ties
                    score = rng.integers(0, hi + 1, (S, n_rot)).astype(np.int64)
                    start = int(rng.integers(n_rot))
                    got = H.plan(score, start, end, max_step)
                    want = brute(score, start, end, max_step)
                    what = f"S={S} n_rot={n_rot} max_step={max_step} start={start} end={end}\n{score}"
                    assert got[0] == want[0], what
                    assert got[1].tolist() == list(want[1]) and got[2].tolist() == list(want[2]), what
                    assert got[3:] == want[3:], what


def random_splines(rng, n, shape, voxel, lens=(7, 9, 12), spill=0.0):
    """n trajectories of the given lengths whose control points lie in the grid's box, widened by `spill` of its size
    on every side."""
    v = float(np.float32(voxel))
    size = np.array(shape, np.float64) * v
    pts, ofs = [], [0]
    for j in range(n):
        N = lens[j % len(lens)]
        a, b = rng.uniform(-spill, 1 + spill, 3) * size, rng.uniform(-spill, 1 + spill, 3) * size
        q = a + np.linspace(0, 1, N)[:, None] * (b - a) + rng.standard_normal((N, 3)) * v
        pts.append(q)
        ofs.append(ofs[-1] + N)
    return np.concatenate(pts), np.array(ofs, np.int32)


@pytest.mark.parametrize("unknown_blocks", [0, 1])
def test_counts_equal_gain_jobs(unknown_blocks):
    rng = np.random.default_rng(10 + unknown_blocks)
    shape, voxel, origin = (20, 18, 8), 0.25, (-3, 2, -1)
    nonzero = np.zeros(2, bool)
    for trial in range(3):
        st = scene(rng, shape, n_blobs=8)
        pts, ofs = random_splines(rng, 2, shape, voxel, spill=0.2)
        pts = pts + np.asarray(origin) * np.float64(np.float32(voxel))
        rot = rotations(6, (0.0, -0.4))
        c = cam(6 * voxel, unknown_blocks)
        K = 2
        req = H.requests([(0, -1, 2), (3, 5, 1)])
        info, recs, samples, counts = H.job(st, origin, voxel, c, rot, K, pts, ofs, req, 3, 5)
        pos = H.sample_positions(pts, ofs, K)
        want = np.concatenate([tj.curve_samples(pts[ofs[j]:ofs[j + 1]], K) for j in range(2)])
        assert samples["p"].tobytes() == want.tobytes() == pos.tobytes()
        poses = np.array([np.concatenate([R.reshape(3, 3), p[:, None]], axis=1).reshape(12) for p in pos for R in rot])
        _, g = G.gains(st, origin, voxel, c, poses)
        g = g.reshape(len(pos), len(rot))
        assert (counts["n_unknown"] == g["n_unknown"]).all() and (counts["n_frontier"] == g["n_frontier"]).all()
        nonzero |= [(g["n_unknown"] > 0).any(), (g["n_frontier"] > 0).any()]
        outside = (g["status"] == 1).all(axis=1)
        assert (g["status"][~outside] == 0).all()
        assert recs["n_outside"].sum() == outside.sum()
        score = 3 * counts["n_unknown"].astype(np.int64) + 5 * counts["n_frontier"]
        for j, r in enumerate(recs):
            s = slice(r["sample_offset"], r["sample_offset"] + r["n_samples"])
            assert r["n_samples"] == K * (ofs[j + 1] - ofs[j] - 3) + 1
            status, rr, tt, tot, steps = H.plan(score[s], int(req[j]["start"]), int(req[j]["end"]), int(req[j]["max_step"]))
            assert (r["status"], r["score"], r["steps"]) == (status, tot, steps)
            assert samples["rotation"][s].tolist() == rr.tolist() and samples["turn"][s].tolist() == tt.tolist()
        assert info["n_samples"] == len(pos) and info["n_rot"] == len(rot) and info["n_status"].sum() == 2
    assert nonzero.all()


def corridor(n_rot, max_step, end=-1, start=0, slab=True, K=2):
    """A free grid with an unknown slab along its +y side and a straight trajectory along x through the middle."""
    shape, voxel = (40, 30, 6), 0.2
    st = np.full(shape[::-1], FREE, np.uint8)
    if slab:
        st[:, 22:, :] = UNKNOWN
    line = np.linspace([1.5, 3.0, 0.6], [6.5, 3.0, 0.6], 7)
    req = H.requests([(start, end, max_step)])
    return H.job(st, (0, 0, 0), voxel, cam(12 * voxel), rotations(n_rot), K, line, [0, 7], req, 1, 1)


def test_the_heading_turns_toward_the_unknown_slab_as_fast_as_allowed():
    _, recs, samples, counts = corridor(8, 1)
    rot = samples["rotation"]
    assert recs[0]["status"] == 0
    assert (counts["n_unknown"][:, 2] > counts["n_unknown"][:, 1]).all() and (counts["n_unknown"][:, 1] > counts["n_unknown"][:, 0]).all()
    assert rot[:3].tolist() == [0, 1, 2] and (rot[2:] == 2).all()   # +y is rotation 2, reached one step per sample
    assert samples["turn"][-1] == 2 and recs[0]["steps"] == 2
    _, recs2, samples2, _ = corridor(8, 2)
    assert samples2["rotation"][:2].tolist() == [0, 2] and recs2[0]["score"] > recs[0]["score"]


def test_max_step_zero_holds_the_start():
    _, recs, samples, _ = corridor(8, 0, start=5)
    assert recs[0]["status"] == 0 and recs[0]["steps"] == 0
    assert (samples["rotation"] == 5).all() and (samples["turn"] == 0).all()


def test_an_unreachable_end_gives_status_1():
    # K = 1 and 7 points: 5 samples, 4 intervals; 16 rotations at one step per interval reach rotation 4, not 5
    info, recs, samples, _ = corridor(16, 1, end=4, K=1)
    assert recs[0]["status"] == 0 and samples["rotation"][-1] == 4 and samples["turn"][-1] == 4
    info, recs, samples, _ = corridor(16, 1, end=5, K=1)
    assert recs[0]["status"] == 1 and info["n_status"].tolist() == [0, 1]
    assert (samples["rotation"] == -1).all() and (samples["turn"] == 0).all()
    assert recs[0]["score"] == 0 and recs[0]["steps"] == 0
    assert (samples["p"] == H.sample_positions(np.linspace([1.5, 3.0, 0.6], [6.5, 3.0, 0.6], 7), [0, 7], 1)).all()


def test_the_shortest_turn_wraps_through_rotation_0():
    _, recs, samples, counts = corridor(8, 1, start=1, end=6, slab=False, K=1)
    assert (counts["n_unknown"] == 0).all() and (counts["n_frontier"] == 0).all()
    assert recs[0]["status"] == 0 and recs[0]["steps"] == 3 and recs[0]["score"] == 0
    # four intervals for three steps: the first step in the tie order is 0, so the turn starts one sample late
    assert samples["rotation"].tolist() == [1, 1, 0, 7, 6] and samples["turn"].tolist() == [0, 0, -1, -2, -3]


def test_samples_outside_the_grid_count_zero():
    shape, voxel = (16, 16, 6), 0.2
    st = np.full(shape[::-1], UNKNOWN, np.uint8)
    st[2:4, 4:12, 4:12] = FREE
    line = np.linspace([-1.0, 1.6, 0.6], [2.2, 1.6, 0.6], 8)
    info, recs, samples, counts = H.job(st, (0, 0, 0), voxel, cam(8 * voxel, 0), rotations(4), 3, line, [0, 8], H.requests([(0, -1, 1)]), 1, 0)
    out = np.floor(samples["p"][:, 0] / np.float64(np.float32(voxel))) < 0
    assert 0 < out.sum() < len(out) and recs[0]["n_outside"] == out.sum()
    assert (counts["n_unknown"][out] == 0).all() and (counts["n_unknown"][~out] > 0).any()


def test_refusals():
    c = cam(1.0)
    rot = rotations(4)
    pts = np.linspace([0.0, 0.0, 0.0], [1.0, 0.0, 0.0], 8)
    ofs = [0, 8]
    req = H.requests([(0, -1, 1)])
    H.check_request(c, 0.1, pts, ofs, rot, 4, req, 1, 1)

    def bad(**kw):
        a = dict(camera=c, voxel=0.1, points=pts, offsets=ofs, rotations=rot, K=4, reqs=req, w_unknown=1, w_frontier=1)
        a.update(kw)
        with pytest.raises(ValueError):
            H.check_request(**a)

    bad(camera=c._replace(fx=0.0))
    bad(camera=c._replace(cy=np.nan))
    bad(camera=c._replace(width=0))
    bad(camera=c._replace(height=65537))
    bad(camera=c._replace(unknown_blocks=2))
    bad(camera=c._replace(max_range=0.0))
    bad(camera=c._replace(max_range=float(np.float32(12.81))))   # above 128 v
    bad(rotations=np.zeros((0, 9)))
    bad(rotations=rotations(65))
    bad(rotations=np.where(np.arange(36).reshape(4, 9) == 5, np.inf, rot))
    bad(K=0)
    bad(K=65)
    bad(w_unknown=-1)
    bad(w_frontier=(1 << 16) + 1)
    bad(offsets=[0, 6])
    bad(offsets=[1, 8])
    bad(offsets=[0])
    bad(offsets=[0, 9])
    bad(points=np.zeros((257, 3)), offsets=[0, 257])
    bad(points=np.where(np.arange(24).reshape(8, 3) == 7, np.nan, pts))
    bad(reqs=H.requests([(4, -1, 1)]))
    bad(reqs=H.requests([(-1, -1, 1)]))
    bad(reqs=H.requests([(0, 4, 1)]))
    bad(reqs=H.requests([(0, -2, 1)]))
    bad(reqs=H.requests([(0, -1, 5)]))
    bad(reqs=H.requests([(0, -1, -1)]))
    bad(reqs=H.requests([(0, -1, 1), (0, -1, 1)]))
    H.check_request(c, 0.1, pts, ofs, rot, 4, H.requests([(3, 3, 4)]), 1 << 16, 0)
    # max_samples and the work bound: 21 samples of (2 ceil(R / v) + 3)^3 voxels
    H.check_request(c, 0.1, pts, ofs, rot, 4, req, 1, 1, max_samples=21)
    bad(max_samples=20)
    R = float(np.float32(12.8))            # 128 voxels: 259^3 voxels per sample
    m3 = 259 ** 3
    n_ok = H.MAX_WORK // m3
    S_per = 4 * 5 + 1
    n_traj = n_ok // S_per
    many = np.tile(pts, (n_traj + 1, 1))
    many_ofs = np.arange(n_traj + 2) * 8
    reqs = H.requests([(0, -1, 1)] * (n_traj + 1))
    assert (n_traj + 1) * S_per * m3 > H.MAX_WORK >= n_traj * S_per * m3
    with pytest.raises(ValueError):
        H.check_request(c._replace(max_range=R), 0.1, many, many_ofs, rot, 4, reqs, 1, 1)
    H.check_request(c._replace(max_range=R), 0.1, many[:8 * n_traj], many_ofs[:n_traj + 1], rot, 4, reqs[:n_traj], 1, 1)
    for caps in ((0, 1), (1, 0), ((1 << 22) + 1, 1), (1, (1 << 22) + 1)):
        with pytest.raises(ValueError):
            H.check_enable(*caps)
    H.check_enable(1 << 22, 1 << 22)
