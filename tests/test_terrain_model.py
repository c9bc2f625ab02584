"""oracle/pyoracle_terrain: the terrain of a known field (DESIGN.md §8.20) against a literal per-column and per-cell
restatement in plain Python loops on random grids for all six up axes, the symmetries that map one up axis onto
another, the clearance against the known field's distance and a brute-force minimum, hand cases and every refusal."""
import itertools

import numpy as np
import pytest

import pyoracle_field_known
import pyoracle_terrain as TR
from pyoracle_field_known import FREE, OCCUPIED, UNKNOWN


def literal(state, up, headroom, max_step):
    """The definition of include/dsm.h, one column and one cell at a time."""
    nz, ny, nx = state.shape
    n = (nx, ny, nz)
    a = abs(up) - 1
    m = list(n)
    m[a] = 1

    def at(q):
        return int(state[q[2], q[1], q[0]])

    level = np.full((m[2], m[1], m[0]), -1, np.int16)
    for c2, c1, c0 in itertools.product(range(m[2]), range(m[1]), range(m[0])):
        for k in (range(n[a] - 1, -1, -1) if up > 0 else range(n[a])):
            q = [c0, c1, c2]
            q[a] = k
            if at(q) != OCCUPIED:
                continue
            ok = True
            for h in range(1, headroom + 1):
                kk = k + h if up > 0 else k - h
                if not 0 <= kk < n[a]:
                    ok = False
                    break
                q[a] = kk
                if at(q) != FREE:
                    ok = False
                    break
            if ok:
                level[c2, c1, c0] = k
                break
    hor = [k for k in range(3) if k != a]
    step = np.zeros_like(level, np.uint8)
    status = np.zeros_like(level, np.uint8)
    for c2, c1, c0 in itertools.product(range(m[2]), range(m[1]), range(m[0])):
        c = [c0, c1, c2]
        lv = int(level[c2, c1, c0])
        if lv < 0:
            continue
        worst = 0
        for d0 in (-1, 0, 1):
            for d1 in (-1, 0, 1):
                if d0 == 0 and d1 == 0:
                    continue
                q = list(c)
                q[hor[0]] += d0
                q[hor[1]] += d1
                if not all(0 <= q[k] < m[k] for k in range(3)):
                    continue
                ln = int(level[q[2], q[1], q[0]])
                if ln >= 0:
                    worst = max(worst, abs(lv - ln))
        step[c2, c1, c0] = min(worst, 255)
        status[c2, c1, c0] = 1 if worst > max_step else 2
    return level, status, step


def random_state(rng, shape, p):
    """A grid [nz][ny][nx] with occupied, free and unknown voxels in proportions p."""
    nx, ny, nz = shape
    return rng.choice(np.array([OCCUPIED, FREE, UNKNOWN], np.uint8), size=(nz, ny, nx), p=p)


@pytest.mark.parametrize("up", TR.UPS)
def test_model_equals_the_literal_definition(up):
    rng = np.random.default_rng(abs(up) * 7 + (up > 0))
    for shape, p in (((7, 6, 5), (0.3, 0.6, 0.1)), ((5, 9, 4), (0.2, 0.7, 0.1)), ((6, 4, 8), (0.5, 0.4, 0.1)), ((1, 6, 5), (0.3, 0.6, 0.1))):
        state = random_state(rng, shape, p)
        n_a = shape[abs(up) - 1]
        for headroom in sorted({1, 2, max(1, n_a - 1)}):
            if headroom > n_a - 1:
                continue
            for max_step in (0, 1, 3):
                info, lev, status, step, clear = TR.job(state, (1, -2, 3), 0.2, up, headroom, max_step)
                want = literal(state, up, headroom, max_step)
                assert lev.tobytes() == want[0].tobytes(), (shape, headroom)
                assert status.tobytes() == want[1].tobytes(), (shape, headroom, max_step)
                assert step.tobytes() == want[2].tobytes(), (shape, headroom)
                assert info["n_blocked"] == (want[1] == 1).sum() and info["n_traversable"] == (want[1] == 2).sum()
                assert info["n_support"] == (want[0] >= 0).sum()
                assert list(info["m"]) == list(TR.terrain_shape(shape, up)) and info["up"] == up


def test_steps_above_255_are_stored_clamped():
    st = np.full((300, 1, 2), FREE, np.uint8)
    st[0, 0, 0] = OCCUPIED        # level 0
    st[280, 0, 1] = OCCUPIED      # level 280
    _, lev, status, step, _ = TR.job(st, (0, 0, 0), 0.1, 3, 5, 1023)
    assert lev.reshape(-1).tolist() == [0, 280] and step.reshape(-1).tolist() == [255, 255] and status.reshape(-1).tolist() == [2, 2]
    _, _, status, _, _ = TR.job(st, (0, 0, 0), 0.1, 3, 5, 279)
    assert status.reshape(-1).tolist() == [1, 1]


@pytest.mark.parametrize("up", TR.UPS)
def test_transposes_and_flips_map_one_up_axis_onto_another(up):
    """The grid seen with up = +3 is the transposed grid seen with up: the same levels (mirrored for a negative up), the
    same planes in the transposed layout."""
    rng = np.random.default_rng(11 + up)
    base = random_state(rng, (6, 5, 7), (0.3, 0.6, 0.1))   # [z][y][x], up = +3 along z
    a = abs(up) - 1
    # put grid axis 2 (numpy axis 0) on grid axis a (numpy axis 2 - a), flipped for a negative up
    moved = np.moveaxis(base, 0, 2 - a)
    if up < 0:
        moved = np.flip(moved, axis=2 - a)
    moved = np.ascontiguousarray(moved)
    _, lev0, st0, sp0, cl0 = TR.job(base, (0, 0, 0), 0.1, 3, 2, 1)
    _, lev, st, sp, cl = TR.job(moved, (0, 0, 0), 0.1, up, 2, 1)
    n_a = base.shape[0]
    lev0_m = np.where(lev0 >= 0, lev0 if up > 0 else n_a - 1 - lev0, -1).astype(np.int16)
    for got, want in ((lev, lev0_m), (st, st0), (sp, sp0), (cl, cl0)):
        assert np.moveaxis(got, 2 - a, 0).tobytes() == want.tobytes() if a != 2 else got.tobytes() == want.tobytes()
    # the transpose of the horizontal axes keeps every plane transposed
    _, lev_t, st_t, sp_t, cl_t = TR.job(np.ascontiguousarray(base.transpose(0, 2, 1)), (0, 0, 0), 0.1, 3, 2, 1)
    for got, want in ((lev_t, lev0), (st_t, st0), (sp_t, sp0), (cl_t, cl0)):
        assert got.transpose(0, 2, 1).tobytes() == want.tobytes()


def test_clearance_is_the_known_distance_of_the_status_plane_and_a_brute_force_minimum():
    rng = np.random.default_rng(3)
    for up in (-2, 3, 1):
        state = random_state(rng, (9, 8, 7), (0.35, 0.55, 0.1))
        _, lev, status, _, clear = TR.job(state, (0, 0, 0), 0.25, up, 1, 1)
        assert clear.tobytes() == pyoracle_field_known.state_field(status, 0.25)[0].tobytes()
        blocked = np.argwhere(status != 2)
        v = np.float32(0.25)
        for idx in np.ndindex(status.shape):
            d2 = ((blocked - np.array(idx)) ** 2).sum(axis=1).min() if len(blocked) else None
            want = np.float32(np.inf) if d2 is None else np.float32(np.sqrt(np.float32(d2))) * v
            assert clear[idx] == want, (up, idx)


def flat(nx=6, ny=5, nz=8, ground=2, up=3):
    """Ground at z = ground (z up), observed free above it, unknown below."""
    st = np.full((nz, ny, nx), UNKNOWN, np.uint8)
    st[ground] = OCCUPIED
    st[ground + 1:] = FREE
    return st


def test_flat_ground():
    info, lev, status, step, clear = TR.job(flat(), (0, 0, -1), 0.5, 3, 3, 0)
    assert (lev == 2).all() and (status == 2).all() and (step == 0).all() and np.isinf(clear).all()
    assert info["n_support"] == info["n_traversable"] == 30 and info["n_blocked"] == 0
    assert np.allclose(TR.height(lev, (0, 0, -1), 0.5, 3), (-1 + 2 + 1) * 0.5)


def test_a_one_voxel_curb():
    st = flat()
    st[3, :, 3:] = OCCUPIED        # a curb one voxel high on x >= 3
    _, lev, status, step, _ = TR.job(st, (0, 0, 0), 0.5, 3, 3, 1)
    assert (lev[0, :, :3] == 2).all() and (lev[0, :, 3:] == 3).all()
    assert (step[0, :, 2:4] == 1).all() and (status == 2).all()
    _, _, status, _, clear = TR.job(st, (0, 0, 0), 0.5, 3, 3, 0)
    assert (status[0, :, 2:4] == 1).all() and (status[0, :, [0, 1, 4, 5]] == 2).all()
    assert (clear[0, :, 2:4] == 0).all() and (clear[0, :, 1] == 0.5).all()


def test_a_box():
    """A 3x3 box two voxels high: its top is supported at box height, its edge cells are blocked by the step, and the
    top's middle is traversable."""
    st = flat(9, 9, 10)
    st[3:5, 3:6, 3:6] = OCCUPIED
    _, lev, status, step, _ = TR.job(st, (0, 0, 0), 0.2, 3, 3, 1)
    assert (lev[0, 3:6, 3:6] == 4).all() and lev[0, 0, 0] == 2
    top = status[0, 3:6, 3:6]
    assert top[1, 1] == 2 and (np.delete(top.reshape(-1), 4) == 1).all()
    assert step[0, 4, 3] == 2 and step[0, 4, 2] == 2 and status[0, 4, 2] == 1 and status[0, 4, 1] == 2


def test_a_deck_with_observed_headroom_and_an_unknown_top():
    st = flat(6, 5, 10)
    st[5, :, 1:5] = OCCUPIED       # a deck at z = 5, free from the road up to it, its top never seen
    st[6:, :, 1:5] = UNKNOWN
    _, lev, status, _, _ = TR.job(st, (0, 0, 0), 0.2, 3, 2, 1)
    assert (lev[0, :, 1:5] == 2).all() and (status[0, :, 1:5] == 2).all()   # the road under it
    st[6:, :, 1:5] = FREE          # now its top is seen
    _, lev, _, _, _ = TR.job(st, (0, 0, 0), 0.2, 3, 2, 1)
    assert (lev[0, :, 1:5] == 5).all()


def test_a_deck_too_low_for_the_headroom():
    st = flat(6, 5, 10)
    st[4, :, 1:5] = OCCUPIED       # one free voxel between road and deck
    st[5:, :, 1:5] = UNKNOWN
    _, lev, status, _, _ = TR.job(st, (0, 0, 0), 0.2, 3, 2, 1)
    assert (lev[0, :, 1:5] == -1).all() and (status[0, :, 1:5] == 0).all()
    _, lev, _, _, _ = TR.job(st, (0, 0, 0), 0.2, 3, 1, 1)
    assert (lev[0, :, 1:5] == 2).all()


def test_headroom_cut_by_the_top_face():
    st = flat(4, 4, 6, ground=2)   # free voxels 3, 4, 5 above the ground
    assert (TR.job(st, (0, 0, 0), 0.2, 3, 3, 1)[1] == 2).all()
    assert (TR.job(st, (0, 0, 0), 0.2, 3, 4, 1)[1] == -1).all()
    assert (TR.job(st[::-1].copy(), (0, 0, 0), 0.2, -3, 3, 1)[1] == 3).all()   # the same seen with up = -3


def test_one_unknown_voxel_in_the_headroom():
    st = flat(4, 4, 8)
    st[5, 1, 2] = UNKNOWN
    _, lev, status, _, clear = TR.job(st, (0, 0, 0), 0.2, 3, 3, 1)
    assert lev[0, 1, 2] == -1 and status[0, 1, 2] == 0 and clear[0, 1, 2] == 0
    assert (np.delete(lev.reshape(-1), 1 * 4 + 2) == 2).all()


@pytest.mark.parametrize("up", [1, 2, 3])
def test_in_plane_axes_of_length_one(up):
    rng = np.random.default_rng(up)
    shape = [1, 1, 1]
    shape[up - 1] = 12
    other = [k for k in range(3) if k != up - 1]
    for ln in (1, 7):
        sh = list(shape)
        sh[other[0]] = ln
        state = random_state(rng, sh, (0.3, 0.6, 0.1))
        for u in (up, -up):
            got = TR.job(state, (0, 0, 0), 0.1, u, 2, 0)
            want = literal(state, u, 2, 0)
            assert all(g.tobytes() == w.tobytes() for g, w in zip(got[1:4], want))


def test_every_refused_request():
    for up in (0, 4, -4, 7):
        with pytest.raises(ValueError):
            TR.check_enable(up)
    for up, headroom, max_step in ((3, 0, 0), (3, 8, 0), (-1, 6, 0), (2, 5, 0), (3, 1, -1), (3, 1, 1024)):
        with pytest.raises(ValueError):
            TR.check_request((6, 5, 8), up, headroom, max_step)
    TR.check_request((6, 5, 8), 3, 7, 1023)
    TR.check_request((6, 5, 8), -1, 5, 0)
    with pytest.raises(ValueError):
        TR.job(np.zeros((1, 4, 4), np.uint8), (0, 0, 0), 0.1, 3, 1, 0)    # n_a = 1: no headroom fits
