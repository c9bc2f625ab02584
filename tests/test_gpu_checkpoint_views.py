"""dsm_checkpoint_views_enable (DESIGN.md §8.18): the captured views travel with every checkpoint.  A context that loads
a file resumes known space exactly where the saver was: the same known fields (and the oracle's), frontiers and reach
results after the load and after every later frame.  The asynchronous file and every resolved journal record equal a
twin's dsm_map_save at the enqueue position; a record lists exactly the slots captured since the previous checkpoint;
the enable order, the state rules and the load checks hold, and a context without the call still writes version 1."""
import filecmp

import numpy as np
import pytest

import pyoracle_field_known
from densesurfelmapping_b200 import capi
from checkpoint_files import HEADER, RHEADER, fnv1a64
from densesurfelmapping_b200 import synth
from densesurfelmapping_b200.elements import POINT_DTYPE, SURFEL_DTYPE
from known_space import MAX_RANGE, RELOAD, Views, node_args, rejected
from node_drive import node_script, run_driver
from resident_map import SAVES, STORE, T, camera, field_points, loop_warp, map_state, new_ctx, simple_lists, \
    stored_keyframes, warp, windowed

pytestmark = pytest.mark.gpu

SHAPE, VOXEL = (64, 64, 32), 0.1
SLOTS = 6
LISTS = simple_lists()


class Drive:
    """A context with a field, frontier and reach jobs and SLOTS view slots, driven through windowed calls that capture
    every frame; `views` is the test's side of the slot table."""

    def __init__(self, opt_in=True, checkpoint=None, max_views=SLOTS):
        self.ctx = new_ctx(store=STORE)
        self.ctx.field_enable(VOXEL, *SHAPE)
        if checkpoint == "before":
            self.ctx.checkpoint_enable()
        self.views = Views(self.ctx, max_views)
        self.ctx.frontier_enable(256, 1 << 18)
        self.ctx.reach_enable(64, 1 << 16, 4096)
        if opt_in:
            self.ctx.checkpoint_views_enable()
        if checkpoint == "after":
            self.ctx.checkpoint_enable()
        self.calls = 0
        self.captured = set()   # slots captured since the last checkpoint

    def run(self, t0, t1, chunk):
        for s in range(t0, t1, chunk):
            e = min(t1, s + chunk)
            windowed(self.ctx, s, e, LISTS, want_counts=False)
            first = self.views.n
            self.views.capture_call(self.calls, s, e)
            self.captured |= {n % self.views.max for n in range(first, self.views.n)}
            self.calls += 1

    def warp(self):
        loop_warp(self.ctx, stored_keyframes(self.ctx))
        self.views.warp(warp(1))

    def known(self, t):
        """The known field at the camera of frame t over every filled slot, and the frontier and reach jobs on it."""
        slots, poses = self.views.request()
        self.ctx.field_enqueue_known(camera(t), 5, slots, poses)
        field = self.ctx.field_wait()
        state = self.ctx.field_state()
        self.ctx.frontier_enqueue(1)
        fr = self.ctx.frontier_wait()
        self.ctx.reach_enqueue(camera(t), 0.2, 0, camera(0)[None, :], True, True)
        reach = self.ctx.reach_wait()
        return field, state, fr, reach

    def close(self):
        self.ctx.close()


def blob(x):
    if x is None:
        return b"-"
    if isinstance(x, (tuple, list)):
        return b"|".join(blob(y) for y in x)
    if isinstance(x, (int, float, np.integer, np.floating)):
        return np.asarray(x).tobytes()
    return np.asarray(x).tobytes()


def assert_same_known(a, b, t, what):
    ka, kb = a.known(t), b.known(t)
    for name, x, y in zip(("field", "state", "frontier", "reach"), ka, kb):
        assert blob(x) == blob(y), f"{what}: {name}"
    return ka


def file_views(raw):
    """(slots, rays [n, S, 4]) of a version-2 file."""
    h = np.frombuffer(raw, HEADER, 1)[0]
    assert h["format"] == 2
    S = int(h["zero"])
    o = HEADER.itemsize + (int(h["n_pool"]) + int(h["n_store"])) * 44 + 12 * int(h["n_segments"])
    n = int(np.frombuffer(raw, "<i4", 1, o)[0])
    slots = np.frombuffer(raw, "<i4", n, o + 4)
    rays = np.frombuffer(raw, np.float32, n * S * 4, o + 4 + 4 * n).reshape(n, S, 4)
    return slots.tolist(), rays


def records(journal):
    """The view slot list of every record of a version-2 journal."""
    out, pos = [], 32
    S = int(np.frombuffer(journal, "<u4", 1, 12)[0])
    while pos < len(journal):
        r = np.frombuffer(journal, RHEADER, 1, pos)[0]
        kp, ks, kv = int(r["k_pool"]), int(r["k_store"]), int(r["zero"])
        lists = np.frombuffer(journal, "<i4", kp + ks + kv, pos + RHEADER.itemsize)
        pay = 0
        for i, c in enumerate(lists[:kp + ks]):
            n = int(r["n_pool"] if i < kp else r["n_store"])
            pay += min(256, n - 256 * int(c)) * 44
        out.append(lists[kp + ks:].tolist())
        pos += RHEADER.itemsize + 4 * len(lists) + pay + 16 * S * kv + 12 * int(r["n_segments"]) + int(r["extra_bytes"]) + 16
    assert pos == len(journal)
    return out


def fresh_loader(path, opt_in=True):
    b = Drive(opt_in=opt_in)
    extra = b.ctx.map_load(path)
    return b, extra


@pytest.mark.parametrize("chunk", [1, 4])
@pytest.mark.parametrize("save", list(SAVES))
def test_a_loaded_context_resumes_known_space(tmp_path, save, chunk):
    k, when = SAVES[save]
    a = Drive()
    a.run(0, k, chunk)
    if when == "before":
        a.warp()
    path = tmp_path / "map.dsm"
    a.ctx.map_save(path, b"poses")
    raw = path.read_bytes()
    slots, rays = file_views(raw)
    assert slots == sorted(a.views.rays), "file slots"
    for s, r in zip(slots, rays):   # the oracle's kept rays with w = 1, every other seed all zero
        kept = r[:, 3] == 1
        assert r[kept, :3].tobytes() == a.views.rays[s].tobytes(), f"rays of slot {s}"
        assert not r[~kept].view(np.uint32).any(), f"seeds without a ray in slot {s}"
    b, extra = fresh_loader(path)
    assert extra == b"poses"
    b.views.rays, b.views.poses, b.views.n = dict(a.views.rays), dict(a.views.poses), a.views.n
    if when == "after":
        a.warp()
        b.warp()
    # right after the load: equal to the saver and to the oracle
    field, state = assert_same_known(a, b, k - 1, f"{save}: after the load")[:2]
    want = pyoracle_field_known.known_field(field_points(b.ctx, 5), VOXEL, SHAPE, camera(k - 1),
                                            b.views.oracle_views(sorted(b.views.rays)), MAX_RANGE)
    assert field[0].tobytes() == want[0].tobytes() and field[2] == want[2], f"{save}: oracle field"
    assert state[0].tobytes() == want[3].tobytes() and state[1] == want[4], f"{save}: oracle state"
    for s in range(k, T, chunk):
        e = min(T, s + chunk)
        a.run(s, e, chunk)
        b.run(s, e, chunk)
        assert_same_known(a, b, e - 1, f"{save}: after frames {s}-{e - 1}")
    assert map_state(a.ctx) == map_state(b.ctx)
    a.close()
    b.close()


@pytest.mark.parametrize("order", ["before", "after"])
def test_the_asynchronous_file_equals_a_twin_save(tmp_path, order):
    a, b = Drive(checkpoint=order), Drive()
    for call, t0 in enumerate(range(0, T - 2, 2)):
        for d in (a, b):
            d.run(t0, t0 + 2, 2)
        a.ctx.checkpoint_enqueue(str(tmp_path / f"a{call}.dsm"), b"x")
        b.ctx.map_save(tmp_path / f"b{call}.dsm", b"x")
        a.run(t0 + 2, t0 + 4, 2)            # fuse on and recapture, over slots of the pending file, before the wait
        assert a.ctx.checkpoint_wait(True)
        assert (tmp_path / f"a{call}.dsm").read_bytes() == (tmp_path / f"b{call}.dsm").read_bytes(), f"call {call}"
        a.ctx.map_load(tmp_path / f"b{call}.dsm")   # back to the twin's state
        a.views.rays, a.views.poses, a.views.n = dict(b.views.rays), dict(b.views.poses), b.views.n
    a.close()
    b.close()


def test_every_record_resolves_to_a_twin_save_and_lists_the_new_slots(tmp_path):
    a, b = Drive(opt_in=False, checkpoint="after"), Drive()
    path = str(tmp_path / "chain.dsm")
    journal = tmp_path / "chain.dsm.journal"
    bases = []

    def step(t0, t1, what, expect_base):
        a.run(t0, t1, 2)
        b.run(t0, t1, 2)
        a.ctx.checkpoint_enqueue_incremental(path, what.encode())
        b.ctx.map_save(tmp_path / "twin.dsm", what.encode())
        assert a.ctx.checkpoint_wait(True)
        capi.journal_materialize(path, tmp_path / "resolved.dsm")
        assert (tmp_path / "resolved.dsm").read_bytes() == (tmp_path / "twin.dsm").read_bytes(), what
        j = journal.read_bytes()
        is_base = len(j) == 32
        assert is_base == expect_base, what
        if not is_base:
            assert records(j)[-1] == sorted(a.captured), f"{what}: the record's slots"
        bases.append(is_base)
        a.captured = set()

    # a chain without views, then the enable in the middle of it
    a.run(0, 2, 2)
    b.run(0, 2, 2)
    a.ctx.checkpoint_enqueue_incremental(path, b"v1")
    assert a.ctx.checkpoint_wait(True)
    assert np.frombuffer(open(path, "rb").read(), HEADER, 1)[0]["format"] == 1
    a.ctx.checkpoint_views_enable()
    a.captured = set()
    step(2, 4, "enabled mid-chain", True)
    step(4, 6, "record", False)
    step(6, 8, "record 2", False)
    # a failed save ends the chain
    a.ctx.checkpoint_enqueue_incremental(str(tmp_path / "missing" / "x.dsm"), b"")
    with pytest.raises(capi.DsmError) as e:
        a.ctx.checkpoint_wait(True)
    assert e.value.code == -9
    step(8, 10, "after a failed save", True)
    step(10, 12, "record 3", False)
    # a load forces a base
    a.ctx.map_load(tmp_path / "twin.dsm")
    a.captured = set()
    step(12, 14, "after a load", True)
    step(14, 16, "record 4", False)
    assert bases == [True, False, False, True, False, True, False]
    a.close()
    b.close()


def test_a_reserve_makes_the_next_record_a_base(tmp_path):
    """dsm_inactive_reserve needs an empty store: a drive without window lists, reserved after two checkpoints."""
    lists = [(t // 2, [], []) for t in range(T)]
    pair = []
    for with_checkpoint in (True, False):
        c = new_ctx(store=0)
        c.field_enable(VOXEL, *SHAPE)
        if with_checkpoint:
            c.checkpoint_enable()
        pair.append((c, Views(c, SLOTS)))
        c.checkpoint_views_enable()
    (a, _), (b, _) = pair
    path = str(tmp_path / "chain.dsm")
    for call, t0 in enumerate(range(0, 6, 2)):
        if call == 2:
            a.inactive_reserve(STORE)
            b.inactive_reserve(STORE)
        for c, views in pair:
            windowed(c, t0, t0 + 2, lists, want_counts=False, empty=True)
            views.capture_call(call, t0, t0 + 2)
        a.checkpoint_enqueue_incremental(path)
        b.map_save(tmp_path / "twin.dsm")
        assert a.checkpoint_wait(True)
        capi.journal_materialize(path, tmp_path / "resolved.dsm")
        assert (tmp_path / "resolved.dsm").read_bytes() == (tmp_path / "twin.dsm").read_bytes(), f"call {call}"
        n = len(records((tmp_path / "chain.dsm.journal").read_bytes()))
        assert n == [0, 1, 0][call], f"call {call}: {n} records"
    a.close()
    b.close()


def test_state_rules_and_load_checks(tmp_path):
    ctx = new_ctx(store=STORE)
    with pytest.raises(capi.DsmError) as e:
        ctx.checkpoint_views_enable()
    assert e.value.code == -7
    ctx.field_enable(VOXEL, *SHAPE)
    with pytest.raises(capi.DsmError) as e:
        ctx.checkpoint_views_enable()
    assert e.value.code == -7
    ctx.views_enable(4, MAX_RANGE)
    ctx.checkpoint_views_enable()
    with pytest.raises(capi.DsmError) as e:
        ctx.checkpoint_views_enable()
    assert e.value.code == -7
    ctx.close()

    a = Drive()
    a.run(0, 6, 2)                         # slots 0..5 filled
    path = tmp_path / "views.dsm"
    a.ctx.map_save(path)
    raw = path.read_bytes()
    # a context without the call: the file is refused, map and views unchanged; it still writes version 1
    plain = Drive(opt_in=False)
    plain.run(0, 2, 2)
    before = map_state(plain.ctx), blob(plain.known(1))
    with pytest.raises(capi.DsmError) as e:
        plain.ctx.map_load(path)
    assert e.value.code == -7
    assert (map_state(plain.ctx), blob(plain.known(1))) == before
    plain.ctx.map_save(tmp_path / "plain.dsm")
    assert np.frombuffer((tmp_path / "plain.dsm").read_bytes(), HEADER, 1)[0]["format"] == 1

    def refused(data, code, max_views=SLOTS):
        d = Drive(max_views=max_views)
        d.run(0, 2, 2)
        before = map_state(d.ctx), blob(d.known(1))
        (tmp_path / "bad.dsm").write_bytes(data)
        with pytest.raises(capi.DsmError) as e:
            d.ctx.map_load(tmp_path / "bad.dsm")
        assert e.value.code == code
        assert (map_state(d.ctx), blob(d.known(1))) == before
        d.close()

    refused(raw, -6, max_views=4)          # slots 4 and 5 do not fit
    slots, rays = file_views(raw)
    kept = rays.reshape(-1, 4)[:, 3] == 1
    ray, none = int(np.flatnonzero(kept)[0]), int(np.flatnonzero(~kept)[0])
    base = len(raw) - 8 - rays.nbytes
    cases = [(ray, 12, np.float32(0.5)), (ray, 12, np.float32(2.0)),                 # w neither 0 nor 1
             (none, 0, np.float32(-0.0)), (none, 4, np.float32(1e-30)),              # w = 0 with a byte set
             (ray, 0, np.float32(np.nan)), (ray, 8, np.float32(np.inf))]             # w = 1, a coordinate not finite
    for r, off, v in cases:
        bad = bytearray(raw)
        o = base + 16 * r + off
        bad[o:o + 4] = v.tobytes()
        bad[-8:] = np.array([fnv1a64(bytes(bad[:-8]))], "<u8").tobytes()
        refused(bytes(bad), -1)
    a.close()
    plain.close()


def test_a_rejected_frame_gives_no_record_then_a_base(tmp_path):
    first = next(t for t in range(T) if LISTS[t][1])
    ctx = new_ctx(store=1)                 # the first retirement does not fit the store
    ctx.field_enable(VOXEL, *SHAPE)
    ctx.checkpoint_enable()
    views = Views(ctx, 4)
    ctx.checkpoint_views_enable()
    path = str(tmp_path / "chain.dsm")
    journal = tmp_path / "chain.dsm.journal"
    for call, t in enumerate(range(first + 1)):
        windowed(ctx, t, t + 1, LISTS, want_counts=False)
        views.capture_call(call, t, t + 1)
        ctx.checkpoint_enqueue_incremental(path)
        if t < first:
            assert ctx.checkpoint_wait(True)
    before = journal.read_bytes()
    assert len(records(before)) >= 1
    rejected(lambda: ctx.checkpoint_wait(True))
    assert journal.read_bytes() == before, "no record for the rejected frame"
    rejected(ctx.pool_size)                # reports and clears the error
    ctx.checkpoint_enqueue_incremental(path)
    assert ctx.checkpoint_wait(True)
    assert len(journal.read_bytes()) == 32, "a base after the rejected frame"
    ctx.map_save(tmp_path / "now.dsm")
    assert open(path, "rb").read() == (tmp_path / "now.dsm").read_bytes()
    ctx.close()


# ---- the node: tests/cpp/checkpoint_views_main.cpp ----
NODE_FRAMES = 24


def node_views(r):
    return r.i(), r.lst(np.int32).tolist(), r.lst(np.float64).tobytes()


def node_frame(r):
    return (r.i(), r.lst(np.float32).tobytes(), r.lst(np.uint8).tobytes(), r.lst(capi.FRONTIER_CLUSTER_DTYPE).tobytes(),
            r.lst(np.int32).tobytes(), r.i(), r.lst(POINT_DTYPE).tobytes(), r.lst(POINT_DTYPE).tobytes())


def drive_nodes(tmp_path, mode, a_views, b_views):
    cam = synth.KITTI
    prefix = str(tmp_path / f"node{mode}{a_views}{b_views}")
    r = run_driver("checkpoint_views_main", str(tmp_path), cam, node_script(cam, NODE_FRAMES),
                   node_args() + [RELOAD, mode, a_views, b_views], tag=f"{mode}{a_views}{b_views}", after=[prefix])
    rc_save, rc_load = r.i(), r.i()
    return r, prefix, rc_save, rc_load, node_views(r), node_views(r)


@pytest.mark.parametrize("mode", [0, 1, 2], ids=["save_state", "save_state_async", "save_state_incremental"])
def test_a_resumed_node_is_the_node_that_saved(tmp_path, mode):
    r, prefix, rc_save, rc_load, va, vb = drive_nodes(tmp_path, mode, 1, 1)
    assert (rc_save, rc_load) == (0, 0)
    assert va == vb and len(va[1]) > 0, "known_views and captures right after the load"
    later = NODE_FRAMES - RELOAD - (mode == 1)
    carved = 0
    for t in range(later):
        fa, fb = node_frame(r), node_frame(r)
        assert fa[0] == 0 and fa == fb, f"message {t}: " + str([k for k in range(len(fa)) if fa[k] != fb[k]])
        carved += (np.frombuffer(fa[2], np.uint8) == 2).sum()
    assert carved > 0
    assert r.lst(SURFEL_DTYPE).tobytes() == r.lst(SURFEL_DTYPE).tobytes() and r.o == len(r.raw)
    for ext in (".ply", ".pcd"):
        assert filecmp.cmp(prefix + "a" + ext, prefix + "b" + ext, shallow=False), ext


def test_a_version_1_section_resumes_with_an_empty_table(tmp_path):
    r, prefix, rc_save, rc_load, va, vb = drive_nodes(tmp_path, 0, 0, 1)
    assert (rc_save, rc_load) == (0, 0) and len(va[1]) > 0
    assert vb == (0, [], b""), "an empty slot table"
    for t in range(NODE_FRAMES - RELOAD):
        fa, fb = node_frame(r), node_frame(r)
        assert fa[5:] == fb[5:], f"message {t}: clouds"


def test_a_node_without_view_checkpoints_refuses_a_version_2_section(tmp_path):
    r, prefix, rc_save, rc_load, va, vb = drive_nodes(tmp_path, 0, 1, 0)
    assert (rc_save, rc_load) == (0, -1)
    assert vb == (0, [], b"") and r.i() == 1, "the node is unchanged"
    assert r.o == len(r.raw)
