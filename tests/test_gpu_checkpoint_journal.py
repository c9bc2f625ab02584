"""Incremental checkpoints (dsm_checkpoint_enqueue_incremental, dsm_map_load_journal, DESIGN.md §8.6).

After every call of a drive the base and its journal resolve to exactly the file dsm_map_save writes at the same stream
position; every record lists exactly the 256-surfel chunks that differ between the two consecutive dsm_map_save files
(not a superset); a base is written on every trigger of include/dsm.h and after a rejected frame; journal checkpoints
leave the map as a drive without them; a fresh context resumes from the journal; and dsm::SurfelMapNode's
save_state_incremental / load_state_incremental (tests/cpp/checkpoint_journal_main.cpp)."""
import os

import numpy as np
import pytest

from densesurfelmapping_b200 import capi, synth
from checkpoint_files import JHEADER, RHEADER, changed, parse
from node_drive import node_script, run_driver
from resident_map import SAVES, STORE, T, loop_warp, made, new_ctx, readers, run, simple_lists, stored_keyframes, windowed

pytestmark = pytest.mark.gpu

DSM_E_CAPACITY = -6


def journal_ctx(constants="drive", **kw):
    ctx = made(constants, **kw)
    ctx.checkpoint_enable()
    return ctx


def last_record(path):
    """(pool chunk list, store chunk list) of the journal's last record, found by walking the records from the header."""
    j = open(str(path) + ".journal", "rb").read()
    pos, last = JHEADER.itemsize + 8, None
    while pos < len(j):
        h = np.frombuffer(j, RHEADER, 1, pos)[0]
        kp, ks = int(h["k_pool"]), int(h["k_store"])
        lists = np.frombuffer(j, "<i4", kp + ks, pos + RHEADER.itemsize)
        payload = sum(min(256, int(h["n_pool"]) - 256 * int(c)) for c in lists[:kp])
        payload += sum(min(256, int(h["n_store"]) - 256 * int(c)) for c in lists[kp:])
        n = RHEADER.itemsize + 4 * (kp + ks) + 44 * payload + 12 * int(h["n_segments"]) + int(h["extra_bytes"]) + 16
        last = (lists[:kp].tolist(), lists[kp:].tolist())
        pos += n
    assert pos == len(j)
    return last


class Journal:
    """Checkpoints `a` incrementally to `path` and checks each against `b`'s dsm_map_save at the same position."""

    def __init__(self, tmp_path, a, b, name="map.dsm"):
        self.tmp, self.a, self.b, self.path = tmp_path, a, b, tmp_path / name
        self.prev = None          # the previous checkpoint's state as dsm_map_save wrote it
        self.records = 0          # records the journal should resolve with
        self.kinds = []

    def checkpoint(self, extra=b"", base=None):
        jp = str(self.path) + ".journal"
        if base is None:          # the fixed rule: a base after the journal outgrew its base, or with no chain yet
            base = self.prev is None or os.path.getsize(jp) > os.path.getsize(self.path)
        self.a.checkpoint_enqueue_incremental(str(self.path), extra=extra)
        assert self.a.checkpoint_wait()
        want = self.tmp / "want.dsm"
        self.b.map_save(str(want), extra=extra)
        raw = want.read_bytes()
        self.records = 0 if base else self.records + 1
        self.kinds.append("base" if base else "record")
        assert capi.map_peek_journal(self.path)[2] == self.records, self.kinds
        out = self.tmp / "resolved.dsm"
        capi.journal_materialize(self.path, out)
        assert out.read_bytes() == raw, self.kinds
        if base:
            assert self.path.read_bytes() == raw
        else:                     # exactly the chunks that differ between the two dsm_map_save files
            _, p0, s0, _, _, _ = parse(self.prev)
            _, p1, s1, _, _, _ = parse(raw)
            assert last_record(self.path) == (changed(p0, p1), changed(s0, s1)), self.kinds
        self.prev = raw


@pytest.mark.parametrize("save", sorted(SAVES))
@pytest.mark.parametrize("chunk", [1, 4, 8])
@pytest.mark.parametrize("constants", ["drive", "rgbd"])
def test_every_checkpoint_resolves_to_map_save(tmp_path, save, chunk, constants):
    """A checkpoint after every call, with the loop-closure warp of the save point before or after its checkpoint."""
    lists = simple_lists()
    k, when = SAVES[save]
    a, b = journal_ctx(constants, store=STORE), made(constants, store=STORE)
    j = Journal(tmp_path, a, b)
    bounds = sorted(set(list(range(0, T, chunk)) + [k, T]))
    for s, e in zip(bounds, bounds[1:]):
        for c in (a, b):
            run(c, lists, s, e, chunk)
        if e == k and when == "before":
            kfs = stored_keyframes(b)
            loop_warp(a, kfs)
            loop_warp(b, kfs)
        j.checkpoint(extra=bytes([e]) * 3)
        if e == k and when == "after":
            kfs = stored_keyframes(b)
            loop_warp(a, kfs)
            loop_warp(b, kfs)
            j.checkpoint(extra=b"warp")
    assert j.kinds[0] == "base" and j.kinds[1] == "record"
    assert sorted(os.listdir(tmp_path)) == ["map.dsm", "map.dsm.journal", "resolved.dsm", "want.dsm"]
    a.close()
    b.close()


def test_a_base_after_every_trigger(tmp_path):
    lists = simple_lists()
    a, b = journal_ctx(store=STORE), made(store=STORE)
    j = Journal(tmp_path, a, b)

    def step(t0, t1):
        for c in (a, b):
            run(c, lists, t0, t1, t1 - t0)

    step(0, 4)
    j.checkpoint()
    step(4, 5)
    j.checkpoint(base=False)
    # another path, then back: each is a base
    other = Journal(tmp_path, a, b, name="other.dsm")
    other.checkpoint(base=True)
    j.checkpoint(base=True)
    step(5, 6)
    j.checkpoint(base=False)
    # a full checkpoint rewrites the device image
    a.checkpoint_enqueue(str(tmp_path / "full.dsm"))
    assert a.checkpoint_wait()
    j.checkpoint(base=True)
    # the map replaced: dsm_map_load, dsm_map_load_journal, dsm_inactive_load
    step(6, 7)
    j.checkpoint(base=False)
    a.map_save(str(tmp_path / "now.dsm"))
    a.map_load(str(tmp_path / "now.dsm"))
    j.checkpoint(base=True)
    step(7, 8)
    j.checkpoint(base=False)
    assert a.map_load_journal(str(j.path))[1] == 1
    j.checkpoint(base=True)
    step(8, 9)
    j.checkpoint(base=False)
    a.inactive_load(a.inactive_download(-1), a.inactive_segments())
    j.checkpoint(base=True)
    # the constants
    step(9, 10)
    j.checkpoint(base=False)
    a.set_constants(capi.CONSTANTS_DRIVE)
    j.checkpoint(base=True)
    # the journal outgrows its base: a warp of the pool and of every stored keyframe changes every chunk, so the third
    # record after a base would make it larger than the base
    for t in range(10, 14):
        step(t, t + 1)
        kfs = stored_keyframes(b)
        loop_warp(a, kfs)
        loop_warp(b, kfs)
        j.checkpoint()
    assert "base" in j.kinds[-4:], j.kinds
    # dsm_inactive_reserve (on an empty store)
    c, d = journal_ctx(store=0), made(store=0)
    for x in (c, d):
        x.inactive_reserve(STORE // 2)
        windowed(x, 0, 3, lists, want_counts=False, empty=True)
    jc = Journal(tmp_path, c, d, name="c.dsm")
    jc.checkpoint(base=True)
    jc.checkpoint(base=False)
    c.inactive_reserve(STORE)
    d.inactive_reserve(STORE)
    jc.checkpoint(base=True)
    for x in (a, b, c, d):
        x.close()


def test_a_rejected_frame_writes_no_record_and_then_a_base(tmp_path):
    lists = simple_lists()
    first = next(t for t in range(T) if lists[t][1])
    assert first >= 2
    a, b = new_ctx(store=1), new_ctx(store=1)              # the first retirement does not fit
    a.checkpoint_enable()
    j = Journal(tmp_path, a, b)
    for c in (a, b):
        run(c, lists, 0, first - 1, 1)
    j.checkpoint(base=True)
    for c in (a, b):
        run(c, lists, first - 1, first, 1)
    j.checkpoint(base=False)
    base, journal = j.path.read_bytes(), (tmp_path / "map.dsm.journal").read_bytes()
    windowed(a, first, first + 2, lists, want_counts=False)
    a.checkpoint_enqueue_incremental(str(j.path))
    with pytest.raises(capi.DsmError) as e:
        a.checkpoint_wait()
    assert e.value.code == DSM_E_CAPACITY
    assert j.path.read_bytes() == base and (tmp_path / "map.dsm.journal").read_bytes() == journal
    with pytest.raises(capi.DsmError) as e:
        a.pool_size()                                     # the next synchronising reader reports and clears it
    assert e.value.code == DSM_E_CAPACITY
    j.checkpoint(base=True)                               # the map of the last applied frame, as a base
    a.close()
    b.close()


@pytest.mark.parametrize("chunk,every", [(1, 1), (4, 1), (1, 3)])
def test_journal_checkpoints_leave_the_map_as_a_drive_without_them(tmp_path, chunk, every):
    """Checkpoints polled without blocking on the next calls; pool, store, table and both clouds equal the same drive
    without checkpoints after every call."""
    lists = simple_lists()
    a, b = journal_ctx(store=STORE), made(store=STORE)
    a.publish_enable()
    b.publish_enable()
    path, pending, n = str(tmp_path / "map.dsm"), False, 0
    for i, s in enumerate(range(0, T, chunk)):
        for c in (a, b):
            run(c, lists, s, min(T, s + chunk), chunk)
            c.publish_enqueue(5)
        if pending and a.checkpoint_wait(block=False):
            pending = False
        if i % every == 0 and not pending:
            a.checkpoint_enqueue_incremental(path, extra=bytes([i]))
            pending, n = True, n + 1
        pa, pb = a.publish_wait(), b.publish_wait()
        assert pa[0].tobytes() == pb[0].tobytes() and pa[1].tobytes() == pb[1].tobytes()
        assert readers(a) == readers(b), f"frames {s}-{min(T, s + chunk) - 1}"
    if pending:
        assert a.checkpoint_wait()
    assert n > 1 and readers(a) == readers(b)
    a.close()
    b.close()


@pytest.mark.parametrize("k", [10, 14])
def test_resume_from_the_journal(tmp_path, k):
    lists = simple_lists()
    a, ref = journal_ctx(store=STORE), made(store=STORE)
    path = str(tmp_path / "map.dsm")
    for s in range(0, k, 2):
        for c in (a, ref):
            run(c, lists, s, min(k, s + 2), 2)
        a.checkpoint_enqueue_incremental(path, extra=b"resume %d" % s)
        assert a.checkpoint_wait()
    for _ in range(2):                                    # if the first is a base (the journal outgrew it), the second is a record
        a.checkpoint_enqueue_incremental(path, extra=b"resume")
        assert a.checkpoint_wait()
    extra, table, n = capi.map_peek_journal(path)
    assert extra == b"resume" and n >= 1
    b = made(store=STORE)
    assert b.map_load_journal(path) == (extra, n)
    assert readers(b) == readers(ref)
    for s in range(k, T, 2):
        for c in (b, ref):
            run(c, lists, s, min(T, s + 2), 2)
        assert readers(b) == readers(ref), f"frames from {s}"
    for c in (a, b, ref):
        c.close()


# ---- the node ----
N_NODE = 24


# every: messages between incremental saves; j: messages fed before node B resumes from A's journal
@pytest.mark.parametrize("drift_free_poses,every,j", [(1, 6, 3 * 16 + 1), (10, 3, 3 * 9 + 2), (2, 9, 3 * 13 + 3)])
def test_node_save_state_incremental(tmp_path, drift_free_poses, every, j):
    cam = synth.KITTI
    sc = node_script(cam, N_NODE)
    args = [drift_free_poses, every, j, tmp_path / "a.dsm"]
    out = run_driver("checkpoint_journal_main", str(tmp_path), cam, sc, args, after=[tmp_path]).take(np.int32, -1).tolist()
    n_rest = 3 * N_NODE - j
    n_saves = -(-j // every)
    assert len(out) == 2 + 2 * n_saves + 3 + 3 * n_rest + 1
    assert out[:2] == [0, 0], "enable on A; twin"
    saves = out[2:2 + 2 * n_saves]
    assert saves[0::2] == [0] * n_saves, "every incremental save of A"
    counts = saves[1::2]
    assert counts[0] == 0 and max(counts) >= 1, f"records after each save: {counts}"
    assert all(c == 0 or c == p + 1 for p, c in zip(counts, counts[1:])), counts
    o = 2 + 2 * n_saves
    assert out[o:o + 3] == [0, counts[-1], 1], "load_state_incremental, records applied, equal after it"
    o += 3
    for m in range(n_rest):
        rb, rt, same = out[o + 3 * m: o + 3 * m + 3]
        assert rb == rt == 0 and same == 1, f"message {j + m}: node B {rb}, twin {rt}, equal {same}"
    assert out[o + 3 * n_rest] == 0, "the files were written"
    for x in ("ply", "pcd"):
        assert (tmp_path / f"b.{x}").read_bytes() == (tmp_path / f"t.{x}").read_bytes(), x
    assert os.path.getsize(tmp_path / "t.ply") > 1000
