"""CPU tests of the journal of incremental checkpoints (dsm_map_peek_journal / dsm_journal_materialize, DESIGN.md §8.6):
a base written with numpy from the version-1 layout plus records written by this module's restatement of the journal
layout resolve to the version-1 file of the final state, byte for byte; a torn, corrupted, foreign or out-of-sequence
record ends the replay; malformed chunk lists are refused; the calls are exported and check their arguments."""
import ctypes
import os

import numpy as np
import pytest

from densesurfelmapping_b200 import capi
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from test_checkpoint_format import build, fnv1a64

JHEADER = np.dtype([("magic", "S8"), ("format", "<u4"), ("zero", "<u4"), ("base", "<u8")])
RHEADER = np.dtype([("sequence", "<u8"), ("n_pool", "<i4"), ("n_store", "<i4"), ("n_segments", "<i4"), ("k_pool", "<i4"),
                    ("k_store", "<i4"), ("zero", "<u4"), ("extra_bytes", "<u8")])
MAGIC, FORMAT, CHUNK = b"DSMJRNL", 1, 256
CALLS = ["dsm_checkpoint_enqueue_incremental", "dsm_map_load_journal", "dsm_map_peek_journal", "dsm_journal_materialize"]
E_INVALID = -1


def u64(v):
    return np.array([v], "<u8").tobytes()


def checksum(raw):
    return int(np.frombuffer(raw[-8:], "<u8")[0])


def journal_header(base_sum):
    h = np.zeros(1, JHEADER)
    h["magic"], h["format"], h["base"] = MAGIC, FORMAT, base_sum
    return h.tobytes() + u64(fnv1a64(h.tobytes()))


def changed(old, new):
    """Indices of the 256-surfel chunks of `new` that differ from `old` or reach beyond its size (what k_map_delta flags)."""
    out = []
    for c in range((len(new) + CHUNK - 1) // CHUNK):
        a, b = c * CHUNK, min(len(new), c * CHUNK + CHUNK)
        if b > len(old) or old[a:b].tobytes() != new[a:b].tobytes():
            out.append(c)
    return out


def record(seq, prev_sum, state, pool_chunks, store_chunks):
    """One record's bytes and its own checksum: state = (pool, store, table, extra) after it."""
    pool, store, table, extra = state
    h = np.zeros(1, RHEADER)
    h["sequence"], h["n_pool"], h["n_store"], h["n_segments"] = seq, len(pool), len(store), len(table)
    h["k_pool"], h["k_store"], h["extra_bytes"] = len(pool_chunks), len(store_chunks), len(extra)
    body = h.tobytes() + np.asarray(pool_chunks, "<i4").tobytes() + np.asarray(store_chunks, "<i4").tobytes()
    for sec, chunks in ((pool, pool_chunks), (store, store_chunks)):
        for c in chunks:
            body += sec[c * CHUNK:c * CHUNK + CHUNK].tobytes()
    body += np.asarray(table, np.int32).tobytes() + bytes(extra) + u64(prev_sum)
    own = fnv1a64(body)
    return body + u64(own), own


def states():
    """Four consecutive map states: growth, an edit plus a shrink, and no change at all."""
    rng = np.random.default_rng(7)

    def surfels(n):
        s = np.zeros(n, SURFEL_DTYPE)
        for f in ("px", "py", "pz", "nx", "ny", "nz", "size", "color", "weight"):
            s[f] = rng.standard_normal(n)
        s["update_times"], s["last_update"] = 1 + rng.integers(0, 9, n), rng.integers(0, 20, n)
        return s

    p0, s0 = surfels(600), surfels(700)
    t0 = np.array([[3, 0, 300], [1, 300, 400]], np.int32)
    p1, s1 = p0.copy(), np.concatenate([s0, surfels(500)])       # a pool edit in chunk 1, the store grows
    p1["px"][300] += 1
    t1 = np.concatenate([t0, [[5, 700, 500]]]).astype(np.int32)
    p2, s2 = p1[:300].copy(), s1.copy()                          # the pool shrinks into chunk 1, one stored surfel moves
    s2["pz"][10] = 42.0
    t2 = t1.copy()
    p3 = p2.copy()
    p3["size"][299] = 3.0                                        # the last record: one small chunk
    return [(p0, s0, t0, b"node 0"), (p1, s1, t1, b"node one"), (p2, s2, t2, b""), (p3, s2, t2, b"n3")]


def write_chain(tmp_path, sts, name="map.dsm"):
    """The base (first state) and a journal with one record per later state; (path, [record bytes])."""
    path = tmp_path / name
    base = build(*sts[0])
    path.write_bytes(base)
    prev, recs = checksum(base), []
    for i in range(1, len(sts)):
        rec, prev = record(i, prev, sts[i], changed(sts[i - 1][0], sts[i][0]), changed(sts[i - 1][1], sts[i][1]))
        recs.append(rec)
    (tmp_path / (name + ".journal")).write_bytes(journal_header(checksum(base)) + b"".join(recs))
    return path, recs


def materialized(path, tmp_path):
    out = tmp_path / "out.dsm"
    capi.journal_materialize(path, out)
    return out.read_bytes()


def test_calls_are_exported_and_declared():
    lib = capi.load_library()
    for name in CALLS:
        assert name in capi.EXPORTS and hasattr(lib, name), name


def test_null_arguments_are_invalid_without_a_device(tmp_path):
    L = capi.load_library()
    p, q = os.fsencode(tmp_path / "map.dsm"), os.fsencode(tmp_path / "out.dsm")
    sz, n = ctypes.c_size_t(0), ctypes.c_int(7)
    assert L.dsm_checkpoint_enqueue_incremental(None, p, None, 0) == E_INVALID
    assert L.dsm_map_load_journal(None, p, None, 0, ctypes.byref(sz), ctypes.byref(n)) == E_INVALID and n.value == 0
    assert L.dsm_map_peek_journal(None, None, 0, None, None, 0, None, None) == E_INVALID
    assert L.dsm_map_peek_journal(p, None, 4, None, None, 0, None, None) == E_INVALID
    assert L.dsm_journal_materialize(None, q) == E_INVALID and L.dsm_journal_materialize(p, None) == E_INVALID
    assert os.listdir(tmp_path) == []


def test_materialize_equals_the_final_state(tmp_path):
    sts = states()
    path, recs = write_chain(tmp_path, sts)
    # the last record: its header, one index, the pool's last chunk cut at 44 surfels, the table, extra, two checksums
    assert len(recs[-1]) == 40 + 4 + 44 * 44 + 3 * 12 + 2 + 16
    assert materialized(path, tmp_path) == build(*sts[-1])
    extra, table, n = capi.map_peek_journal(path)
    assert (extra, table.tolist(), n) == (sts[-1][3], sts[-1][2].tolist(), 3)
    # every prefix of whole records is a state of its own
    j = (tmp_path / "map.dsm.journal").read_bytes()
    for k in range(len(recs) + 1):
        (tmp_path / "map.dsm.journal").write_bytes(j[:32 + sum(len(r) for r in recs[:k])])
        assert materialized(path, tmp_path) == build(*sts[k]) and capi.map_peek_journal(path)[2] == k
    # no journal: the base alone, and dsm_map_peek of the base is untouched by the journal
    os.remove(tmp_path / "map.dsm.journal")
    assert materialized(path, tmp_path) == build(*sts[0]) and capi.map_peek_journal(path)[2] == 0


def test_a_torn_last_record_gives_the_previous_state(tmp_path):
    sts = states()
    path, recs = write_chain(tmp_path, sts)
    full = (tmp_path / "map.dsm.journal").read_bytes()
    want = build(*sts[-2])
    for cut in range(1, len(recs[-1])):
        (tmp_path / "map.dsm.journal").write_bytes(full[:-cut])
        assert materialized(path, tmp_path) == want, cut
    assert capi.map_peek_journal(path)[2] == 2


def test_a_flipped_byte_in_the_last_record_gives_the_previous_state(tmp_path):
    sts = states()
    path, recs = write_chain(tmp_path, sts)
    full = (tmp_path / "map.dsm.journal").read_bytes()
    start = len(full) - len(recs[-1])
    for o in range(start, len(full)):
        for bit in (0x01, 0x80):
            bad = bytearray(full)
            bad[o] ^= bit
            (tmp_path / "map.dsm.journal").write_bytes(bytes(bad))
            assert capi.map_peek_journal(path)[2] == 2, (o - start, bit)
    assert materialized(path, tmp_path) == build(*sts[-2])


def test_a_journal_of_another_base_is_ignored(tmp_path):
    sts = states()
    path, _ = write_chain(tmp_path, sts)
    other = build(sts[0][0], sts[0][1], sts[0][2], b"another base")
    path.write_bytes(other)                                      # a crash between the base's rename and the journal's
    assert materialized(path, tmp_path) == other and capi.map_peek_journal(path)[2] == 0
    # a header whose own checksum fails is ignored too
    path.write_bytes(build(*sts[0]))
    j = bytearray((tmp_path / "map.dsm.journal").read_bytes())
    j[20] ^= 1
    (tmp_path / "map.dsm.journal").write_bytes(bytes(j))
    assert capi.map_peek_journal(path)[2] == 0
    # a journal of another magic or format is refused
    for o, v in ((0, ord("X")), (8, FORMAT + 1)):
        j = bytearray(journal_header(checksum(build(*sts[0]))))
        j[o] = v
        (tmp_path / "map.dsm.journal").write_bytes(bytes(j))
        with pytest.raises(capi.DsmError) as e:
            capi.map_peek_journal(path)
        assert e.value.code == E_INVALID


def test_records_out_of_sequence_or_off_the_chain_end_the_replay(tmp_path):
    sts = states()
    path = tmp_path / "map.dsm"
    base = build(*sts[0])
    path.write_bytes(base)
    s = checksum(base)
    r1, s1 = record(1, s, sts[1], changed(sts[0][0], sts[1][0]), changed(sts[0][1], sts[1][1]))
    r2, s2 = record(2, s1, sts[2], changed(sts[1][0], sts[2][0]), changed(sts[1][1], sts[2][1]))
    r3, _ = record(3, s2, sts[3], changed(sts[2][0], sts[3][0]), [])
    cases = {
        "sequence skips": record(3, s1, sts[2], changed(sts[1][0], sts[2][0]), changed(sts[1][1], sts[2][1]))[0],
        "sequence repeats": record(1, s1, sts[2], changed(sts[1][0], sts[2][0]), changed(sts[1][1], sts[2][1]))[0],
        "chained to the base": record(2, s, sts[2], changed(sts[1][0], sts[2][0]), changed(sts[1][1], sts[2][1]))[0],
    }
    for what, bad in cases.items():
        (tmp_path / "map.dsm.journal").write_bytes(journal_header(s) + r1 + bad + r3)
        assert materialized(path, tmp_path) == build(*sts[1]), what
        assert capi.map_peek_journal(path)[2] == 1, what
    (tmp_path / "map.dsm.journal").write_bytes(journal_header(s) + r1 + r2 + r3)
    assert materialized(path, tmp_path) == build(*sts[3])


def test_malformed_chunk_lists_are_invalid(tmp_path):
    sts = states()
    path = tmp_path / "map.dsm"
    base = build(*sts[0])
    path.write_bytes(base)
    s = checksum(base)
    grown = changed(sts[0][1], sts[1][1])                        # store chunks 2 .. 4: the growth from 700 to 1200
    assert grown == [2, 3, 4]
    cases = {
        "descending": ([1], [4, 3, 2]),
        "repeated": ([1, 1], grown),
        "past the pool": ([1, 3], grown),
        "negative": ([-1, 1], grown),
        "growth chunk missing": ([1], [2, 4]),
        "growth not listed": ([1], [2, 3]),
    }
    for what, (pc, sc) in cases.items():
        rec, _ = record(1, s, sts[1], pc, sc)
        (tmp_path / "map.dsm.journal").write_bytes(journal_header(s) + rec)
        L = capi.load_library()
        assert L.dsm_map_peek_journal(os.fsencode(path), None, 0, None, None, 0, None, None) == E_INVALID, what
        assert L.dsm_journal_materialize(os.fsencode(path), os.fsencode(tmp_path / "out.dsm")) == E_INVALID, what
    # listing an unchanged chunk as well is allowed: a superset is a valid record
    rec, _ = record(1, s, sts[1], [0, 1], [0] + grown)
    (tmp_path / "map.dsm.journal").write_bytes(journal_header(s) + rec)
    assert materialized(path, tmp_path) == build(*sts[1])
    assert not os.path.exists(tmp_path / "out.dsm.tmp")
