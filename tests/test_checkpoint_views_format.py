"""CPU tests of the views in the checkpoint files (DESIGN.md §8.18): a version-2 map file and a version-2 journal, written
here with numpy from the documented layouts, are peeked and materialised by the library; a chain resolves to the file of
its final state, byte for byte; a torn or corrupted last record gives the previous state; a wrong rays-per-view word,
a malformed slot list and a journal of the other version are refused."""
import os

import numpy as np
import pytest

from densesurfelmapping_b200 import capi
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from checkpoint_files import CHUNK, HEADER, JHEADER, RHEADER, build, changed, fnv1a64

E_INVALID = -1
W, H = 16, 8                      # S = (16 / 8) * (8 / 8) = 2 rays per view
S = (W // 8) * (H // 8)
GEOMETRY = (20.0, 20.0, 7.5, 3.5, 30.0, 0.5)


def u64(v):
    return np.array([v], "<u8").tobytes()


def checksum(raw):
    return int(np.frombuffer(raw[-8:], "<u8")[0])


def build_views(pool, store, table, extra, views, rays_per_view=S):
    """The version-2 file: version 1's sections with the views section after the table.  views: {slot: [S, 4] float32}."""
    v1 = build(pool, store, table, extra, width=W, height=H, geometry=GEOMETRY)
    h = np.frombuffer(v1, HEADER, 1).copy()
    h["format"], h["zero"] = 2, rays_per_view
    slots = sorted(views)
    sec = np.array([len(slots)], "<i4").tobytes() + np.asarray(slots, "<i4").tobytes()
    sec += b"".join(np.ascontiguousarray(views[s], np.float32).tobytes() for s in slots)
    o = HEADER.itemsize + len(pool) * SURFEL_DTYPE.itemsize + len(store) * SURFEL_DTYPE.itemsize + 12 * len(table)
    body = h.tobytes() + v1[HEADER.itemsize:o] + sec + bytes(extra)
    return body + u64(fnv1a64(body))


def build_plain(pool, store, table, extra):
    return build(pool, store, table, extra, width=W, height=H, geometry=GEOMETRY)


def journal_header(base_sum, fmt=2, rays_per_view=S):
    h = np.zeros(1, JHEADER)
    h["magic"], h["format"], h["zero"], h["base"] = b"DSMJRNL", fmt, rays_per_view, base_sum
    return h.tobytes() + u64(fnv1a64(h.tobytes()))


def record(seq, prev_sum, state, pool_chunks, store_chunks, views):
    """One version-2 record's bytes and its checksum: state = (pool, store, table, extra) after it, views = {slot: rays}
    captured since the previous state (written in the given key order)."""
    pool, store, table, extra = state
    slots = list(views)
    h = np.zeros(1, RHEADER)
    h["sequence"], h["n_pool"], h["n_store"], h["n_segments"] = seq, len(pool), len(store), len(table)
    h["k_pool"], h["k_store"], h["zero"], h["extra_bytes"] = len(pool_chunks), len(store_chunks), len(slots), len(extra)
    body = h.tobytes() + np.asarray(pool_chunks, "<i4").tobytes() + np.asarray(store_chunks, "<i4").tobytes()
    body += np.asarray(slots, "<i4").tobytes()
    for sec, chunks in ((pool, pool_chunks), (store, store_chunks)):
        for c in chunks:
            body += sec[c * CHUNK:c * CHUNK + CHUNK].tobytes()
    body += b"".join(np.ascontiguousarray(views[s], np.float32).tobytes() for s in slots)
    body += np.asarray(table, np.int32).tobytes() + bytes(extra) + u64(prev_sum)
    own = fnv1a64(body)
    return body + u64(own), own


def rays(seed):
    r = np.random.default_rng(seed).standard_normal((S, 4)).astype(np.float32)
    r[:, 3] = 1.0
    r[seed % S] = 0.0                                            # a seed without a ray
    return r


def states():
    """Four map states with the views filled after each: captures into new and old slots, then none."""
    rng = np.random.default_rng(11)

    def surfels(n):
        s = np.zeros(n, SURFEL_DTYPE)
        for f in ("px", "py", "pz", "nx", "ny", "nz", "size", "color", "weight"):
            s[f] = rng.standard_normal(n)
        s["update_times"], s["last_update"] = 1 + rng.integers(0, 9, n), rng.integers(0, 20, n)
        return s

    p0, s0 = surfels(300), surfels(100)
    t0 = np.array([[3, 0, 100]], np.int32)
    p1 = np.concatenate([p0, surfels(10)])
    p2 = p1.copy()
    p2["px"][5] += 1
    v0 = {2: rays(1), 7: rays(2)}
    v1 = {3: rays(3), 4: rays(4), 7: rays(5)}                    # two new slots and a recapture
    v2 = {0: rays(6)}
    maps = [(p0, s0, t0, b"node 0"), (p1, s0, t0, b"node one"), (p2, s0, t0, b""), (p2, s0, t0, b"n3")]
    captures = [v0, v1, v2, {}]
    filled, out = {}, []
    for m, v in zip(maps, captures):
        filled = {**filled, **v}
        out.append((m, v, dict(filled)))
    return out


def write_chain(tmp_path, sts, name="map.dsm"):
    path = tmp_path / name
    base = build_views(*sts[0][0], sts[0][2])
    path.write_bytes(base)
    prev, recs = checksum(base), []
    for i in range(1, len(sts)):
        (a, _, _), (b, v, _) = sts[i - 1], sts[i]
        rec, prev = record(i, prev, b, changed(a[0], b[0]), changed(a[1], b[1]), dict(sorted(v.items())))
        recs.append(rec)
    (tmp_path / (name + ".journal")).write_bytes(journal_header(checksum(base)) + b"".join(recs))
    return path, recs


def final(sts, k):
    return build_views(*sts[k][0], sts[k][2])


def materialized(path, tmp_path):
    out = tmp_path / "out.dsm"
    capi.journal_materialize(path, out)
    return out.read_bytes()


def peek_rc(path):
    return capi.load_library().dsm_map_peek(os.fsencode(path), None, 0, None, None, 0, None)


def journal_rc(path):
    return capi.load_library().dsm_map_peek_journal(os.fsencode(path), None, 0, None, None, 0, None, None)


def test_the_call_is_exported_and_checks_its_context():
    L = capi.load_library()
    assert "dsm_checkpoint_views_enable" in capi.EXPORTS and hasattr(L, "dsm_checkpoint_views_enable")
    assert L.dsm_checkpoint_views_enable(None) == E_INVALID


def test_a_views_file_is_peeked_and_materialised_unchanged(tmp_path):
    (m, _, views) = states()[1]
    path = tmp_path / "map.dsm"
    raw = build_views(*m, views)
    path.write_bytes(raw)
    extra, table = capi.map_peek(path)
    assert extra == m[3] and table.tolist() == m[2].tolist()
    assert materialized(path, tmp_path) == raw
    # an empty views section is a file of its own, not a version-1 file
    empty = build_views(*m, {})
    path.write_bytes(empty)
    assert capi.map_peek(path)[0] == m[3] and materialized(path, tmp_path) == empty
    assert empty != build_plain(*m)


def test_base_and_records_materialise_to_the_final_state(tmp_path):
    sts = states()
    path, recs = write_chain(tmp_path, sts)
    assert materialized(path, tmp_path) == final(sts, 3)
    extra, table, n = capi.map_peek_journal(path)
    assert (extra, table.tolist(), n) == (sts[3][0][3], sts[3][0][2].tolist(), 3)
    j = (tmp_path / "map.dsm.journal").read_bytes()
    for k in range(len(recs) + 1):
        (tmp_path / "map.dsm.journal").write_bytes(j[:32 + sum(len(r) for r in recs[:k])])
        assert materialized(path, tmp_path) == final(sts, k) and capi.map_peek_journal(path)[2] == k


def test_a_cut_or_flipped_last_record_gives_the_previous_state(tmp_path):
    sts = states()
    sts[3] = (sts[3][0], {5: rays(9)}, {**sts[2][2], 5: rays(9)})   # a last record that carries a view
    path, recs = write_chain(tmp_path, sts)
    full = (tmp_path / "map.dsm.journal").read_bytes()
    want = final(sts, 2)
    for cut in range(1, len(recs[-1]) + 1):
        (tmp_path / "map.dsm.journal").write_bytes(full[:-cut])
        assert materialized(path, tmp_path) == want, cut
    start = len(full) - len(recs[-1])
    for o in range(start, len(full)):
        for bit in (0x01, 0x80):
            bad = bytearray(full)
            bad[o] ^= bit
            (tmp_path / "map.dsm.journal").write_bytes(bytes(bad))
            assert capi.map_peek_journal(path)[2] == 2, (o - start, bit)
    (tmp_path / "map.dsm.journal").write_bytes(full[:start])
    assert materialized(path, tmp_path) == want


def test_a_wrong_rays_per_view_word_is_invalid(tmp_path):
    (m, _, views) = states()[1]
    path = tmp_path / "map.dsm"
    for word in (0, S - 1, S + 1, -S):
        path.write_bytes(build_views(*m, views, rays_per_view=word) if word > 0 else
                         build_views(*m, {}, rays_per_view=word))
        assert peek_rc(path) == E_INVALID, word
    # the journal's word is checked against its base before the header's checksum
    base = build_views(*m, views)
    path.write_bytes(base)
    for word in (0, S + 1):
        (tmp_path / "map.dsm.journal").write_bytes(journal_header(checksum(base), 2, word))
        assert journal_rc(path) == E_INVALID, word
        j = bytearray(journal_header(checksum(base)))
        j[12] = word                                                 # the checksum no longer matches either
        (tmp_path / "map.dsm.journal").write_bytes(bytes(j))
        assert journal_rc(path) == E_INVALID, word


def test_malformed_slot_lists_are_invalid(tmp_path):
    (m, _, _) = states()[1]
    path = tmp_path / "map.dsm"
    for what, slots in {"descending": [5, 2], "repeated": [3, 3], "negative": [-1, 2]}.items():
        raw = bytearray(build_views(*m, {i: rays(i) for i in range(len(slots))}))
        o = HEADER.itemsize + (len(m[0]) + len(m[1])) * SURFEL_DTYPE.itemsize + 12 * len(m[2]) + 4
        raw[o:o + 4 * len(slots)] = np.asarray(slots, "<i4").tobytes()
        raw[-8:] = u64(fnv1a64(bytes(raw[:-8])))
        path.write_bytes(bytes(raw))
        assert peek_rc(path) == E_INVALID, what
    base = build_views(*m, {1: rays(1)})
    path.write_bytes(base)
    for what, views in {"descending": {5: rays(1), 2: rays(2)}, "negative": {-3: rays(1)}}.items():
        rec, _ = record(1, checksum(base), m, [], [], views)
        (tmp_path / "map.dsm.journal").write_bytes(journal_header(checksum(base)) + rec)
        assert journal_rc(path) == E_INVALID, what
        L = capi.load_library()
        assert L.dsm_journal_materialize(os.fsencode(path), os.fsencode(tmp_path / "out.dsm")) == E_INVALID, what
    rec, _ = record(1, checksum(base), m, [], [], {2: rays(1), 6: rays(2)})
    (tmp_path / "map.dsm.journal").write_bytes(journal_header(checksum(base)) + rec)
    assert materialized(path, tmp_path) == build_views(*m, {1: rays(1), 2: rays(1), 6: rays(2)})


def test_a_journal_of_the_other_version_is_invalid(tmp_path):
    (m, _, views) = states()[1]
    path = tmp_path / "map.dsm"
    plain = build_plain(*m)
    path.write_bytes(plain)
    (tmp_path / "map.dsm.journal").write_bytes(journal_header(checksum(plain)))
    assert journal_rc(path) == E_INVALID
    base = build_views(*m, views)
    path.write_bytes(base)
    (tmp_path / "map.dsm.journal").write_bytes(journal_header(checksum(base), 1, 0))
    assert journal_rc(path) == E_INVALID
    # a journal left beside an earlier base of the other version names that base's checksum: it adds nothing
    (tmp_path / "map.dsm.journal").write_bytes(journal_header(checksum(plain), 1, 0))
    assert journal_rc(path) == 0 and materialized(path, tmp_path) == base


@pytest.mark.parametrize("n_views", [0, 3])
def test_a_truncated_views_file_is_an_io_error(tmp_path, n_views):
    (m, _, views) = states()[1]
    raw = build_views(*m, dict(list(views.items())[:n_views]))
    path = tmp_path / "map.dsm"
    for cut in (1, 8, 9, 16 * S + 8):
        path.write_bytes(raw[:-cut])
        assert peek_rc(path) == -9, cut
