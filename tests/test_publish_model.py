"""oracle/pyoracle_publish.mirror_step, the chunk rule of k_cloud_mirror, on hand-made clouds: which 256-point chunks
cross to the host, the lowest changed index and the shadow left behind.  tests/test_gpu_publish.py holds the device to
the same rule (forwarded-chunk count, changed_from)."""
import numpy as np

from pyoracle_publish import CHUNK, mirror_step

CAP = 4 * CHUNK


def cloud(n, seed=0):
    return np.random.default_rng(seed).normal(size=(n, 4)).astype(np.float32)


def publish(shadow, prev, c):
    """One snapshot; also what the host mirror must hold afterwards: the cloud, from the forwarded chunks alone."""
    chunks, cf, new = mirror_step(shadow, prev, c)
    assert new[:len(c)].tobytes() == c.tobytes(), "forwarded chunks + untouched chunks do not add up to the cloud"
    assert new[len(c):].tobytes() == np.asarray(shadow, np.float32)[len(c):].tobytes()
    return chunks, cf, new


def test_first_snapshot_forwards_everything():
    c = cloud(600)
    chunks, cf, _ = publish(np.zeros((CAP, 4), np.float32), 0, c)
    assert chunks == [0, 1, 2] and cf == 0


def test_append_only():
    c = cloud(700)
    _, _, sh = publish(np.zeros((CAP, 4), np.float32), 0, c[:300])
    chunks, cf, _ = publish(sh, 300, c)
    assert chunks == [1, 2] and cf == 300          # chunk 0 is untouched, chunk 1 holds the old tail and the new points


def test_append_forwards_even_when_the_stale_shadow_matches():
    """Indices at or beyond the previous size count as changed whatever the shadow holds there."""
    c = cloud(300)
    _, _, sh = publish(np.zeros((CAP, 4), np.float32), 0, c)
    _, cf, sh = publish(sh, 300, c[:100])
    assert cf == 100
    chunks, cf, _ = publish(sh, 100, c)
    assert chunks == [0, 1] and cf == 100


def test_shrink_and_nothing_changed():
    c = cloud(600)
    _, _, sh = publish(np.zeros((CAP, 4), np.float32), 0, c)
    chunks, cf, sh2 = publish(sh, 600, c[:400])
    assert chunks == [] and cf == 400               # only the size shrank
    chunks, cf, _ = publish(sh2, 400, c[:400])
    assert chunks == [] and cf == 400               # nothing changed


def test_compaction_shift():
    """A segment [100, 150) leaves: everything above moves down by 50."""
    c = cloud(600)
    _, _, sh = publish(np.zeros((CAP, 4), np.float32), 0, c)
    chunks, cf, _ = publish(sh, 600, np.concatenate([c[:100], c[150:]]))
    assert chunks == [0, 1, 2] and cf == 100


def test_in_place_change_in_the_last_partial_chunk():
    c = cloud(600)
    _, _, sh = publish(np.zeros((CAP, 4), np.float32), 0, c)
    d = c.copy()
    d[599, 2] = np.nextafter(d[599, 2], np.float32(10))   # one bit
    chunks, cf, _ = publish(sh, 600, d)
    assert chunks == [2] and cf == 599
    d2 = c.copy()
    d2[10, 3] = -0.0 if c[10, 3] == 0 else -c[10, 3]
    chunks, cf, _ = publish(sh, 600, d2)
    assert chunks == [0] and cf == 10


def test_bitwise_compare():
    c = np.zeros((8, 4), np.float32)
    _, _, sh = publish(np.zeros((CAP, 4), np.float32), 0, c)
    d = c.copy()
    d[3, 0] = -0.0                                     # equal as floats, different bits
    chunks, cf, _ = publish(sh, 8, d)
    assert chunks == [0] and cf == 3
    n = c.copy()
    n[5, 1] = np.nan
    _, _, sh = publish(sh, 8, n)
    chunks, cf, _ = publish(sh, 8, n)                  # a NaN equals itself bit for bit
    assert chunks == [] and cf == 8


def test_size_zero():
    chunks, cf, _ = publish(np.zeros((CAP, 4), np.float32), 0, cloud(0))
    assert chunks == [] and cf == 0
    _, _, sh = publish(np.zeros((CAP, 4), np.float32), 0, cloud(300))
    chunks, cf, _ = publish(sh, 300, cloud(0))
    assert chunks == [] and cf == 0


def test_size_an_exact_multiple_of_the_chunk():
    c = cloud(3 * CHUNK)
    _, _, sh = publish(np.zeros((CAP, 4), np.float32), 0, c[:2 * CHUNK])
    chunks, cf, sh = publish(sh, 2 * CHUNK, c)
    assert chunks == [2] and cf == 2 * CHUNK           # the full chunks below are not touched
    chunks, cf, _ = publish(sh, 3 * CHUNK, c[:2 * CHUNK])
    assert chunks == [] and cf == 2 * CHUNK
