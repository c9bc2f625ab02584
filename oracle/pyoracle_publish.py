"""The chunk rule of k_cloud_mirror (dsm_publish_enqueue) restated in numpy: which 256-point chunks of the inactive cloud
are forwarded to the host mirror, the lowest changed index, and the shadow the device keeps afterwards."""
import numpy as np

CHUNK = 256


def mirror_step(shadow, prev_size, cloud):
    """shadow: (cap, 4) float32, the cloud as the host last received it, [0, prev_size) of it published; cloud: (n, 4)
    float32, the store's points now.  Returns (forwarded chunk indices, changed_from, new shadow).  Points compare bit
    for bit; an index at or beyond prev_size counts as changed; changed_from = n when no index below n changed.  A
    forwarded chunk is rewritten whole (its points below n); every other point of the shadow keeps its old value."""
    cloud = np.ascontiguousarray(cloud, np.float32).reshape(-1, 4)
    shadow = np.array(shadow, np.float32).reshape(-1, 4)
    n = len(cloud)
    assert n <= len(shadow)
    changed = np.ones(n, bool)
    m = min(n, prev_size)
    changed[:m] = (cloud[:m].view(np.uint32) != shadow[:m].view(np.uint32)).any(1)
    idx = np.nonzero(changed)[0]
    changed_from = int(idx[0]) if len(idx) else n
    chunks = sorted(set((idx // CHUNK).tolist()))
    for c in chunks:
        a, b = c * CHUNK, min(n, (c + 1) * CHUNK)
        shadow[a:b] = cloud[a:b]
    return chunks, changed_from, shadow
