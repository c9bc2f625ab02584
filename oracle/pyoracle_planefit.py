"""TEST INFRASTRUCTURE ONLY -- what the first Gauss-Newton pass of the plane fit (calculate_sp_depth_norms_kernel
:792-871, get_huber_norm :104-188) sees, per seed, restated on the host in float64 from the restatement's own
inputs: which seeds are fitted, their inlier count n, and the first-pass margin min_i | |q_i . n0| - HUBER_RANGE |
(q: the centred inlier points, n0: the normalised sum of the inlier pixel normals, b = 0).

The CUDA solver (csrc/dsm_tile.cu, k_gn_solve) skips a pass over the points only while the accumulated step bound
plus 2e-3 stays below that margin; its first step alone adds at least 1e-4, so a seed whose margin is below
2e-3 + 1e-4 is always queued for its phase B.  Tests use the sufficient condition margin < 2e-3 - 1e-4, which leaves
2e-4 for the difference between this float64 value and the kernel's float one.
"""
import numpy as np

SP = 8


def first_pass(cam, labels, seeds, depth, normals, huber_range):
    """labels / seeds after the third update (Restatement.debug_iters(..., 3, True)), the pixel normals
    (Restatement.norm_map() after superpixels()).  Returns per-seed arrays: fitted (bool), n (inlier count, 0 when not
    fitted), margin (float64; inf when not fitted, NaN when n0 is NaN)."""
    H, W = labels.shape
    spw = W // SP
    S = len(seeds)
    lab = np.asarray(labels).reshape(-1)
    dep = np.asarray(depth, np.float32).reshape(-1)
    nrm = np.asarray(normals, np.float32).reshape(-1, 3).astype(np.float64)
    col = (np.arange(W * H) % W).astype(np.float32)
    row = (np.arange(W * H) // W).astype(np.float32)
    # back_project in float (:91-97): the reference's space map
    px = (col - np.float32(cam.cx)) / np.float32(cam.fx) * dep
    py = (row - np.float32(cam.cy)) / np.float32(cam.fy) * dep
    pts = np.stack([px, py, dep], -1).astype(np.float64)
    h = float(huber_range)
    fitted = np.zeros(S, bool)
    n_inl = np.zeros(S, np.int64)
    margin = np.full(S, np.inf)
    off = (np.arange(2 * SP)[:, None] * W + np.arange(2 * SP)[None, :]).reshape(-1)
    for s in range(S):
        xb, yb = (s % spw) * SP - SP // 2, (s // spw) * SP - SP // 2
        pi = yb * W + xb + off  # window bounded by the flat index only (:816)
        pi = pi[(pi >= 0) & (pi < W * H)]
        pi = pi[lab[pi] == s]
        pi = pi[dep[pi].astype(np.float64) > 0.05]
        if len(pi) < 16:
            continue
        r = (np.float32(seeds["mean_depth"][s]) - dep[pi]).astype(np.float64)
        inl = pi[(r < h) & (r > -h)]
        if float(np.float32(len(inl)) / np.float32(len(pi))) < 0.8:
            continue
        fitted[s] = True
        n_inl[s] = len(inl)
        sn = nrm[inl].sum(0)
        with np.errstate(invalid="ignore", divide="ignore"):
            n0 = sn / np.sqrt((sn * sn).sum())
        q = pts[inl] - pts[inl].mean(0)
        margin[s] = np.abs(np.abs(q @ n0) - h).min()
    return {"fitted": fitted, "n": n_inl, "margin": margin}
