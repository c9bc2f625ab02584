"""TEST INFRASTRUCTURE ONLY -- a host replay of the depth half of update_seeds (fusion_functions.cpp:496-556): the mean
of a seed's member depths and its damped Huber-Newton passes, in float32 entry by entry as the reference, vectorised
over the seeds (loop over the window position).  Besides the final mean_depth it reports which branch of the CUDA
schedule's split the seed takes (csrc/dsm_tile.cu, update_seed_newton in k_gather and k_newton_hard):

  SKIPPED   stable when the update runs: update_seeds leaves it alone (:478-479)
  NO_DEPTH  no member depth > 0.1 (nd == 0): mean_depth = 0
  CHAIN     every pass met only in-range entries: k_gather finishes it after `passes` pure-chain passes
  QUEUED    a pass met an out-of-range entry: k_gather queues it at iteration `passes` (0..4) and k_newton_hard
            continues; `reentry` marks a later pass of k_newton_hard back in the pure chain (every entry in range again)

"In range" is the reference's test (double)r < HUBER_RANGE && (double)r > -HUBER_RANGE on r = fl(md - z), evaluated on
every entry; the kernels decide it from the list's extremes, which is the same thing because r is monotone in z.
tests/test_seed_update_paths.py pins the replay's mean_depth to the restatement (oracle/dsm_oracle.c) bit for bit, so
its branch classification is that of the true arithmetic.
"""
import numpy as np

SKIPPED, NO_DEPTH, CHAIN, QUEUED = 0, 1, 2, 3
BRANCH_NAMES = {SKIPPED: "skipped", NO_DEPTH: "nd == 0", CHAIN: "chain", QUEUED: "queued"}

F32 = np.float32
F64 = np.float64
SP = 8  # SP_SIZE (fusion_functions.h:10)


def window_members(labels, depth):
    """Every seed's 16 x 16 window (clamped, END-EXCLUSIVE at W - 1 / H - 1, :483-489) in raster order:
    (z [S, 256] float32 depths, member [S, 256] labelled with the seed, dep [S, 256] member with (double)depth > 0.1)."""
    H, W = labels.shape
    spw, sph = W // SP, H // SP
    S = spw * sph
    s = np.arange(S)
    x0, y0 = (s % spw) * SP - SP // 2, (s // spw) * SP - SP // 2
    xs = x0[:, None] + np.arange(2 * SP)[None, :]  # [S, 16]
    ys = y0[:, None] + np.arange(2 * SP)[None, :]
    inwin = ((ys >= 0) & (ys < H - 1))[:, :, None] & ((xs >= 0) & (xs < W - 1))[:, None, :]
    yc, xc = np.clip(ys, 0, H - 1)[:, :, None], np.clip(xs, 0, W - 1)[:, None, :]
    member = (inwin & (labels[yc, xc] == s[:, None, None])).reshape(S, -1)
    z = np.asarray(depth, F32)[yc, xc].reshape(S, -1)
    dep = member & (z.astype(F64) > 0.1)
    return z, member, dep


def newton_pass(md, zz, dd, h):
    """One damped Huber-Newton pass (:536-549) of every seed from md over its entries zz where dd: (delta, whether
    every entry was in range)."""
    r = (md[:, None] - zz).astype(F32)
    inr = (r.astype(F64) < h) & (r.astype(F64) > -h)
    sa = np.zeros(len(md), F32)
    sb = np.zeros(len(md), F32)
    for j in range(zz.shape[1]):
        m = dd[:, j]
        rin = F32(sa + F32(2) * r[:, j])  # sum_a += 2 * residual: 2 r is exact
        rout = (sa.astype(F64) + np.where(r[:, j] > 0, h, -1 * h)).astype(F32)
        sa = np.where(m, np.where(inr[:, j], rin, rout), sa)
        sb = np.where(m & inr[:, j], F32(sb + F32(2)), sb)
    delta = ((-sa).astype(F64) / (sb.astype(F64) + 10.0)).astype(F32)
    return delta, (inr | ~dd).all(1)


def replay(labels, seeds, depth, huber_range):
    """One update_seeds pass on the labels its assign left, `seeds` as the update finds them (stable flags, old
    mean_depth).  Returns a dict of per-seed arrays: mean_depth (float32, what the update leaves), nd (member depths
    > 0.1; -1 for a skipped seed), branch, passes, reentry (see the module doc), capped (the loop ran all five passes
    and a sixth would still move mean_depth, so the number of passes left at the hand-off decides the result)."""
    labels = np.asarray(labels)
    S = len(seeds)
    z, member, dep = window_members(labels, depth)
    upd = seeds["stable"] == 0
    if (upd & ~member.any(1)).any():  # the chunk-abandoning `return` (:516-517): never for a supported shape
        raise ValueError("a seed to update owns no pixel of its window: the replay does not model :516-517")
    h = float(huber_range)
    nd = np.where(upd, dep.sum(1), -1)
    act = upd & (nd > 0)
    idx = np.nonzero(act)[0]
    zz, dd = z[idx], dep[idx]

    # mean pass: sequential float sum in raster order (:511), then sum / count in float
    sum_d = np.zeros(len(idx), F32)
    for j in range(zz.shape[1]):
        sum_d = np.where(dd[:, j], sum_d + zz[:, j], sum_d)
    md = sum_d / nd[idx].astype(F32)

    n = len(idx)
    branch = np.full(n, CHAIN, np.int8)
    passes = np.zeros(n, np.int32)
    reentry = np.zeros(n, bool)
    live = np.ones(n, bool)
    for it in range(5):  # :534-554
        delta, allin = newton_pass(md, zz, dd, h)
        newq = live & (branch == CHAIN) & ~allin
        reentry |= live & (branch == QUEUED) & allin
        branch[newq] = QUEUED
        passes[newq] = it
        md = np.where(live, F32(md + delta), md)
        passes[live & (branch == CHAIN)] = it + 1
        live &= ~((delta.astype(F64) < 0.01) & (delta.astype(F64) > -0.01))
    # the iteration cap, not the step test, decided the result: one more pass would still move mean_depth
    capped = live & (F32(md + newton_pass(md, zz, dd, h)[0]) != md)

    out_md = np.array(seeds["mean_depth"], F32, copy=True)
    out_md[upd & (nd == 0)] = F32(0)
    out_md[idx] = md
    out_branch = np.where(upd, NO_DEPTH, SKIPPED).astype(np.int8)
    out_branch[idx] = branch
    out_passes = np.zeros(S, np.int32)
    out_passes[idx] = passes
    out_reentry = np.zeros(S, bool)
    out_reentry[idx] = reentry
    out_capped = np.zeros(S, bool)
    out_capped[idx] = capped
    return {"mean_depth": out_md, "nd": nd, "branch": out_branch, "passes": out_passes, "reentry": out_reentry,
            "capped": out_capped}


def replay_pass(restatement, gray, depth, p):
    """Pass p (1..3) of generate_super_pixels on the restatement: stops after p's assign, replays p's update.
    Returns (replay dict, seeds after the restatement's own update of pass p)."""
    lab, before = restatement.debug_iters(gray, depth, p, False)
    rep = replay(lab, before, depth, restatement.constants[0])
    _, after = restatement.debug_iters(gray, depth, p, True)
    return rep, after


def branch_counts(rep):
    """Seed counts per branch class of one replayed pass."""
    b, nd, k = rep["branch"], rep["nd"], rep["passes"]
    return {"skipped": int((b == SKIPPED).sum()),
            "nd == 0": int((b == NO_DEPTH).sum()),
            "1 <= nd < 8": int(((nd >= 1) & (nd < 8)).sum()),
            "nd % 8 != 0": int(((nd > 0) & (nd % 8 != 0)).sum()),
            "chain, 1 pass": int(((b == CHAIN) & (k == 1)).sum()),
            "chain, >= 2 passes": int(((b == CHAIN) & (k >= 2)).sum()),
            "queued at it == 0": int(((b == QUEUED) & (k == 0)).sum()),
            "queued at it >= 1": int(((b == QUEUED) & (k >= 1)).sum()),
            "queued at it >= 1, cut by the 5-pass cap": int(((b == QUEUED) & (k >= 1) & rep["capped"]).sum()),
            "re-entry into the chain": int(rep["reentry"].sum())}
