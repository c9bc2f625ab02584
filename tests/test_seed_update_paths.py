"""CPU tests (-m "not gpu"): the host replay of the Huber-Newton seed update (oracle/pyoracle_newton.py) equals the
restatement bit for bit, and the committed inputs (tests/seed_update_inputs.py) provably reach every branch of the
CUDA schedule's split between k_gather and k_newton_hard, of the shared-memory fallbacks of k_newton_hard and
k_gn_solve, and of k_gn_solve's second phase (oracle/pyoracle_planefit.py).  tests/test_gpu_seed_update.py runs the
same inputs on the GPU, so together they show that each branch computes what the reference does."""
import numpy as np
import pytest

import pyoracle
import pyoracle_newton as pn
import pyoracle_planefit as pf
from densesurfelmapping_b200 import synth
from seed_update_inputs import cam_of, checker_frame, far_frame, plane_frame

# k_newton_hard (csrc/dsm_tile.cu): seeds per CTA and floats of shared list staging per CTA; each list is padded to 4
NW_T, NW_CAP = 64, 5632
# k_gn_solve: seeds per CTA, floats of shared point staging per CTA (three planes of each queued seed's centred points,
# each padded to 4), and the queueing test: a seed stays in phase A after its first step only while that step's bound
# (>= 1e-4) + 2e-3 is below its first-pass margin
GS_T, GS_CAP = 128, 9216
PHASE_B_MARGIN = 2e-3 - 1e-4  # 2e-4 below the certain threshold 2e-3 + 1e-4: room for the kernel's float margin


def inputs():
    """name -> (camera, constant set, gray, depth)."""
    kitti = synth.KITTI
    g, d = synth.make_frame(kitti, 0)
    small = cam_of(139, 76)
    return {"kitti_drive": (kitti, pyoracle.CONSTANTS_DRIVE, g, d),
            "kitti_rgbd": (kitti, pyoracle.CONSTANTS_RGBD, g, d),
            "far_139x76": (small, pyoracle.CONSTANTS_DRIVE) + far_frame(139, 76),
            "checker_139x76": (small, pyoracle.CONSTANTS_DRIVE) + checker_frame(139, 76)}


# Minimum seed counts per input, summed over the three passes (the observed counts are up to twice these)
REACH = {
    "kitti_drive": {"chain, 1 pass": 10000, "queued at it == 0": 3000, "nd == 0": 3, "1 <= nd < 8": 3,
                    "nd % 8 != 0": 10000, "skipped": 10},
    "kitti_rgbd": {"chain, 1 pass": 600, "queued at it == 0": 10000, "nd == 0": 3, "1 <= nd < 8": 3, "skipped": 10},
    "far_139x76": {"chain, 1 pass": 2, "chain, >= 2 passes": 25, "queued at it == 0": 150, "queued at it >= 1": 5,
                   "re-entry into the chain": 25, "nd % 8 != 0": 150, "skipped": 60},
    "checker_139x76": {"queued at it == 0": 100, "nd == 0": 20, "1 <= nd < 8": 20},
}

# The rare branches, in each pass (passes 1, 2, 3)
REACH_PER_PASS = {
    "far_139x76": {"chain, >= 2 passes": (12, 12, 2), "queued at it >= 1": (2, 2, 1), "re-entry into the chain": (10, 12, 3)},
}


@pytest.fixture(scope="module")
def replays():
    """name -> [(replay, restatement's seeds after the update)] for passes 1..3."""
    out = {}
    for name, (cam, consts, g, d) in inputs().items():
        o = pyoracle.Restatement(cam, consts)
        out[name] = [pn.replay_pass(o, g, d, p) for p in (1, 2, 3)]
    return out


def test_replay_equals_the_restatement(replays):
    """Every updated seed of every pass: the replay's mean_depth is the restatement's, bit for bit; stable seeds keep theirs."""
    for name, passes in replays.items():
        for p, (rep, after) in enumerate(passes, 1):
            bad = np.nonzero(rep["mean_depth"].view(np.uint32) != after["mean_depth"].view(np.uint32))[0]
            assert len(bad) == 0, (f"{name} pass {p}: mean_depth differs at {bad[:6]} ({pn.BRANCH_NAMES[int(rep['branch'][bad[0]])]}): "
                                   f"replay {rep['mean_depth'][bad[:6]]} restatement {after['mean_depth'][bad[:6]]}")
            assert (rep["branch"] != pn.SKIPPED).sum() > 0


@pytest.mark.parametrize("name", sorted(REACH))
def test_inputs_reach_every_branch(replays, name):
    """The committed inputs reach each branch of the update with at least the stated number of seeds."""
    tot = {}
    for p, (rep, _) in enumerate(replays[name], 1):
        c = pn.branch_counts(rep)
        print(f"{name} pass {p}: {c}")
        for k, v in c.items():
            tot[k] = tot.get(k, 0) + v
    for k, need in REACH[name].items():
        assert tot[k] >= need, f"{name}: {k}: {tot[k]} seeds < {need}"
    for p, (rep, _) in enumerate(replays[name], 1):
        c = pn.branch_counts(rep)
        for k, need in REACH_PER_PASS.get(name, {}).items():
            assert c[k] >= need[p - 1], f"{name} pass {p}: {k}: {c[k]} seeds < {need[p - 1]}"


def test_edge_tiles_with_dead_slots_are_updated(replays):
    """k_gather works on 8 x 4 seed tiles; where spw % 8 or sph % 4 is not 0 the last tile column / row has dead slots.
    The inputs have both, and seeds of those partial tiles are updated in every pass."""
    for name in ("kitti_drive", "far_139x76"):
        cam = inputs()[name][0]
        spw, sph = cam.width // 8, cam.height // 8
        assert spw % 8 != 0 and sph % 4 != 0, name
        sx, sy = np.arange(spw * sph) % spw, np.arange(spw * sph) // spw
        edge_x, edge_y = sx >= spw // 8 * 8, sy >= sph // 4 * 4
        for rep, _ in replays[name]:
            upd = rep["branch"] != pn.SKIPPED
            assert (upd & edge_x).sum() > 0 and (upd & edge_y).sum() > 0, name


def test_hard_seed_lists_overflow_the_newton_staging(replays):
    """k_newton_hard stages the lists of its 64 seeds in NW_CAP floats of shared memory; lists that do not fit are
    read from global memory.  In passes 1 and 2 of the checkerboard input that fallback is certain whatever the order
    of the hard-seed queue: there are at least 64 hard seeds, and even the 64 shortest padded lists need more than
    NW_CAP floats, so every full CTA overflows."""
    for p, (rep, _) in enumerate(replays["checker_139x76"][:2], 1):
        nd = np.sort(rep["nd"][rep["branch"] == pn.QUEUED])
        assert len(nd) >= NW_T, f"pass {p}: {len(nd)} hard seeds"
        need = int(((nd[:NW_T] + 3) & ~3).sum())
        print(f"checker pass {p}: {len(nd)} hard seeds, the 64 shortest lists need {need} floats > {NW_CAP}")
        assert need > NW_CAP


def test_plane_solver_second_phase_and_its_staging_overflow_are_reached():
    """k_gn_solve queues a seed for its phase B (a pass over the points again) when its first-pass margin leaves no room
    for a step; the plane input has many seeds whose host margin is below 2e-3 - 1e-4, which makes that certain.  In the
    first 128-seed block the certainly-queued seeds alone need more than GS_CAP floats of point staging, so a seed of
    that block reads its points from global memory whatever the order of the block's queue."""
    cam = cam_of(139, 76)
    g, d = plane_frame(139, 76)
    o = pyoracle.Restatement(cam)
    o.superpixels(g, d)
    normals = o.norm_map()
    lab, seeds = o.debug_iters(g, d, 3, True)  # the state the plane fit starts from
    fp = pf.first_pass(cam, lab, seeds, d, normals, pyoracle.CONSTANTS_DRIVE[0])
    queued = fp["fitted"] & (fp["margin"] < PHASE_B_MARGIN)
    use = np.where(queued, 3 * ((fp["n"] + 3) & ~3), 0)
    blocks = [int(use[i:i + GS_T].sum()) for i in range(0, len(use), GS_T)]
    print(f"plane_139x76: {int(fp['fitted'].sum())} fitted seeds, {int(queued.sum())} certainly queued, "
          f"staging per 128-seed block {blocks} (GS_CAP {GS_CAP})")
    assert queued.sum() >= 30
    assert blocks[0] > GS_CAP + 2000
