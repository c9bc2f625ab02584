"""Seeded frames that reach every branch of the Huber-Newton seed update's split between k_gather and k_newton_hard
(csrc/dsm_tile.cu), and the second phase of the plane solver k_gn_solve, shared by tests/test_seed_update_paths.py
(which proves the reach on the host with oracle/pyoracle_newton.py and oracle/pyoracle_planefit.py) and
tests/test_gpu_seed_update.py (which runs them through the kernels)."""
import numpy as np

from densesurfelmapping_b200 import synth

# Generator seeds found with the host replay: at 139 x 76 these inputs reach every branch (test_seed_update_paths.py
# states the counts); at other shapes they are just more frames of the same kind.
FAR_SEED = 9
CHECKER_SEED = 0
PLANE_SEED = 0


def cam_of(w, h):
    return synth.Camera(w, h, 0.8 * w, 0.8 * w, (w - 1) / 2.0, (h - 1) / 2.0, 0.5, 30.0)


def far_frame(w, h, seed=FAR_SEED, lo=3e5, hi=2e6, spread=0.8):
    """Depths of 3e5 - 2e6 m: each 8 x 8 block holds 2 or 3 levels within +-spread of its base depth, 5 % holes; each
    block has its own gray level (+-3).  At these depths the inverse-depth cost is negligible, so a seed's members are
    about its own block, and the rounding of the float mean (0.03 - 0.125 m steps) is large enough to make the Newton
    run several pure-chain passes, go out of range after an in-range pass, and come back into range."""
    rng = np.random.RandomState(seed)
    nby, nbx = (h + 7) // 8, (w + 7) // 8
    base = rng.uniform(lo, hi, (nby, nbx))
    nlev = rng.randint(2, 4, (nby, nbx))
    offs = rng.uniform(-spread, spread, (nby, nbx, 3))
    offs[nlev == 2, 2] = offs[nlev == 2, 0]
    by, bx = np.arange(h)[:, None] // 8, np.arange(w)[None, :] // 8
    pick = rng.randint(0, 3, (h, w))
    depth = (base[by, bx] + offs[by, bx, pick]).astype(np.float32)
    depth[rng.rand(h, w) < 0.05] = 0
    gray = rng.randint(0, 256, (nby, nbx))[by, bx] + rng.randint(-3, 4, (h, w))
    return np.clip(gray, 0, 255).astype(np.uint8), depth


def checker_frame(w, h, seed=CHECKER_SEED):
    """"Big" and "small" seeds on a checkerboard of the seed grid.  A small seed's centre pixel has its own gray level
    and no depth, so it keeps about that pixel alone and the big seeds own about 128 pixels each.  The depth alternates
    by column between 20 and 21 m (spread wider than 2 x the drive Huber range 0.4), so every big seed is hard from its
    first Newton pass, with a long list: the lists of a full 64-seed k_newton_hard CTA overflow its shared staging."""
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    big = ((xx // 8 + yy // 8) % 2) == 0
    gray = 200 + rng.randint(-2, 3, (h, w))
    depth = (20.0 + (xx % 2)).astype(np.float32) + rng.uniform(-0.05, 0.05, (h, w)).astype(np.float32)
    small_centre = (yy % 8 == 4) & (xx % 8 == 4) & ~big
    gray[small_centre] = 20
    depth[small_centre] = 0
    return np.clip(gray, 0, 255).astype(np.uint8), depth.astype(np.float32)


def scene_frame(cam, frame_id):
    """A frame of the synthetic drive (synth.make_frame), metres of a road scene."""
    return synth.make_frame(cam, frame_id, synth.pose_stream(frame_id % 3))


def plane_frame(w, h, seed=PLANE_SEED):
    """The checkerboard's big and small seeds on surfaces at about 5 m, one tilted plane per 8 x 8 block (slopes up to
    0.02 m per pixel in x and y, i.e. up to about 24 degrees at this focal length), whose pixels sit 0.2 - 0.4 m in front
    of or behind it (random per pixel).  Nearly every point of a big seed is an inlier of the plane fit and many
    first-pass residuals lie within 2e-3 of the Huber range: k_gn_solve must classify those seeds' points again (its
    phase B), and in the first 128-seed block of a 139 x 76 frame their point lists overflow its shared staging
    (GS_CAP).  The planes differ from block to block, so a seed fitted against another seed's points is far off."""
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    nby, nbx = (h + 7) // 8, (w + 7) // 8
    sx, sy = rng.uniform(-0.02, 0.02, (nby, nbx)), rng.uniform(-0.02, 0.02, (nby, nbx))
    by, bx = yy // 8, xx // 8
    surface = 5.0 + sx[by, bx] * (xx % 8 - 3.5) + sy[by, bx] * (yy % 8 - 3.5)
    lev = rng.uniform(0.2, 0.4, (h, w)) * rng.choice([-1.0, 1.0], (h, w))
    depth = (surface + lev).astype(np.float32)
    gray = 200 + rng.randint(-2, 3, (h, w))
    big = ((xx // 8 + yy // 8) % 2) == 0
    small_centre = (yy % 8 == 4) & (xx % 8 == 4) & ~big
    gray[small_centre] = 20
    depth[small_centre] = 0
    return np.clip(gray, 0, 255).astype(np.uint8), depth
