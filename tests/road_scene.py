"""DESIGN.md §8.20's synthetic road request for the planner GPU tests that run the ground chain on it: eight fused KITTI
frames, 256 views captured from shifted copies of their poses, and a known request at 0.2 m on a 64 x 20 x 128 grid."""
import numpy as np

from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from known_space import pose12

ROAD_VOXEL, ROAD_SHAPE, ROAD_CENTRE, ROAD_VIEWS = 0.2, (64, 20, 128), (0.0, 1.0, 12.8), 256


def road_request():
    """A context holding the road request, its field waited for; the caller enables its jobs.  Returns (ctx, state,
    origin)."""
    cam = synth.KITTI
    ctx = capi.Context(cam, max_batch=16, max_local_surfels=1 << 18)
    ctx.pool_upload(np.zeros(0, SURFEL_DTYPE))
    imgs = [synth.make_frame(cam, 5000 + t, synth.pose_stream(t)) for t in range(8)]
    ctx.fuse_stream_resident(list(range(8)), np.stack([g for g, _ in imgs]), np.stack([d for _, d in imgs]),
                             np.stack([synth.pose_stream(t) for t in range(8)]))
    ctx.field_enable(ROAD_VOXEL, *ROAD_SHAPE)
    ctx.views_enable(ROAD_VIEWS, 40.0)
    poses = []
    for j in range(ROAD_VIEWS):
        ctx.views_capture(j % 8, j)
        P = pose12(synth.pose_stream(j % 8))
        P[3] += 0.35 * (j // 8 % 8) - 1.2
        P[11] += 0.8 * (j // 64)
        poses.append(P)
    ctx.field_enqueue_known(ROAD_CENTRE, 1, list(range(ROAD_VIEWS)), np.array(poses))
    _, origin, _ = ctx.field_wait()
    state, _ = ctx.field_state()
    return ctx, state.copy(), origin.copy()
