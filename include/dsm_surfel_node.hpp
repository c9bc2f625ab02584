// dsm_surfel_node.hpp — header-only dsm::SurfelMapNode: the reference's whole SurfelMap node (surfel_fusion/src/
// surfel_map.cpp) with the map resident on the GPU, callback for callback, built on the C ABI of dsm.h and the map
// operations of dsm_surfel_map.hpp.  Like dsm_surfel_map.hpp it needs neither ROS, Eigen, OpenCV nor PCL: poses are 7
// doubles in geometry_msgs::Pose order {px, py, pz, qx, qy, qz, qw}, images are a pointer and a row pitch, clouds are
// vectors of dsm_point_t.  A ROS node on top of it is topic glue only (INTEGRATION.md §4).
//
//   SurfelMap member (surfel_map.cpp)                     here
//   ---------------------------------------------------   ---------------------------------------------------------
//   ctor (:14-29, :53)                                    SurfelMapNode(width, ..., drift_free_poses, device, ...)
//   orb_results_input (:205-365)                          orb_results_input(stamp, loop pairs, path, pose, kf, ref)
//   image_input / depth_input (:83-101)                   image_input(stamp, gray, pitch) / depth_input(...)
//   synchronize_msgs (:103-163) + move_add_surfels        one dsm_fuse_stream_window call per fused frame (n = 1)
//     + fuse_map
//   warp_surfels (:681-824)                               dsm_pool_transform + dsm_inactive_transform per moved pose
//   get_driftfree_poses / get_add_remove_poses            driftfree_poses(root, range) / window_lists(root, ...)
//   publish_active/inactive/all/neighbor/raw_pointcloud   active_points / inactive_points / all_points /
//                                                         neighbor_points(reference_index) / raw_points
//   publish_pose_graph / publish_camera_position          pose_graph()
//   save_map / save_mesh / save_cloud (:75-81, :1153-1280) save_map / save_mesh / save_cloud
//
// Pose arithmetic: every fp64 step of the node (pose_ros2eigen, pose_eigen2ros, 4x4 products, inverse, cast to float)
// is restated operation for operation from the Eigen stand-in the repository's reference build uses (DESIGN.md §1.1:
// Quaterniond(Matrix3d) by the trace / largest-diagonal branches, toRotationMatrix, products accumulated left to right
// over the inner index, inverse as adjugate over determinant).  Compiled without floating-point contraction
// (-ffp-contract=off, or any x86-64 build without -mfma), fuse poses, warp matrices and the stored poses equal that
// build bit for bit; against real Eigen they agree to about 1e-7.
//
// The loop-closure warp follows the schedule of that build: the active warp W = (T_loop * T_cam^-1).cast<float>() of
// the first local pose is taken before any cam_pose is overwritten and applied to the pool; then every pose whose
// position moved gets its own W_i on the inactive store (a pose in the drift-free window has nothing stored and is
// skipped) and takes cam_pose = loop_pose.
//
// Deviations from the reference, each deliberate:
//   * inactive_points / all_points / save_cloud hold every stored point of a warped pose warped; the reference's
//     inactive_pointcloud keeps the last point of each warped slice stale (std::copy(&front, &back), :742).
//   * synchronize_msgs spins forever when the oldest image or depth is newer than the oldest pose (:114-139 have no
//     `>` branch); here that pose is dropped without a fuse and the next one is tried.
//   * Input the reference would index out of bounds with (a reference index or loop pair outside the pose database,
//     a loop path that is empty while poses exist) is rejected with DSM_E_INVALID, or skipped for the empty path.
//   * A frame that does not fit the pool or the inactive store is not applied (nor any later one); DSM_E_CAPACITY
//     comes back from the next call that reads the map, as dsm_fuse_stream_window specifies.
//
// A fused frame never waits for the GPU: the callbacks only enqueue.  The readers (clouds, save_*) synchronise.
//
// Publishing after every frame, as synchronize_msgs does (:191-198), through those readers costs several round trips
// and a copy of the whole inactive cloud per frame.  enable_publishing() makes every fused frame enqueue a snapshot of
// the active and the inactive cloud right behind its fuse (dsm_publish_enqueue(ctx, 5)), and published_clouds() hands
// out the snapshot of the latest fused frame: called right after the depth callback it waits for that frame alone;
// called at the start of the next frame's callback it finds the snapshot finished and waits for nothing, one frame
// late.  The clouds are the library's pinned buffers, valid until the next frame is fused; the inactive cloud below
// inactive_changed_from is bit-identical to the one handed out before, so a long-lived copy needs only its tail
// rewritten.  One snapshot can be in flight: a frame fused while the previous snapshot is unread first waits for that
// snapshot and drops it (a pose callback may have enqueued loop-closure warps in between, so it cannot be reused).
// published_clouds() never clears a capacity error: after a frame that did not fit, it and every later call return
// DSM_E_CAPACITY with the clouds of the last applied frame, and no later frame is applied, until a synchronising reader
// (local_surfels(), active_points(), ... or dsm_pool_size on context()) has reported and cleared the error.  A node
// that only ever publishes must call one of them to resume.
// Without enable_publishing() nothing is enqueued and the node behaves exactly as before.
//
// A planner wants a distance field, not clouds.  enable_distance_field(voxel, nx, ny, nz) makes every fused frame
// enqueue one more job behind its fuse (and behind its snapshot when publishing): the exact Euclidean distance field of
// the map on an nx x ny x nz grid centred on the frame's camera, the translation of its fuse pose, with the active
// cloud's threshold of 5 updates (dsm_field_enqueue(ctx, centre, 5), DESIGN.md §8.7).  distance_field() hands it out
// with the same one-frame-late pattern, lifetime and capacity rule as published_clouds(); an unread field is retired
// before the next fuse and before load_state*, as an unread snapshot is.  Without enable_distance_field() nothing is
// enqueued.  enable_distance_field(..., false) keeps every field on the device (dsm_field_enqueue_resident):
// distance_field() then hands out dist == nullptr with the origin and the count, and the planner asks the field what it
// needs instead (DESIGN.md §8.8): after enable_field_queries(), field_samples() (distance and gradient at points) and
// trajectory_clearance() (the clearance of candidate paths) read the field of the latest fused frame, one enqueue and
// one wait each, without touching the one-frame-late distance_field() handout.
// enable_signed_distance(), after enable_distance_field, makes every field also build the signed grid (DESIGN.md §8.16):
// negative inside obstacles (and, with known space, inside unknown space), so that a gradient points out of them.
// signed_distance_field() hands out the signed grid of the field distance_field() handed out last, and field_samples()
// and trajectory_clearance() read it with signed_field = true.
// The field counts every voxel without an obstacle point as free, seen or not.  enable_known_space(max_views, max_range),
// after enable_distance_field, makes it measure the distance to anything not known to be free (DESIGN.md §8.9): the
// first fused frame of each new reference keyframe is captured into slot captures % max_views (its superpixel rays, in
// camera coordinates) and the node keeps (reference_index, relative) per slot; every field request then carries every
// filled slot at its current world pose cam_pose[ref] * relative, in fuse_pose's arithmetic, so a loop closure moves the
// views with the map.  known_space() returns the state grid of the field distance_field() handed out last.  Without
// enable_view_checkpoints() views are not part of a checkpoint: load_state* empties the slot table, which refills as
// keyframes are fused.  enable_view_checkpoints(), after enable_known_space, makes every save_state* carry the views
// (the library's rays, DESIGN.md §8.18, and the node's slot table in its section) and load_state* restore them, so a
// resumed node carves the same free space as one that never stopped.
// An exploring planner asks where to look next.  enable_frontiers(max_clusters, max_voxels), after enable_known_space,
// lets frontiers() find the exploration frontiers of the latest fused frame's known field on the device (DESIGN.md
// §8.10): the clusters of free voxels that border unknown space, their statistics and member voxels, one enqueue and one
// wait, without touching the one-frame-late distance_field() handout.
// Which frontier is worth the trip?  enable_reach(max_targets, max_path_voxels, max_rounds), after enable_known_space,
// lets reach() find paths through the known free space of the latest fused frame's field on the device (DESIGN.md
// §8.11): the travel cost from a start point to goal points and, after a frontiers() call on that frame, to every
// frontier cluster, with each target's viewpoint and path, one enqueue and one wait.
// In which order should the viewpoints be visited?  enable_reach_matrix(max_sites, max_tiles, max_rounds), after
// enable_known_space, lets reach_matrix() price an exploration tour on the device (DESIGN.md §8.13): the travel costs
// between every pair of up to max_sites points through the known free space of the latest fused frame's field, one
// enqueue and one wait.  A planner chains frontiers(), then reach(with_frontiers) from the robot for each cluster's
// viewpoint, then reach_matrix over the robot's position and those viewpoints, and hands the matrix to its tour solver:
// enable_tour(max_sites, max_starts) lets tour() order the sites on the device (DESIGN.md §8.14), a deterministic
// multi-start local search over the matrix as it stands, one enqueue and one wait; it reads no field, so it needs
// neither known space nor a fused frame.
// What would the robot see from there?  enable_view_gain(max_views), after enable_known_space, lets view_gain() score
// candidate camera poses against the latest fused frame's known field on the device (DESIGN.md §8.12): per pose, with
// the node's own intrinsics, the frustum voxels and the free, unknown, occupied, frontier and (after a frontiers() call
// on that frame) cluster voxels it would see, one enqueue and one wait.
// Where should the camera look along the way?  enable_headings(max_trajectories, max_samples), after
// enable_known_space, lets headings() plan the camera's heading along trajectories on the device (DESIGN.md §8.19): the
// unknown and frontier voxels seen at every sample and rotation, then the best rate-limited rotation sequence per
// trajectory, one enqueue and one wait.
// Where can a ground robot drive?  enable_terrain(up), after enable_known_space, lets terrain() find the supporting
// surface of every column of the latest fused frame's known field along the up axis on the device (DESIGN.md §8.20):
// its level, the step to its neighbours, whether it is traversable and the clearance to the nearest cell that is not,
// one enqueue and one wait.  A ground planner's exploration chain runs on that plane: terrain(), then frontiers(), then
// reach_terrain(with_frontiers) from the robot (DESIGN.md §8.21), then viewpoints_terrain(with_reach) for the cells whose
// camera, eye voxels above the ground, would see each cluster best (§8.23), then reach_matrix_terrain over the robot's
// position and those cameras (§8.22), then tour() on that matrix.
// device < 0 builds the node without a context: the callbacks run the whole pose logic (pose database, sync, window
// bookkeeping) and fuse nothing; any call that reads the map returns DSM_E_STATE.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstring>
#include <deque>
#include <set>
#include <string>
#include <utility>
#include <vector>
#include "dsm_surfel_map.hpp"

namespace dsm
{
// geometry_msgs::Pose: position, then orientation x, y, z, w
struct Pose
{
    double x, y, z, qx, qy, qz, qw;
};
struct Point3
{
    double x, y, z;
};

namespace node_math
{
// a column-major 4x4 fp64 matrix (Eigen::Matrix4d memory order)
struct M4
{
    double d[16];
    double &operator()(int i, int j) { return d[j * 4 + i]; }
    double operator()(int i, int j) const { return d[j * 4 + i]; }
};
inline M4 identity()
{
    M4 m;
    for (int i = 0; i < 16; i++) m.d[i] = (i % 5 == 0) ? 1.0 : 0.0;
    return m;
}
inline M4 mul(const M4 &a, const M4 &b)
{
    M4 r;
    for (int k = 0; k < 4; k++)
        for (int i = 0; i < 4; i++)
        {
            double acc = a(i, 0) * b(0, k);
            for (int j = 1; j < 4; j++) acc = acc + a(i, j) * b(j, k);
            r(i, k) = acc;
        }
    return r;
}
inline M4 inverse(const M4 &a)
{
    const double *m = a.d;
    double v[16];
    v[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
    v[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
    v[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
    v[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
    v[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
    v[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
    v[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
    v[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
    v[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
    v[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
    v[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
    v[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
    v[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
    v[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
    v[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
    v[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
    const double det = m[0] * v[0] + m[1] * v[4] + m[2] * v[8] + m[3] * v[12];
    const double inv_det = 1.0 / det;
    M4 out;
    for (int i = 0; i < 16; i++) out.d[i] = v[i] * inv_det;
    return out;
}
// pose_ros2eigen (surfel_map.cpp:367-379): T = I, T.block<3,3>(0,0) = Quaterniond(w, x, y, z).toRotationMatrix(), T(:3,3) = p
inline M4 from_pose(const Pose &p)
{
    M4 r = identity();
    const double tx = 2.0 * p.qx, ty = 2.0 * p.qy, tz = 2.0 * p.qz;
    const double twx = tx * p.qw, twy = ty * p.qw, twz = tz * p.qw;
    const double txx = tx * p.qx, txy = ty * p.qx, txz = tz * p.qx;
    const double tyy = ty * p.qy, tyz = tz * p.qy, tzz = tz * p.qz;
    r(0, 0) = 1.0 - (tyy + tzz), r(0, 1) = txy - twz, r(0, 2) = txz + twy;
    r(1, 0) = txy + twz, r(1, 1) = 1.0 - (txx + tzz), r(1, 2) = tyz - twx;
    r(2, 0) = txz - twy, r(2, 1) = tyz + twx, r(2, 2) = 1.0 - (txx + tyy);
    r(0, 3) = p.x, r(1, 3) = p.y, r(2, 3) = p.z;
    return r;
}
// pose_eigen2ros (surfel_map.cpp:381-391): Quaterniond(T.block<3,3>(0,0)) and T(:3,3)
inline Pose to_pose(const M4 &m)
{
    Pose p;
    double q[3], qw;
    double t = m(0, 0) + m(1, 1) + m(2, 2);
    if (t > 0.0)
    {
        t = std::sqrt(t + 1.0);
        qw = 0.5 * t;
        t = 0.5 / t;
        q[0] = (m(2, 1) - m(1, 2)) * t;
        q[1] = (m(0, 2) - m(2, 0)) * t;
        q[2] = (m(1, 0) - m(0, 1)) * t;
    }
    else
    {
        int i = 0;
        if (m(1, 1) > m(0, 0)) i = 1;
        if (m(2, 2) > m(i, i)) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        t = std::sqrt(m(i, i) - m(j, j) - m(k, k) + 1.0);
        q[i] = 0.5 * t;
        t = 0.5 / t;
        qw = (m(k, j) - m(j, k)) * t;
        q[j] = (m(j, i) + m(i, j)) * t;
        q[k] = (m(k, i) + m(i, k)) * t;
    }
    p.qx = q[0], p.qy = q[1], p.qz = q[2], p.qw = qw;
    p.x = m(0, 3), p.y = m(1, 3), p.z = m(2, 3);
    return p;
}
// Matrix4d::cast<float>(), column-major
inline void to_float(const M4 &m, float out[16])
{
    for (int i = 0; i < 16; i++) out[i] = (float)m.d[i];
}
inline Pose read_pose(const double *p7)
{
    Pose p;
    p.x = p7[0], p.y = p7[1], p.z = p7[2], p.qx = p7[3], p.qy = p7[4], p.qz = p7[5], p.qw = p7[6];
    return p;
}
inline bool same_position(const Pose &a, const Pose &b) { return a.x == b.x && a.y == b.y && a.z == b.z; }
} // namespace node_math

// PoseElement (surfel_map.h): what the node keeps per keyframe; the attached surfels live in the device store
struct NodePose
{
    Pose cam_pose, loop_pose;
    double cam_stamp;
    std::vector<int> linked_pose_index;
};

// one transform issued by a loop closure: pose -1 is the active pool, else the keyframe whose stored surfels moved
struct NodeWarp
{
    int pose;
    float W[16];
};

// publish_pose_graph / publish_camera_position (surfel_map.cpp:906-1026) of the last fused frame
struct NodePoseGraph
{
    std::vector<Pose> path;         // fusion_loop_path: every cam_pose, index order
    std::vector<Point3> loop_edges; // loop_marker: loop_pose positions, two per non-consecutive link j > i
    std::vector<Point3> driftfree;  // driftfree_loop_path, "driftfree": cam_pose positions of get_driftfree_poses(ref)
    std::vector<Point3> drift;      // "drift": every other pose, index order
    Pose camera;                    // camera_marker: the fuse pose
};

class SurfelMapNode
{
  public:
    // The surfel_map.cpp:14-29 parameters (cam_*, fuse_far_distence, fuse_near_distence, drift_free_poses); the CUDA
    // device (< 0: pose logic only, no context), the pool capacity, the inactive-store reservation in surfels and
    // optionally a constant set (DSM_CONSTANTS_DRIVE when null).  Check last_error() after construction.
    SurfelMapNode(int cam_width, int cam_height, double cam_fx, double cam_fy, double cam_cx, double cam_cy, double far_dist,
                  double near_dist, int drift_free_poses, int device = 0, int max_local_surfels = 1 << 21,
                  int max_inactive_surfels = 1 << 22, const dsm_constants *constants = nullptr)
        : ctx_("dsm::SurfelMapNode"), width_(cam_width), height_(cam_height), drift_free_poses_(drift_free_poses), last_ref_(-1),
          fused_(false)
    {
        const double cam[6] = {cam_fx, cam_fy, cam_cx, cam_cy, far_dist, near_dist};
        std::memcpy(cam_, cam, sizeof(cam_));
        std::memset(transform_kitti_.d, 0, sizeof(transform_kitti_.d));
        std::memset(&last_fuse_pose_, 0, sizeof(last_fuse_pose_));
        if (device < 0) return;
        // two frame slots: the copy of frame t+1 overlaps the kernels of frame t
        const dsm_params p = detail::Context::params(cam_width, cam_height, (float)cam_fx, (float)cam_fy, (float)cam_cx, (float)cam_cy,
                                                     (float)far_dist, (float)near_dist, 2, max_local_surfels);
        ctx_.open("SurfelMapNode", p, device, true, &max_inactive_surfels, constants);
    }

    // ---- the three callbacks of ros_node.cpp ----

    // orb_results_input (surfel_map.cpp:205-365).  loop_pairs: n_loops pairs of keyframe indices (the loop_stamps
    // channel); loop_path7: n_path poses of 7 doubles (the loop path, ORB's frame); this_pose7: the frame's pose;
    // is_keyframe / reference_index: pose.covariance[0] > 0 / pose.covariance[1].  Queues the frame and runs the sync.
    int orb_results_input(double stamp, const int *loop_pairs, int n_loops, const double *loop_path7, int n_path, const double *this_pose7,
                          bool is_keyframe, int reference_index)
    {
        using namespace node_math;
        const int n_poses = (int)poses_.size();
        if (!this_pose7 || n_loops < 0 || n_path < 0 || (n_loops && !loop_pairs) || (n_path && !loop_path7)) return ctx_.done(DSM_E_INVALID, "orb_results_input");
        const bool new_kf = is_keyframe || n_poses == 0;
        // a new keyframe links to its reference, which must exist already; any other frame refers to an existing pose
        const int n_after = n_poses + (new_kf ? 1 : 0);
        if (reference_index < 0 || reference_index >= (new_kf && n_poses > 0 ? n_poses : n_after)) return ctx_.done(DSM_E_INVALID, "orb_results_input");
        for (int i = 0; i < 2 * n_loops; i++)
            if (loop_pairs[i] < 0) return ctx_.done(DSM_E_INVALID, "orb_results_input");

        last_warp_.clear();
        // the KITTI axis fix-up, fixed by the first pose (:214-232)
        const M4 received = from_pose(read_pose(this_pose7));
        if (n_poses == 0)
        {
            M4 idea;
            std::memset(idea.d, 0, sizeof(idea.d));
            idea(0, 0) = 1.0, idea(1, 2) = 1.0, idea(2, 1) = -1.0, idea(3, 3) = 1.0;
            transform_kitti_ = mul(idea, inverse(received));
        }
        const Pose input_pose = to_pose(mul(transform_kitti_, received));

        // loop_pose of every pose the path covers (:237-253)
        bool loop_changed = false;
        for (int i = 0; i < n_poses && i < n_path; i++)
        {
            poses_[i].loop_pose = to_pose(mul(transform_kitti_, from_pose(read_pose(loop_path7 + 7 * i))));
            if (!same_position(poses_[i].loop_pose, poses_[i].cam_pose)) loop_changed = true;
        }
        // the last correction carried to the poses the path does not cover yet (:255-272); an empty path has no last
        // correction (the reference reads pose -1)
        if (n_poses > n_path && n_path > 0)
        {
            const int last = n_path - 1;
            const M4 warp = mul(from_pose(poses_[last].loop_pose), inverse(from_pose(poses_[last].cam_pose)));
            for (int i = n_path; i < n_poses; i++) poses_[i].loop_pose = to_pose(mul(warp, from_pose(poses_[i].cam_pose)));
        }
        if (loop_changed) warp_surfels();

        // covisibility links without duplicates (:290-316)
        for (int i = 0; i < n_loops; i++)
        {
            const int a = loop_pairs[2 * i], b = loop_pairs[2 * i + 1];
            if (a >= n_poses || b >= n_poses) continue;
            std::vector<int> &la = poses_[a].linked_pose_index, &lb = poses_[b].linked_pose_index;
            if (std::find(la.begin(), la.end(), b) != la.end()) continue;
            la.push_back(b);
            if (std::find(lb.begin(), lb.end(), a) == lb.end()) lb.push_back(a);
        }

        // a new keyframe (:319-353)
        if (new_kf)
        {
            NodePose e;
            const int index = n_poses;
            e.cam_pose = input_pose, e.loop_pose = input_pose, e.cam_stamp = stamp;
            if (n_poses > 0)
            {
                e.linked_pose_index.push_back(reference_index);
                poses_[reference_index].linked_pose_index.push_back(index);
            }
            poses_.push_back(e);
            local_.insert(index);
        }

        // the pose relative to its reference, after its round trip through geometry_msgs::Pose (:356-363)
        PendingPose q;
        q.stamp = stamp;
        q.reference_index = reference_index;
        q.relative = to_pose(mul(inverse(from_pose(poses_[reference_index].cam_pose)), from_pose(input_pose)));
        pose_buffer_.push_back(q);
        return synchronize();
    }

    // image_input / depth_input (surfel_map.cpp:83-101): the frame is copied (row pitch in bytes), then the sync runs
    int image_input(double stamp, const uint8_t *gray, size_t pitch)
    {
        if (!gray || pitch < (size_t)width_) return ctx_.done(DSM_E_INVALID, "image_input");
        image_buffer_.push_back(std::make_pair(stamp, std::vector<uint8_t>((size_t)width_ * height_)));
        for (int y = 0; y < height_; y++) std::memcpy(&image_buffer_.back().second[(size_t)y * width_], gray + (size_t)y * pitch, (size_t)width_);
        return synchronize();
    }
    int depth_input(double stamp, const float *depth, size_t pitch)
    {
        if (!depth || pitch < (size_t)width_ * 4) return ctx_.done(DSM_E_INVALID, "depth_input");
        depth_buffer_.push_back(std::make_pair(stamp, std::vector<float>((size_t)width_ * height_)));
        const uint8_t *src = reinterpret_cast<const uint8_t *>(depth);
        for (int y = 0; y < height_; y++)
            std::memcpy(&depth_buffer_.back().second[(size_t)y * width_], src + (size_t)y * pitch, (size_t)width_ * 4);
        return synchronize();
    }

    // ---- the pose graph ----
    const std::vector<NodePose> &poses() const { return poses_; }
    const std::set<int> &local_surfels_indexs() const { return local_; }
    // get_driftfree_poses (surfel_map.cpp:1643-1674): breadth-first over the links, `range` levels including the root
    std::vector<int> driftfree_poses(int root_index, int range) const
    {
        std::vector<int> out;
        if (root_index < 0 || (int)poses_.size() < root_index + 1) return out;
        std::vector<int> this_level(1, root_index), next_level;
        out.push_back(root_index);
        for (int i = 1; i < range; i++)
        {
            for (size_t a = 0; a < this_level.size(); a++)
            {
                const std::vector<int> &links = poses_[(size_t)this_level[a]].linked_pose_index;
                for (size_t b = 0; b < links.size(); b++)
                    if (std::find(out.begin(), out.end(), links[b]) == out.end())
                    {
                        next_level.push_back(links[b]);
                        out.push_back(links[b]);
                    }
            }
            this_level.swap(next_level);
            next_level.clear();
        }
        return out;
    }
    // get_add_remove_poses (surfel_map.cpp:1597-1641): the lists move_add_surfels(root) would use now
    void window_lists(int root_index, std::vector<int> &poses_to_remove, std::vector<int> &poses_to_add) const
    {
        const std::vector<int> df = driftfree_poses(root_index, drift_free_poses_);
        poses_to_add.clear(), poses_to_remove.clear();
        for (size_t i = 0; i < df.size(); i++)
            if (!local_.count(df[i])) poses_to_add.push_back(df[i]);
        for (std::set<int>::const_iterator it = local_.begin(); it != local_.end(); ++it)
            if (std::find(df.begin(), df.end(), *it) == df.end()) poses_to_remove.push_back(*it);
    }
    // the oldest queued frame that has not been fused: its reference index (returned, -1 when none), the pose
    // fuse_map will receive (column-major float) and its window lists, all as of now
    int pending_frame(float pose16[16], std::vector<int> &poses_to_remove, std::vector<int> &poses_to_add) const
    {
        if (pose_buffer_.empty()) return -1;
        const PendingPose &q = pose_buffer_.front();
        node_math::to_float(fuse_pose(q), pose16);
        window_lists(q.reference_index, poses_to_remove, poses_to_add);
        return q.reference_index;
    }
    // the transforms the last orb_results_input issued, the active pool first (pose -1); empty when its path moved no pose
    const std::vector<NodeWarp> &last_warp() const { return last_warp_; }
    NodePoseGraph pose_graph() const
    {
        NodePoseGraph g;
        for (size_t i = 0; i < poses_.size(); i++)
        {
            g.path.push_back(poses_[i].cam_pose);
            const std::vector<int> &l = poses_[i].linked_pose_index;
            for (size_t j = 0; j < l.size(); j++)
                if (l[j] != (int)i - 1 && l[j] != (int)i + 1 && l[j] > (int)i)
                {
                    g.loop_edges.push_back(position(poses_[i].loop_pose));
                    g.loop_edges.push_back(position(poses_[(size_t)l[j]].loop_pose));
                }
        }
        const std::vector<int> df = driftfree_poses(last_ref_, drift_free_poses_);
        for (size_t i = 0; i < df.size(); i++) g.driftfree.push_back(position(poses_[(size_t)df[i]].cam_pose));
        for (size_t i = 0; i < poses_.size(); i++)
            if (std::find(df.begin(), df.end(), (int)i) == df.end()) g.drift.push_back(position(poses_[i].cam_pose));
        g.camera = last_fuse_pose_;
        return g;
    }

    // ---- the clouds the node publishes; each replaces `points` ----
    // publish_active_pointcloud (:1398-1417): local surfels with update_times >= 5, pool order
    int active_points(std::vector<dsm_point_t> &points)
    {
        points.clear();
        return ctx_.run("active_points", [&] { return detail::pool_cloud(ctx_, 5, points); });
    }
    // publish_inactive_pointcloud (:1385-1396): the inactive store, store order, every warped point warped
    int inactive_points(std::vector<dsm_point_t> &points)
    {
        points.clear();
        return ctx_.run("inactive_points", [&] { return detail::inactive_cloud(ctx_, points); });
    }
    // publish_all_pointcloud (:1419-1454)
    int all_points(std::vector<dsm_point_t> &points)
    {
        points.clear();
        if (!ctx_.ready("all_points")) return ctx_.err;
        int rc = detail::pool_cloud(ctx_, 5, points);
        if (rc == DSM_OK) rc = detail::inactive_cloud(ctx_, points);
        return ctx_.done(rc, "all_points");
    }
    // ---- the active and inactive clouds of every fused frame, from inside the stream (see the top of this file) ----
    int enable_publishing()
    {
        if (ctx_.run("enable_publishing", [&] { return dsm_publish_enable(ctx_.ctx); }) == DSM_OK) publishing_ = true;
        return ctx_.err;
    }
    // active_points() and inactive_points() as they were right after the latest fused frame; DSM_E_STATE when no frame
    // has been fused since the last call.  A map whose latest frame did not fit returns DSM_E_CAPACITY with the clouds
    // of the last applied frame.
    int published_clouds(const dsm_point_t *&active, int &n_active, const dsm_point_t *&inactive, int &n_inactive, int &inactive_changed_from)
    {
        if (!ctx_.ready("published_clouds")) return ctx_.err;
        if (!snapshot_) return ctx_.done(DSM_E_STATE, "published_clouds");
        snapshot_ = false;
        return ctx_.done(dsm_publish_wait(ctx_.ctx, &active, &n_active, &inactive, &n_inactive, &inactive_changed_from), "published_clouds");
    }
    // ---- the map as a distance field around the camera, for a planner (see the top of this file, DESIGN.md §8.7) ----
    // host_copy = false: the grid stays on the device; distance_field() hands out dist == nullptr
    int enable_distance_field(float voxel, int nx, int ny, int nz, bool host_copy = true)
    {
        const dsm_field_params p = {voxel, nx, ny, nz};
        if (ctx_.run("enable_distance_field", [&] { return dsm_field_enable(ctx_.ctx, &p); }) == DSM_OK)
            distance_field_ = true, field_host_copy_ = host_copy;
        return ctx_.err;
    }
    // ---- the signed distance field (DESIGN.md §8.16) ----
    // once, after enable_distance_field: every field from then on also builds the signed grid (negative depth inside
    // obstacles, and inside unknown space with known space)
    int enable_signed_distance()
    {
        return ctx_.run("enable_signed_distance", [&] { return dsm_field_signed_enable(ctx_.ctx); });
    }
    // the signed grid [nz][ny][nx] in metres of the field distance_field() handed out last (the library's pinned buffer,
    // valid until the next frame is fused; nullptr for a field kept on the device).  DSM_E_STATE without
    // enable_signed_distance() before that field, or before distance_field() has handed out a field.
    int signed_distance_field(const float *&sdist)
    {
        if (!ctx_.ready("signed_distance_field")) return ctx_.err;
        return ctx_.done(dsm_field_signed(ctx_.ctx, &sdist), "signed_distance_field");
    }
    // ---- free versus unknown space (see the top of this file, DESIGN.md §8.9) ----
    // once, after enable_distance_field: max_views capture slots, rays cut to max_range metres
    int enable_known_space(int max_views, float max_range)
    {
        if (ctx_.run("enable_known_space", [&] { return dsm_views_enable(ctx_.ctx, max_views, max_range); }) == DSM_OK)
        {
            known_.assign((size_t)max_views, KnownView{-1, Pose()});
            known_range_ = max_range;
        }
        return ctx_.err;
    }
    // once, after enable_known_space (DSM_E_STATE before it): every checkpoint from now on carries the captured views and
    // the slot table (node section version 2), and every load restores them (DESIGN.md §8.18).  A version-1 section
    // still loads, with an empty table; a node without this call refuses a version-2 section with DSM_E_INVALID.
    int enable_view_checkpoints()
    {
        if (known_.empty()) return ctx_.done(DSM_E_STATE, "enable_view_checkpoints");
        if (ctx_.run("enable_view_checkpoints", [&] { return dsm_checkpoint_views_enable(ctx_.ctx); }) == DSM_OK) view_checkpoints_ = true;
        return ctx_.err;
    }
    // the state grid [nz][ny][nx] (0 unknown, 1 occupied, 2 free; the library's pinned buffer, valid until the next frame
    // is fused; nullptr for a field kept on the device) and the free voxels of the field distance_field() handed out last.
    // DSM_E_STATE without known space or before distance_field() has handed out a field.
    int known_space(const uint8_t *&state, int &n_free)
    {
        if (!ctx_.ready("known_space")) return ctx_.err;
        return ctx_.done(dsm_field_state(ctx_.ctx, &state, &n_free), "known_space");
    }
    // the views a field request would carry now: the filled slots, ascending, and their world poses (12 doubles each,
    // row-major [R | t], camera to world); and the number of captures so far (the latest went to slot
    // (captures - 1) % max_views)
    int known_views(std::vector<int32_t> &slots, std::vector<double> &poses) const
    {
        slots.clear(), poses.clear();
        for (size_t i = 0; i < known_.size(); i++)
        {
            if (known_[i].ref < 0) continue;
            const node_math::M4 m = node_math::mul(node_math::from_pose(poses_[(size_t)known_[i].ref].cam_pose), node_math::from_pose(known_[i].relative));
            slots.push_back((int32_t)i);
            for (int r = 0; r < 3; r++)
                for (int c = 0; c < 4; c++) poses.push_back(m(r, c));
        }
        return captures_;
    }

    // ---- exploration frontiers of the latest fused frame's known field (DESIGN.md §8.10) ----
    // once, after enable_known_space: the capacities of the cluster table and the voxel list
    int enable_frontiers(int max_clusters, int max_voxels)
    {
        if (ctx_.run("enable_frontiers", [&] { return dsm_frontier_enable(ctx_.ctx, max_clusters, max_voxels); }) == DSM_OK)
            frontier_clusters_ = max_clusters;
        return ctx_.err;
    }
    // the clusters of at least min_voxels frontier voxels (include/dsm.h), the voxel list and the counts of the latest
    // fused frame's known field; clusters receives min(n_clusters, max_clusters) records and voxels n_listed indices.
    // DSM_E_STATE without known space, before any field, and after load_state* until the next fused frame;
    // DSM_E_CAPACITY with the frontiers of the last applied frame's field, as distance_field().
    int frontiers(int min_voxels, std::vector<dsm_frontier_cluster_t> &clusters, std::vector<int32_t> &voxels, dsm_frontier_counts_t &counts)
    {
        clusters.clear();
        voxels.clear();
        counts = dsm_frontier_counts_t();
        const dsm_frontier_cluster_t *c = nullptr;
        const int32_t *v = nullptr;
        return job("frontiers", KNOWN_FIELD, true, [&] { return dsm_frontier_enqueue(ctx_.ctx, min_voxels); },
                   [&] { return dsm_frontier_wait(ctx_.ctx, &c, &v, &counts); },
                   [&] {
                       clusters.assign(c, c + std::min(counts.n_clusters, frontier_clusters_));
                       voxels.assign(v, v + counts.n_listed);
                   });
    }

    // ---- paths through the known free space of the latest fused frame's field (DESIGN.md §8.11) ----
    // once, after enable_known_space: the capacities of the target table and the path list, and the rounds of a job
    int enable_reach(int max_targets, int max_path_voxels, int max_rounds)
    {
        if (ctx_.run("enable_reach", [&] { return dsm_reach_enable(ctx_.ctx, max_targets, max_path_voxels, max_rounds); }) == DSM_OK)
            reach_targets_ = max_targets;
        return ctx_.err;
    }
    // the travel cost from `start` through voxels free and at least `radius` from anything not known to be free, to the
    // goals (xyz doubles, goals.size() / 3 of them) and, with with_frontiers, to the clusters the frontiers() call on
    // this frame found (include/dsm.h): targets receives info.n_targets records and path info.n_path_voxels indices.
    // DSM_E_STATE without known space, before any field, after load_state* until the next fused frame, and with
    // with_frontiers without a frontiers() call since the frame was fused; DSM_E_CAPACITY with the paths of the last
    // applied frame's field, as distance_field().
    int reach(const double start[3], float radius, int approach, const std::vector<double> &goals, bool with_frontiers, dsm_reach_info_t &info,
              std::vector<dsm_reach_target_t> &targets, std::vector<int32_t> &path)
    {
        targets.clear();
        path.clear();
        info = dsm_reach_info_t();
        const dsm_reach_target_t *t = nullptr;
        const int32_t *p = nullptr;
        return job(
            "reach", KNOWN_FIELD, goals.size() % 3 == 0,
            [&] { return dsm_reach_enqueue(ctx_.ctx, start, radius, approach, goals.data(), (int)(goals.size() / 3), with_frontiers, 0); },
            [&] { return dsm_reach_wait(ctx_.ctx, &info, &t, &p, nullptr); },
            [&] {
                targets.assign(t, t + std::min(info.n_targets, reach_targets_));
                path.assign(p, p + info.n_path_voxels);
            });
    }

    // ---- travel costs between many points of the latest fused frame's field (DESIGN.md §8.13) ----
    // once, after enable_known_space: the most sites of one call, the most active tiles of a field, and the rounds
    int enable_reach_matrix(int max_sites, int max_tiles, int max_rounds)
    {
        return ctx_.run("enable_reach_matrix", [&] { return dsm_reach_matrix_enable(ctx_.ctx, max_sites, max_tiles, max_rounds); });
    }
    // the travel costs between the points (xyz doubles, points.size() / 3 of them) through voxels free and at least
    // `radius` from anything not known to be free (include/dsm.h): sites receives one record per point and matrix the
    // n x n costs, row i from point i.  Chained after reach(with_frontiers), the points are the robot and the targets'
    // viewpoints (their voxel centres ((origin + x) + 0.5) * voxel snap to themselves).  DSM_E_STATE without known
    // space, before any field and after load_state* until the next fused frame; DSM_E_CAPACITY with the costs of the
    // last applied frame's field, as distance_field().
    int reach_matrix(const std::vector<double> &points, float radius, int approach, dsm_reach_matrix_info_t &info,
                     std::vector<dsm_reach_site_t> &sites, std::vector<uint32_t> &matrix)
    {
        sites.clear();
        matrix.clear();
        info = dsm_reach_matrix_info_t();
        const dsm_reach_site_t *s = nullptr;
        const uint32_t *m = nullptr;
        return job("reach_matrix", KNOWN_FIELD, points.size() % 3 == 0,
                   [&] { return dsm_reach_matrix_enqueue(ctx_.ctx, points.data(), (int)(points.size() / 3), radius, approach); },
                   [&] { return dsm_reach_matrix_wait(ctx_.ctx, &info, &s, &m); },
                   [&] {
                       sites.assign(s, s + info.n_sites);
                       matrix.assign(m, m + (size_t)info.n_sites * info.n_sites);
                   });
    }

    // ---- the order of an exploration tour over a travel-cost matrix (DESIGN.md §8.14) ----
    // once: the most sites and starts of one tour() call
    int enable_tour(int max_sites, int max_starts)
    {
        return ctx_.run("enable_tour", [&] { return dsm_tour_enable(ctx_.ctx, max_sites, max_starts); });
    }
    // the best of n_starts local searches over the n x n matrix (row-major, row i from site i, UINT32_MAX: no path; the
    // matrix of reach_matrix() as it stands), site 0 being the robot (include/dsm.h): starts receives one record per start
    // and order the best tour's sites, order[0] = 0 and -1 past info.n_included.  open = 1: a path from the robot; 0: a
    // tour back to it.  Reads no field, so load_state* does not affect it.
    int tour(const std::vector<uint32_t> &matrix, int n, int open, int n_starts, int max_passes, uint64_t seed, dsm_tour_info_t &info,
             std::vector<dsm_tour_start_t> &starts, std::vector<int32_t> &order)
    {
        starts.clear();
        order.clear();
        info = dsm_tour_info_t();
        const dsm_tour_start_t *s = nullptr;
        const int32_t *o = nullptr;
        return job("tour", NO_FIELD, n >= 0 && matrix.size() == (size_t)n * n,
                   [&] { return dsm_tour_enqueue(ctx_.ctx, matrix.data(), n, open, n_starts, max_passes, seed); },
                   [&] { return dsm_tour_wait(ctx_.ctx, &info, &s, &o); },
                   [&] {
                       starts.assign(s, s + info.n_starts);
                       order.assign(o, o + info.n_sites);
                   });
    }

    // ---- view gain against the known field of the latest fused frame (DESIGN.md §8.12) ----
    // once, after enable_known_space: the most views one view_gain() call scores
    int enable_view_gain(int max_views)
    {
        return ctx_.run("enable_view_gain", [&] { return dsm_gain_enable(ctx_.ctx, max_views); });
    }
    // the gain of n_views camera poses (poses: 12 doubles each, row-major [R | t], camera to world) seen with the node's
    // intrinsics out to max_range (include/dsm.h): gains receives n_views records.  clusters is empty or names, per
    // view, a cluster of the frontiers() call on this frame (-1: none).  DSM_E_STATE without known space, before any
    // field, after load_state* until the next fused frame, and with clusters without a frontiers() call since the frame
    // was fused; DSM_E_CAPACITY with the gains of the last applied frame's field, as distance_field().
    int view_gain(const double *poses, int n_views, float max_range, int unknown_blocks, const std::vector<int32_t> &clusters,
                  dsm_gain_info_t &info, std::vector<dsm_view_gain_t> &gains)
    {
        gains.clear();
        info = dsm_gain_info_t();
        const dsm_gain_camera_t cam = gain_camera(max_range, unknown_blocks);
        const dsm_view_gain_t *g = nullptr;
        return job("view_gain", KNOWN_FIELD, clusters.empty() || (int)clusters.size() == n_views,
                   [&] { return dsm_gain_enqueue(ctx_.ctx, &cam, poses, clusters.empty() ? nullptr : clusters.data(), n_views); },
                   [&] { return dsm_gain_wait(ctx_.ctx, &info, &g); }, [&] { gains.assign(g, g + info.n_views); });
    }

    // ---- viewpoints of frontier clusters against the known field of the latest fused frame (DESIGN.md §8.15) ----
    // once, after enable_known_space: the most clusters of one viewpoints() call and the most (cluster, offset) pairs
    int enable_viewpoints(int max_clusters, int max_candidates)
    {
        return ctx_.run("enable_viewpoints", [&] { return dsm_viewpoint_enable(ctx_.ctx, max_clusters, max_candidates); });
    }
    // clear candidate positions around each named cluster of the frontiers() call on this frame, each scored at the best
    // of n_rotations rotations (9 doubles each, row-major camera to world) with the node's intrinsics out to max_range
    // (include/dsm.h); params.with_reach is taken from with_reach, which ranks by the costs of the reach() call on this
    // frame.  cluster_records receives one record per cluster and viewpoints params.top_k slots per cluster; their voxel
    // centres ((origin + x) + 0.5) * voxel are the sites for reach_matrix().  DSM_E_STATE without known space, before
    // any field, after load_state* until the next fused frame, without a frontiers() call since the frame was fused,
    // and with with_reach without a reach() call since then; DSM_E_CAPACITY with the viewpoints of the last applied
    // frame's field, as distance_field().
    int viewpoints(dsm_viewpoint_params_t params, const double *rotations, int n_rotations, float max_range, int unknown_blocks,
                   const std::vector<int32_t> &clusters, int with_reach, dsm_viewpoint_info_t &info,
                   std::vector<dsm_viewpoint_cluster_t> &cluster_records, std::vector<dsm_viewpoint_t> &viewpoints)
    {
        cluster_records.clear();
        viewpoints.clear();
        info = dsm_viewpoint_info_t();
        const dsm_gain_camera_t cam = gain_camera(max_range, unknown_blocks);
        params.with_reach = with_reach;
        const dsm_viewpoint_cluster_t *c = nullptr;
        const dsm_viewpoint_t *v = nullptr;
        return job(
            "viewpoints", KNOWN_FIELD, true,
            [&] { return dsm_viewpoint_enqueue(ctx_.ctx, &cam, rotations, n_rotations, clusters.data(), (int)clusters.size(), &params); },
            [&] { return dsm_viewpoint_wait(ctx_.ctx, &info, &c, &v); },
            [&] {
                cluster_records.assign(c, c + info.n_clusters);
                viewpoints.assign(v, v + (size_t)info.n_clusters * info.top_k);
            });
    }
    // ---- viewpoints of a ground robot on the terrain of the latest fused frame (DESIGN.md §8.23) ----
    // viewpoints() on the plane of the terrain() call on this frame, with params.dz_max 0: candidate cells around each
    // cluster's column, traversable at least `radius` from any other cell, each camera `eye` voxels above the cell's
    // support (eye in [1, headroom] of that terrain() call); with_reach ranks by the costs of the reach_terrain() call on
    // that terrain.  Slot voxels are cells q P + p of the terrain grid; the camera's field voxel is the cell's column at
    // level + eye (up > 0) or level - eye (up < 0), and its centre, snapped to its column, is the cell's site for
    // reach_matrix_terrain().  DSM_E_STATE without a terrain() call on this frame, without a frontiers() call since the
    // frame was fused, with with_reach without a reach_terrain() call on that terrain, and after load_state* until the
    // next fused frame; DSM_E_CAPACITY with the viewpoints of the last applied frame's terrain.
    int viewpoints_terrain(dsm_viewpoint_params_t params, int eye, const double *rotations, int n_rotations, float max_range,
                           int unknown_blocks, const std::vector<int32_t> &clusters, int with_reach, dsm_viewpoint_info_t &info,
                           std::vector<dsm_viewpoint_cluster_t> &cluster_records, std::vector<dsm_viewpoint_t> &viewpoints)
    {
        cluster_records.clear();
        viewpoints.clear();
        info = dsm_viewpoint_info_t();
        const dsm_gain_camera_t cam = gain_camera(max_range, unknown_blocks);
        params.with_reach = with_reach;
        const dsm_viewpoint_cluster_t *c = nullptr;
        const dsm_viewpoint_t *v = nullptr;
        return job(
            "viewpoints_terrain", KNOWN_FIELD, true,
            [&] {
                return terrain_frame_ ? dsm_viewpoint_enqueue_terrain(ctx_.ctx, &cam, rotations, n_rotations, clusters.data(),
                                                                      (int)clusters.size(), &params, eye)
                                      : DSM_E_STATE;
            },
            [&] { return dsm_viewpoint_wait(ctx_.ctx, &info, &c, &v); },
            [&] {
                cluster_records.assign(c, c + info.n_clusters);
                viewpoints.assign(v, v + (size_t)info.n_clusters * info.top_k);
            });
    }

    // ---- planner queries against the field of the latest fused frame (DESIGN.md §8.8) ----
    // once, after enable_distance_field: the capacities of one query
    int enable_field_queries(int max_points, int max_trajectories, int max_waypoints)
    {
        return ctx_.run("enable_field_queries", [&] { return dsm_field_query_enable(ctx_.ctx, max_points, max_trajectories, max_waypoints); });
    }
    // distance and gradient at n points (xyz doubles); out receives n samples.  DSM_E_STATE when no field exists;
    // DSM_E_CAPACITY with the samples of the last applied frame's field, as distance_field().  signed_field: on the
    // signed grid (dsm_field_query_enqueue_signed); DSM_E_STATE also when that field was requested without it.
    int field_samples(const double *points, int n, std::vector<dsm_field_sample_t> &out, bool signed_field = false)
    {
        out.clear();
        return query("field_samples", signed_field, points, n, nullptr, nullptr, 0, 1.f, 0.f, &out, nullptr);
    }
    // the clearance of n trajectories (waypoints xyz doubles, offsets[n + 1]) sampled every `step` metres against
    // `radius`; out receives n records (include/dsm.h); signed_field as field_samples()
    int trajectory_clearance(const double *waypoints, const int32_t *offsets, int n, float step, float radius, std::vector<dsm_clearance_t> &out,
                             bool signed_field = false)
    {
        out.clear();
        return query("trajectory_clearance", signed_field, nullptr, 0, waypoints, offsets, n, step, radius, nullptr, &out);
    }
    // ---- trajectory optimisation on the signed grid of the latest fused frame (DESIGN.md §8.17) ----
    // once, after enable_signed_distance: the most trajectories, control points and L-BFGS pairs of one trajectories()
    int enable_trajectories(int max_trajectories, int max_points, int max_memory)
    {
        return ctx_.run("enable_trajectories", [&] { return dsm_trajectory_enable(ctx_.ctx, max_trajectories, max_points, max_memory); });
    }
    // n uniform cubic B-splines (control points xyz doubles, offsets[n + 1], knot intervals dt[n]) optimised against the
    // signed grid of the latest fused frame's field (include/dsm.h): records receives n records and optimised the
    // control points, laid out as the request's.  DSM_E_STATE without enable_signed_distance() before that field, before
    // any field, and after load_state* until the next fused frame; DSM_E_CAPACITY with the results of the last applied
    // frame's field, as distance_field().
    int trajectories(const double *points, const int32_t *offsets, const double *dt, int n, const dsm_trajectory_params_t &params,
                     dsm_trajectory_info_t &info, std::vector<dsm_trajectory_t> &records, std::vector<double> &optimised)
    {
        records.clear();
        optimised.clear();
        info = dsm_trajectory_info_t();
        const dsm_trajectory_t *r = nullptr;
        const double *q = nullptr;
        return job("trajectories", ANY_FIELD, true, [&] { return dsm_trajectory_enqueue(ctx_.ctx, points, offsets, dt, n, &params); },
                   [&] { return dsm_trajectory_wait(ctx_.ctx, &info, &r, &q); },
                   [&] {
                       records.assign(r, r + info.n_trajectories);
                       optimised.assign(q, q + 3 * (size_t)info.n_points);
                   });
    }
    // ---- headings along trajectories against the known field of the latest fused frame (DESIGN.md §8.19) ----
    // once, after enable_known_space: the most trajectories and samples of one headings() call
    int enable_headings(int max_trajectories, int max_samples)
    {
        return ctx_.run("enable_headings", [&] { return dsm_heading_enable(ctx_.ctx, max_trajectories, max_samples); });
    }
    // the camera heading along n uniform cubic B-splines (control points xyz doubles and offsets[n + 1], as
    // trajectories() takes and returns them), sampled `samples` times per segment and scored at n_rot rotations (9
    // doubles each, row-major camera to world, neighbouring headings next to each other, cyclically) with the node's
    // intrinsics out to max_range (include/dsm.h): records receives n records, samples_out one position, rotation and
    // turn per sample, and counts n_rot counts per sample.  DSM_E_STATE without known space, before any field and after
    // load_state* until the next fused frame; DSM_E_CAPACITY with the results of the last applied frame's field, as
    // distance_field().
    int headings(const double *points, const int32_t *offsets, int n, const double *rotations, int n_rot, int samples,
                 const dsm_heading_request_t *requests, float max_range, int unknown_blocks, int32_t w_unknown, int32_t w_frontier,
                 dsm_heading_info_t &info, std::vector<dsm_heading_t> &records, std::vector<dsm_heading_sample_t> &samples_out,
                 std::vector<dsm_heading_count_t> &counts)
    {
        records.clear();
        samples_out.clear();
        counts.clear();
        info = dsm_heading_info_t();
        const dsm_gain_camera_t cam = gain_camera(max_range, unknown_blocks);
        const dsm_heading_t *r = nullptr;
        const dsm_heading_sample_t *s = nullptr;
        const dsm_heading_count_t *c = nullptr;
        return job(
            "headings", KNOWN_FIELD, true,
            [&] { return dsm_heading_enqueue(ctx_.ctx, points, offsets, n, &cam, rotations, n_rot, samples, requests, w_unknown, w_frontier); },
            [&] { return dsm_heading_wait(ctx_.ctx, &info, &r, &s, &c); },
            [&] {
                records.assign(r, r + info.n_trajectories);
                samples_out.assign(s, s + info.n_samples);
                counts.assign(c, c + (size_t)info.n_samples * info.n_rot);
            });
    }
    // ---- the terrain of the known field of the latest fused frame (DESIGN.md §8.20) ----
    // once, after enable_known_space: up in {+-1, +-2, +-3}, the field grid's axis |up| - 1 toward + or - (-2 for the
    // y-down camera frames of KITTI poses)
    int enable_terrain(int up) { return ctx_.run("enable_terrain", [&] { return dsm_terrain_enable(ctx_.ctx, up); }); }
    // per cell of the field grid collapsed along the up axis ([m2][m1][m0], info.m): the support level, status (0 no
    // support, 1 blocked by the step, 2 traversable), step and clearance in metres (include/dsm.h) for `headroom` free
    // voxels above the support and steps of at most max_step voxels.  DSM_E_STATE without known space, before any field
    // and after load_state* until the next fused frame; DSM_E_CAPACITY with the terrain of the last applied frame's
    // field, as distance_field().
    int terrain(int headroom, int max_step, dsm_terrain_info_t &info, std::vector<int16_t> &level, std::vector<uint8_t> &status,
                std::vector<uint8_t> &step, std::vector<float> &clearance)
    {
        level.clear();
        status.clear();
        step.clear();
        clearance.clear();
        info = dsm_terrain_info_t();
        const int16_t *l = nullptr;
        const uint8_t *s = nullptr, *t = nullptr;
        const float *c = nullptr;
        return job("terrain", KNOWN_FIELD, true, [&] { return dsm_terrain_enqueue(ctx_.ctx, headroom, max_step); },
                   [&] { return dsm_terrain_wait(ctx_.ctx, &info, &l, &s, &t, &c); },
                   [&] {
                       const size_t n = (size_t)info.m[0] * info.m[1] * info.m[2];
                       level.assign(l, l + n);
                       status.assign(s, s + n);
                       step.assign(t, t + n);
                       clearance.assign(c, c + n);
                       terrain_frame_ = true;
                   });
    }
    // ---- driving paths on the terrain of the latest fused frame (DESIGN.md §8.21), after enable_reach ----
    // reach() on the plane of the terrain() call on this frame: the travel cost from the column of `start` over the
    // traversable cells at least `radius` from any other, to the columns of the goals (xyz doubles) and, with
    // with_frontiers, to the clusters of the frontiers() call on this frame.  Cells, viewpoints and path entries are
    // indices q P + p of the terrain grid; a cell's surface point lies on the level plane of terrain().  DSM_E_STATE
    // without a terrain() call on this frame, with with_frontiers without a frontiers() call on it, and after
    // load_state* until the next fused frame; DSM_E_CAPACITY with the paths of the last applied frame's terrain.
    int reach_terrain(const double start[3], float radius, int approach, const std::vector<double> &goals, bool with_frontiers,
                      dsm_reach_info_t &info, std::vector<dsm_reach_target_t> &targets, std::vector<int32_t> &path)
    {
        targets.clear();
        path.clear();
        info = dsm_reach_info_t();
        const dsm_reach_target_t *t = nullptr;
        const int32_t *p = nullptr;
        return job(
            "reach_terrain", KNOWN_FIELD, goals.size() % 3 == 0,
            [&] {
                return terrain_frame_ ? dsm_reach_enqueue_terrain(ctx_.ctx, start, radius, approach, goals.data(), (int)(goals.size() / 3),
                                                                  with_frontiers, 0)
                                      : DSM_E_STATE;
            },
            [&] { return dsm_reach_wait(ctx_.ctx, &info, &t, &p, nullptr); },
            [&] {
                targets.assign(t, t + std::min(info.n_targets, reach_targets_));
                path.assign(p, p + info.n_path_voxels);
            });
    }
    // ---- driving costs between many points on the terrain of the latest fused frame (DESIGN.md §8.22), after
    // enable_reach_matrix ----
    // reach_matrix() on the plane of the terrain() call on this frame: the travel costs between the columns of the points
    // (xyz doubles) over the traversable cells at least `radius` from any other; site voxels are cells q P + p of the
    // terrain grid.  Chained after reach_terrain(with_frontiers), the points are the robot and the viewpoint cells'
    // centres, which snap to themselves at any height.  DSM_E_STATE without a terrain() call on this frame and after
    // load_state* until the next fused frame; DSM_E_CAPACITY with the costs of the last applied frame's terrain.
    int reach_matrix_terrain(const std::vector<double> &points, float radius, int approach, dsm_reach_matrix_info_t &info,
                             std::vector<dsm_reach_site_t> &sites, std::vector<uint32_t> &matrix)
    {
        sites.clear();
        matrix.clear();
        info = dsm_reach_matrix_info_t();
        const dsm_reach_site_t *s = nullptr;
        const uint32_t *m = nullptr;
        return job(
            "reach_matrix_terrain", KNOWN_FIELD, points.size() % 3 == 0,
            [&] {
                return terrain_frame_ ? dsm_reach_matrix_enqueue_terrain(ctx_.ctx, points.data(), (int)(points.size() / 3), radius, approach)
                                      : DSM_E_STATE;
            },
            [&] { return dsm_reach_matrix_wait(ctx_.ctx, &info, &s, &m); },
            [&] {
                sites.assign(s, s + info.n_sites);
                matrix.assign(m, m + (size_t)info.n_sites * info.n_sites);
            });
    }
    // the field of the latest fused frame: dist [nz][ny][nx] in metres (the library's pinned buffer, valid until the next
    // frame is fused; nullptr for a field kept on the device), the grid's origin in voxels and the occupied voxels.  DSM_E_STATE when no frame has been fused
    // since the last call; DSM_E_CAPACITY with the field of the last applied frame, as published_clouds().
    int distance_field(const float *&dist, int32_t origin[3], int &n_occupied)
    {
        if (!ctx_.ready("distance_field")) return ctx_.err;
        if (!field_) return ctx_.done(DSM_E_STATE, "distance_field");
        field_ = false;
        return ctx_.done(dsm_field_wait(ctx_.ctx, &dist, origin, &n_occupied), "distance_field");
    }
    // publish_neighbor_pointcloud (:1283-1383): live local points, then the stored points of get_driftfree_poses(ref,
    // 2 * drift_free_poses) in list order
    int neighbor_points(int reference_index, std::vector<dsm_point_t> &points)
    {
        points.clear();
        return ctx_.run("neighbor_points",
                        [&] { return detail::neighbourhood(ctx_, driftfree_poses(reference_index, 2 * drift_free_poses_), points); });
    }
    // publish_raw_pointcloud (:1115-1151) of the last fused frame at its fuse pose
    int raw_points(std::vector<dsm_point_t> &points)
    {
        points.clear();
        if (!ctx_.ready("raw_points")) return ctx_.err;
        if (!fused_) return ctx_.done(DSM_E_STATE, "raw_points");
        const double p7[7] = {last_fuse_pose_.x, last_fuse_pose_.y, last_fuse_pose_.z, last_fuse_pose_.qx,
                              last_fuse_pose_.qy, last_fuse_pose_.qz, last_fuse_pose_.qw};
        return ctx_.done(detail::raw_cloud(ctx_, p7, width_ * height_, points), "raw_points");
    }
    // local_surfels, pool order
    int local_surfels(std::vector<dsm_surfel_t> &out)
    {
        out.clear();
        return ctx_.run("local_surfels", [&] { return detail::whole_pool(ctx_, out); });
    }
    // PoseElement::attached_surfels of one keyframe
    int attached_surfels(int pose_index, std::vector<dsm_surfel_t> &out)
    {
        out.clear();
        return ctx_.run("attached_surfels", [&] { return detail::attached(ctx_, pose_index, out); });
    }

    // ---- files ----
    // save_map (:75-81)
    int save_map(const std::string &save_name) { return save_mesh(save_name); }
    // save_mesh (:1219-1280): the attached surfels of every pose in index order, then the local surfels with
    // update_times >= 5; one hexagon each, ASCII PLY
    int save_mesh(const std::string &save_path_name)
    {
        if (!ctx_.ready("save_mesh")) return ctx_.err;
        std::vector<dsm_surfel_t> all;
        for (size_t i = 0; i < poses_.size(); i++)
        {
            if (local_.count((int)i)) continue; // a pose in the window has nothing stored
            const int rc = detail::attached(ctx_, (int)i, all);
            if (rc != DSM_OK) return ctx_.done(rc, "save_mesh");
        }
        return ctx_.done(detail::save_mesh(ctx_, save_path_name, std::move(all)), "save_mesh");
    }
    // save_cloud (:1153-1173): local points with update_times >= 5, then the inactive cloud; PCD v0.7 ASCII
    int save_cloud(const std::string &save_path_name)
    {
        return ctx_.run("save_cloud", [&] { return detail::save_cloud<dsm_point_t>(ctx_, save_path_name, nullptr); });
    }

    // ---- checkpoint and resume (DESIGN.md §8.4) ----
    // save_state writes the device map (dsm_map_save) with the node's own section as its extra bytes: the construction
    // parameters, the KITTI fix-up, every pose, the window, the queued poses, images and depths, the last warp and the
    // last fuse.  Doubles are stored bit for bit, so a node that loads the file and receives the remaining messages
    // equals, byte for byte, the node that saved it and received them.  load_state returns DSM_E_INVALID, with the node
    // unchanged, for a file without a node section, parameters other than this node's, or a stored segment whose
    // keyframe is outside the pose database or in the window; the file's own errors are dsm_map_load's.  An unread
    // publish snapshot is retired first; publishing stays as it was.  Both need a context (DSM_E_STATE).
    int save_state(const std::string &path)
    {
        if (!ctx_.ready("save_state")) return ctx_.err;
        std::vector<uint8_t> section;
        write_section(section);
        return ctx_.done(detail::save_state(ctx_, path, section), "save_state");
    }
    // The same file without stopping the node (DESIGN.md §8.5, INTEGRATION.md §4).  enable_checkpoints once after
    // construction.  save_state_async writes the node's section now -- the host state of exactly the fuses enqueued so
    // far -- and enqueues the device map behind those fuses; a thread of the context writes the file while the node goes
    // on.  Meant for a checkpoint every N keyframes from the image callback, with wait_state_saved(false, &finished)
    // polled on the next call (finished = false while the file is written; once finished it returns the write's result
    // and the next save_state_async may follow).  An unread publish snapshot stays as it is.  The file equals save_state's
    // at the same message, and load_state resumes from it.
    int enable_checkpoints()
    {
        return ctx_.run("enable_checkpoints", [&] { return dsm_checkpoint_enable(ctx_.ctx); });
    }
    int save_state_async(const std::string &path)
    {
        if (!ctx_.ready("save_state_async")) return ctx_.err;
        std::vector<uint8_t> section;
        write_section(section);
        return ctx_.done(detail::save_state_async(ctx_, path, section), "save_state_async");
    }
    int wait_state_saved(bool block, bool *finished)
    {
        return ctx_.run("wait_state_saved", [&] { return detail::wait_state_saved(ctx_, block, finished); });
    }
    int load_state(const std::string &path) { return load_from(path, false, nullptr, "load_state"); }
    // Incremental checkpoints (DESIGN.md §8.6, INTEGRATION.md §4): save_state_incremental is save_state_async, written as
    // one record of the changed chunks (and the whole node section) appended to <path>.journal, or as a new base file at
    // path when a record cannot be (the first save to path, a failed save, the map replaced, the journal larger than its
    // base).  wait_state_saved retires it.  load_state_incremental is load_state on the state base and journal resolve
    // to, with the same checks on its node section and table; *records (optional) receives the records applied.
    int save_state_incremental(const std::string &path)
    {
        if (!ctx_.ready("save_state_incremental")) return ctx_.err;
        std::vector<uint8_t> section;
        write_section(section);
        return ctx_.done(detail::save_state_incremental(ctx_, path, section), "save_state_incremental");
    }
    int load_state_incremental(const std::string &path, int *records = nullptr)
    {
        return load_from(path, true, records, "load_state_incremental");
    }

    int last_error() const { return ctx_.err; }
    dsm_ctx *context() { return ctx_.ctx; }

  private:
    // what a planner job reads: nothing, the latest fused frame's field, or its known field
    enum JobField
    {
        NO_FIELD,
        ANY_FIELD,
        KNOWN_FIELD,
    };
    // One synchronous planner job: the context ready, DSM_E_STATE without the field it reads, DSM_E_INVALID unless
    // `valid` (the caller's own argument check), then enqueue and wait, and assign takes the results of a job that
    // returned DSM_OK or DSM_E_CAPACITY (the results of the last applied frame's field, as distance_field())
    template <typename Enqueue, typename Wait, typename Assign>
    int job(const char *what, JobField reads, bool valid, Enqueue enqueue, Wait wait, Assign assign)
    {
        if (!ctx_.ready(what)) return ctx_.err;
        if ((reads == KNOWN_FIELD && known_.empty()) || (reads != NO_FIELD && !field_exists_)) return ctx_.done(DSM_E_STATE, what);
        if (!valid) return ctx_.done(DSM_E_INVALID, what);
        int rc = enqueue();
        if (rc != DSM_OK) return ctx_.done(rc, what);
        rc = wait();
        if (rc == DSM_OK || rc == DSM_E_CAPACITY) assign();
        return ctx_.done(rc, what);
    }
    // the camera of view_gain() and viewpoints(): the node's intrinsics and image size
    dsm_gain_camera_t gain_camera(float max_range, int unknown_blocks) const
    {
        dsm_gain_camera_t cam;
        cam.fx = cam_[0], cam.fy = cam_[1], cam.cx = cam_[2], cam.cy = cam_[3];
        cam.width = width_, cam.height = height_;
        cam.max_range = max_range;
        cam.unknown_blocks = unknown_blocks;
        return cam;
    }
    int query(const char *what, bool signed_field, const double *points, int n_points, const double *waypoints, const int32_t *offsets,
              int n_traj, float step, float radius, std::vector<dsm_field_sample_t> *samples, std::vector<dsm_clearance_t> *clearance)
    {
        const dsm_field_sample_t *s = nullptr;
        const dsm_clearance_t *c = nullptr;
        return job(what, ANY_FIELD, true,
                   [&] {
                       return (signed_field ? dsm_field_query_enqueue_signed : dsm_field_query_enqueue)(ctx_.ctx, points, n_points, waypoints,
                                                                                                         offsets, n_traj, step, radius);
                   },
                   [&] { return dsm_field_query_wait(ctx_.ctx, &s, &c); },
                   [&] {
                       if (samples) samples->assign(s, s + n_points);
                       if (clearance) clearance->assign(c, c + n_traj);
                   });
    }

    // load_state / load_state_incremental: the file (journal = false) or base + journal (true) peeked and checked against
    // this node before the map is touched, then loaded
    int load_from(const std::string &path, bool journal, int *records, const char *what)
    {
        if (records) *records = 0;
        if (!ctx_.ready(what)) return ctx_.err;
        size_t n_extra = 0;
        int n_seg = 0;
        auto peek = [&](void *extra, size_t cap, size_t *ne, int32_t *table, int seg_cap, int *ns) {
            return journal ? dsm_map_peek_journal(path.c_str(), extra, cap, ne, table, seg_cap, ns, nullptr)
                           : dsm_map_peek(path.c_str(), extra, cap, ne, table, seg_cap, ns);
        };
        int rc = peek(nullptr, 0, &n_extra, nullptr, 0, &n_seg);
        if (rc != DSM_OK) return ctx_.done(rc, what);
        std::vector<uint8_t> section(n_extra + 1);
        std::vector<int32_t> table(3 * (size_t)n_seg + 3);
        rc = peek(section.data(), n_extra, nullptr, table.data(), n_seg, nullptr);
        if (rc != DSM_OK) return ctx_.done(rc, what);
        section.resize(n_extra);
        State s;
        if (!read_section(section, s)) return ctx_.done(DSM_E_INVALID, what);
        for (int i = 0; i < n_seg; i++)
            if (table[3 * i] >= (int)s.poses.size() || s.local.count(table[3 * i])) return ctx_.done(DSM_E_INVALID, what);
        if (retire_unread(what) != DSM_OK) return ctx_.err; // as fuse_front does
        std::vector<uint8_t> extra;
        rc = journal ? detail::load_state_incremental(ctx_, path, extra, records) : detail::load_state(ctx_, path, extra);
        if (rc != DSM_OK) return ctx_.done(rc, what);
        transform_kitti_ = s.transform_kitti;
        poses_.swap(s.poses);
        local_.swap(s.local);
        pose_buffer_.swap(s.pose_buffer);
        image_buffer_.swap(s.image_buffer);
        depth_buffer_.swap(s.depth_buffer);
        last_warp_.swap(s.last_warp);
        last_fuse_pose_ = s.last_fuse_pose;
        last_ref_ = s.last_ref;
        fused_ = s.fused;
        field_exists_ = false; // the loaded map has no field until its next fused frame
        terrain_frame_ = false;
        // a version-2 section restores the slot table the library's views match; without one the table starts empty
        for (size_t i = 0; i < known_.size(); i++)
            known_[i] = s.views ? KnownView{s.view_ref[i], s.view_rel[i]} : KnownView{-1, Pose()};
        captures_ = s.views ? s.captures : 0, captured_ref_ = s.views ? s.captured_ref : -1;
        return ctx_.done(DSM_OK, what);
    }

    struct PendingPose
    {
        double stamp;
        Pose relative;
        int reference_index;
    };

    // ---- the node's section of a checkpoint, in order; little-endian, doubles bit for bit ----
    //   char magic[8] "DSMNODE\0", uint32 version, int32 width, height, double fx, fy, cx, cy, far, near (as given),
    //   int32 drift_free_poses, double transform_kitti[16] (column-major),
    //   int32 n_poses, per pose: double cam_pose[7], loop_pose[7], cam_stamp, int32 n_links, int32 links[n_links],
    //   int32 n_local, int32 local[n_local] (ascending),
    //   int32 n_pose_buffer, per entry: double stamp, double relative[7], int32 reference_index,
    //   int32 n_images, per image: double stamp, uint8 gray[H*W];  int32 n_depths, per depth: double stamp, float depth[H*W],
    //   int32 n_warp, per transform: int32 pose, float W[16],
    //   double last_fuse_pose[7], int32 last_ref, int32 fused
    // version 2 (enable_view_checkpoints) appends: int32 max_views, float max_range, int32 captures, captured_ref,
    //   per slot: int32 reference_index (-1: empty), double relative[7]
    enum { kSectionVersion = 1, kSectionVersionViews = 2 };
    struct State
    {
        node_math::M4 transform_kitti;
        std::vector<NodePose> poses;
        std::set<int> local;
        std::deque<PendingPose> pose_buffer;
        std::deque<std::pair<double, std::vector<uint8_t> > > image_buffer;
        std::deque<std::pair<double, std::vector<float> > > depth_buffer;
        std::vector<NodeWarp> last_warp;
        Pose last_fuse_pose;
        int last_ref;
        bool fused;
        bool views = false; // a version-2 section: the slot table below
        int captures = 0, captured_ref = -1;
        std::vector<int> view_ref;
        std::vector<Pose> view_rel;
    };
    static const char *section_magic() { return "DSMNODE"; } // with its terminating zero: 8 bytes
    struct Writer
    {
        std::vector<uint8_t> &b;
        void raw(const void *p, size_t n)
        {
            const uint8_t *q = static_cast<const uint8_t *>(p);
            b.insert(b.end(), q, q + n);
        }
        template <class T>
        void put(const T &v)
        {
            raw(&v, sizeof(T));
        }
    };
    struct Reader
    {
        const std::vector<uint8_t> &b;
        size_t o;
        bool raw(void *p, size_t n)
        {
            if (n > b.size() - o) return false;
            if (n) std::memcpy(p, &b[o], n);
            o += n;
            return true;
        }
        template <class T>
        bool get(T &v)
        {
            return raw(&v, sizeof(T));
        }
        // a count that the rest of the section can hold at `each` bytes per element
        bool count(int32_t &n, size_t each) { return get(n) && n >= 0 && (size_t)n <= (b.size() - o) / each; }
    };
    void write_section(std::vector<uint8_t> &out) const
    {
        Writer w = {out};
        w.raw(section_magic(), 8);
        w.put((uint32_t)(view_checkpoints_ ? kSectionVersionViews : kSectionVersion));
        w.put((int32_t)width_), w.put((int32_t)height_);
        w.raw(cam_, sizeof(cam_));
        w.put((int32_t)drift_free_poses_);
        w.raw(transform_kitti_.d, sizeof(transform_kitti_.d));
        w.put((int32_t)poses_.size());
        for (size_t i = 0; i < poses_.size(); i++)
        {
            const NodePose &p = poses_[i];
            w.put(p.cam_pose), w.put(p.loop_pose), w.put(p.cam_stamp);
            w.put((int32_t)p.linked_pose_index.size());
            for (size_t j = 0; j < p.linked_pose_index.size(); j++) w.put((int32_t)p.linked_pose_index[j]);
        }
        w.put((int32_t)local_.size());
        for (std::set<int>::const_iterator it = local_.begin(); it != local_.end(); ++it) w.put((int32_t)*it);
        w.put((int32_t)pose_buffer_.size());
        for (size_t i = 0; i < pose_buffer_.size(); i++)
            w.put(pose_buffer_[i].stamp), w.put(pose_buffer_[i].relative), w.put((int32_t)pose_buffer_[i].reference_index);
        w.put((int32_t)image_buffer_.size());
        for (size_t i = 0; i < image_buffer_.size(); i++) w.put(image_buffer_[i].first), w.raw(image_buffer_[i].second.data(), image_buffer_[i].second.size());
        w.put((int32_t)depth_buffer_.size());
        for (size_t i = 0; i < depth_buffer_.size(); i++)
            w.put(depth_buffer_[i].first), w.raw(depth_buffer_[i].second.data(), depth_buffer_[i].second.size() * 4);
        w.put((int32_t)last_warp_.size());
        for (size_t i = 0; i < last_warp_.size(); i++) w.put((int32_t)last_warp_[i].pose), w.raw(last_warp_[i].W, sizeof(last_warp_[i].W));
        w.put(last_fuse_pose_), w.put((int32_t)last_ref_), w.put((int32_t)fused_);
        if (!view_checkpoints_) return;
        w.put((int32_t)known_.size()), w.put(known_range_), w.put((int32_t)captures_), w.put((int32_t)captured_ref_);
        for (size_t i = 0; i < known_.size(); i++) w.put((int32_t)known_[i].ref), w.put(known_[i].relative);
    }
    // false for anything but a section of version 1, or of version 2 on a node with view checkpoints, written by a node
    // with this node's parameters (and, in version 2, its max_views and max_range, every slot's keyframe in the database)
    bool read_section(const std::vector<uint8_t> &in, State &s) const
    {
        static_assert(sizeof(Pose) == 56, "Pose: 7 doubles");
        Reader r = {in, 0};
        char magic[8];
        uint32_t version = 0;
        int32_t w = 0, h = 0, dfp = 0, n = 0;
        double cam[6];
        if (!r.raw(magic, 8) || std::memcmp(magic, section_magic(), 8) != 0 || !r.get(version)) return false;
        s.views = version == (uint32_t)kSectionVersionViews;
        if (version != (uint32_t)kSectionVersion && !(s.views && view_checkpoints_)) return false;
        if (!r.get(w) || !r.get(h) || !r.raw(cam, sizeof(cam)) || !r.get(dfp)) return false;
        if (w != width_ || h != height_ || std::memcmp(cam, cam_, sizeof(cam)) != 0 || dfp != drift_free_poses_) return false;
        if (!r.raw(s.transform_kitti.d, sizeof(s.transform_kitti.d)) || !r.count(n, 2 * sizeof(Pose) + 12)) return false;
        s.poses.resize((size_t)n);
        for (size_t i = 0; i < s.poses.size(); i++)
        {
            NodePose &p = s.poses[i];
            int32_t nl = 0;
            if (!r.get(p.cam_pose) || !r.get(p.loop_pose) || !r.get(p.cam_stamp) || !r.count(nl, 4)) return false;
            p.linked_pose_index.resize((size_t)nl);
            for (int32_t j = 0; j < nl; j++)
            {
                int32_t k = 0;
                if (!r.get(k) || k < 0 || k >= n) return false;
                p.linked_pose_index[(size_t)j] = k;
            }
        }
        int32_t m = 0;
        if (!r.count(m, 4)) return false;
        for (int32_t j = 0; j < m; j++)
        {
            int32_t k = 0;
            if (!r.get(k) || k < 0 || k >= n) return false;
            s.local.insert(k);
        }
        if (!r.count(m, 8 + sizeof(Pose) + 4)) return false;
        for (int32_t j = 0; j < m; j++)
        {
            PendingPose q;
            int32_t ref = 0;
            if (!r.get(q.stamp) || !r.get(q.relative) || !r.get(ref) || ref < 0 || ref >= n) return false;
            q.reference_index = ref;
            s.pose_buffer.push_back(q);
        }
        const size_t px = (size_t)width_ * height_;
        if (!r.count(m, 8 + px)) return false;
        for (int32_t j = 0; j < m; j++)
        {
            s.image_buffer.push_back(std::make_pair(0.0, std::vector<uint8_t>(px)));
            if (!r.get(s.image_buffer.back().first) || !r.raw(s.image_buffer.back().second.data(), px)) return false;
        }
        if (!r.count(m, 8 + 4 * px)) return false;
        for (int32_t j = 0; j < m; j++)
        {
            s.depth_buffer.push_back(std::make_pair(0.0, std::vector<float>(px)));
            if (!r.get(s.depth_buffer.back().first) || !r.raw(s.depth_buffer.back().second.data(), 4 * px)) return false;
        }
        if (!r.count(m, sizeof(NodeWarp))) return false;
        s.last_warp.resize((size_t)m);
        for (size_t j = 0; j < s.last_warp.size(); j++)
        {
            int32_t pose = 0;
            if (!r.get(pose) || !r.raw(s.last_warp[j].W, sizeof(s.last_warp[j].W))) return false;
            s.last_warp[j].pose = pose;
        }
        int32_t ref = 0, fused = 0;
        if (!r.get(s.last_fuse_pose) || !r.get(ref) || !r.get(fused)) return false;
        s.last_ref = ref, s.fused = fused != 0;
        if (s.views)
        {
            int32_t max_views = 0, captures = 0, captured_ref = 0;
            float max_range = 0.f;
            if (!r.get(max_views) || !r.get(max_range) || !r.get(captures) || !r.get(captured_ref)) return false;
            if (max_views != (int32_t)known_.size() || std::memcmp(&max_range, &known_range_, 4) != 0 || captures < 0) return false;
            if (captured_ref < -1 || captured_ref >= n) return false;
            s.captures = captures, s.captured_ref = captured_ref;
            s.view_ref.resize((size_t)max_views);
            s.view_rel.resize((size_t)max_views);
            for (int32_t j = 0; j < max_views; j++)
            {
                int32_t k = 0;
                if (!r.get(k) || k < -1 || k >= n || !r.get(s.view_rel[(size_t)j])) return false;
                s.view_ref[(size_t)j] = k;
            }
        }
        return r.o == in.size();
    }

    static Point3 position(const Pose &p)
    {
        Point3 q;
        q.x = p.x, q.y = p.y, q.z = p.z;
        return q;
    }
    // synchronize_msgs (:147-150): cam_pose of the reference now, times the queued relative pose
    node_math::M4 fuse_pose(const PendingPose &q) const
    {
        return node_math::mul(node_math::from_pose(poses_[(size_t)q.reference_index].cam_pose), node_math::from_pose(q.relative));
    }

    // synchronize_msgs (:103-163): the oldest pose is fused once an image and a depth with exactly its stamp are there
    int synchronize()
    {
        while (!pose_buffer_.empty())
        {
            const double t = pose_buffer_.front().stamp;
            bool find_image = false, find_depth = false, newer = false;
            while (!image_buffer_.empty() && image_buffer_.front().first < t) image_buffer_.pop_front();
            if (!image_buffer_.empty()) (image_buffer_.front().first == t ? find_image : newer) = true;
            while (!depth_buffer_.empty() && depth_buffer_.front().first < t) depth_buffer_.pop_front();
            if (!depth_buffer_.empty()) (depth_buffer_.front().first == t ? find_depth : newer) = true;
            if (newer)
            { // this pose's image or depth never came: drop it, try the next
                pose_buffer_.pop_front();
                continue;
            }
            if (!find_image || !find_depth) return DSM_OK;
            return fuse_front();
        }
        return DSM_OK;
    }

    // the fuse of synchronize_msgs (:144-163): move_add_surfels and fuse_map as one dsm_fuse_stream_window call
    int fuse_front()
    {
        const PendingPose q = pose_buffer_.front();
        const node_math::M4 fuse = fuse_pose(q);
        float pose16[16];
        node_math::to_float(fuse, pose16);
        std::vector<int> remove, add;
        window_lists(q.reference_index, remove, add);
        if (ctx_.ctx)
        {
            if (retire_unread("fuse") != DSM_OK) return ctx_.err;
            const int rc = detail::fuse_window(ctx_, q.reference_index, image_buffer_.front().second.data(),
                                               depth_buffer_.front().second.data(), pose16, remove, add);
            if (ctx_.done(rc, "fuse") != DSM_OK) return rc;
        }
        for (size_t i = 0; i < remove.size(); i++) local_.erase(remove[i]);
        local_.insert(add.begin(), add.end());
        last_fuse_pose_ = node_math::to_pose(fuse);
        last_ref_ = q.reference_index;
        fused_ = true;
        pose_buffer_.pop_front();
        // after the bookkeeping: the frame is enqueued, so the host window follows the device whatever this returns
        if (!known_.empty() && q.reference_index != captured_ref_)
        { // the first fused frame of a new reference keyframe: frame 0 of the call just made
            const int slot = captures_ % (int)known_.size();
            if (ctx_.done(dsm_views_capture(ctx_.ctx, 0, slot), "fuse") == DSM_OK)
            {
                known_[(size_t)slot] = KnownView{q.reference_index, q.relative};
                captures_++;
                captured_ref_ = q.reference_index;
            }
        }
        if (publishing_) snapshot_ = ctx_.done(dsm_publish_enqueue(ctx_.ctx, 5), "fuse") == DSM_OK;
        if (distance_field_ && (!publishing_ || snapshot_))
        { // centred on the fuse pose's translation, with the threshold of the published active cloud
            const double c[3] = {last_fuse_pose_.x, last_fuse_pose_.y, last_fuse_pose_.z};
            int rc;
            if (!known_.empty())
            {
                std::vector<int32_t> slots;
                std::vector<double> poses;
                known_views(slots, poses);
                rc = dsm_field_enqueue_known(ctx_.ctx, c, 5, slots.data(), poses.data(), (int)slots.size(), field_host_copy_ ? 1 : 0);
            }
            else
                rc = field_host_copy_ ? dsm_field_enqueue(ctx_.ctx, c, 5) : dsm_field_enqueue_resident(ctx_.ctx, c, 5);
            field_ = ctx_.done(rc, "fuse") == DSM_OK;
            terrain_frame_ = false; // a new field: terrain() has not run on it
            field_exists_ = field_exists_ || field_;
        }
        return publishing_ || distance_field_ ? ctx_.err : DSM_OK;
    }
    // the unread snapshot and field of the previous frame are retired (a pose callback may have enqueued loop-closure
    // warps since, so neither can be reused); a capacity report stays with the readers
    int retire_unread(const char *what)
    {
        if (snapshot_)
        {
            const int rc = dsm_publish_wait(ctx_.ctx, nullptr, nullptr, nullptr, nullptr, nullptr);
            snapshot_ = false;
            if (rc != DSM_OK && rc != DSM_E_CAPACITY) return ctx_.done(rc, what);
        }
        if (field_)
        {
            const int rc = dsm_field_wait(ctx_.ctx, nullptr, nullptr, nullptr);
            field_ = false;
            if (rc != DSM_OK && rc != DSM_E_CAPACITY) return ctx_.done(rc, what);
        }
        return DSM_OK;
    }

    // warp_surfels (:681-824) in the schedule described at the top of this file
    void warp_surfels()
    {
        using namespace node_math;
        if (local_.empty()) return;
        NodeWarp w;
        const NodePose &lp = poses_[(size_t)*local_.begin()];
        w.pose = -1;
        to_float(mul(from_pose(lp.loop_pose), inverse(from_pose(lp.cam_pose))), w.W);
        last_warp_.push_back(w);
        for (size_t i = 0; i < poses_.size(); i++)
        {
            NodePose &p = poses_[i];
            if (same_position(p.cam_pose, p.loop_pose)) continue;
            if (!local_.count((int)i))
            {
                w.pose = (int)i;
                to_float(mul(from_pose(p.loop_pose), inverse(from_pose(p.cam_pose))), w.W);
                last_warp_.push_back(w);
            }
            p.cam_pose = p.loop_pose;
        }
        if (!ctx_.ctx) return;
        for (size_t i = 0; i < last_warp_.size(); i++)
        {
            const NodeWarp &x = last_warp_[i];
            const int rc = x.pose < 0 ? dsm_pool_transform(ctx_.ctx, x.W) : dsm_inactive_transform(ctx_.ctx, x.pose, x.W);
            if (rc != DSM_OK && ctx_.err == DSM_OK) ctx_.done(rc, "warp_surfels");
        }
    }

    detail::Context ctx_;
    int width_, height_, drift_free_poses_;
    double cam_[6]; // fx, fy, cx, cy, far, near as given to the constructor
    node_math::M4 transform_kitti_;
    std::vector<NodePose> poses_;
    std::set<int> local_;
    std::deque<PendingPose> pose_buffer_;
    std::deque<std::pair<double, std::vector<uint8_t> > > image_buffer_;
    std::deque<std::pair<double, std::vector<float> > > depth_buffer_;
    std::vector<NodeWarp> last_warp_;
    Pose last_fuse_pose_;
    int last_ref_;
    bool fused_;
    bool publishing_ = false, snapshot_ = false; // enable_publishing; a snapshot is enqueued and not yet handed out
    bool distance_field_ = false, field_ = false; // enable_distance_field; a field is enqueued and not yet handed out
    bool field_host_copy_ = true;  // enable_distance_field's host_copy
    bool field_exists_ = false;    // a fused frame has enqueued a field: the queries have a grid to read
    bool terrain_frame_ = false;   // terrain() has run on the latest fused frame's field: reach_terrain() has a plane
    // enable_known_space: per capture slot, the reference keyframe (-1: empty) and the pose relative to it
    struct KnownView
    {
        int ref;
        Pose relative;
    };
    std::vector<KnownView> known_; // empty without known space
    int captures_ = 0, captured_ref_ = -1; // captures so far; the reference keyframe of the latest
    float known_range_ = 0.f;              // enable_known_space's max_range
    bool view_checkpoints_ = false;        // enable_view_checkpoints: section version 2
    int frontier_clusters_ = 0;            // enable_frontiers' max_clusters
    int reach_targets_ = 0;                // enable_reach's max_targets
};
} // namespace dsm
