// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with known space, with or without enable_terrain(-2), enable_frontiers(), enable_reach() and enable_viewpoints(), and
// dumps the ground viewpoints of every fused frame with the grid, frontiers, reach start, rotations and parameters they
// were chosen on, and the node's clouds.  A ground planner's chain: terrain(3, 1), frontiers(1), reach_terrain() from the
// field's middle, then viewpoints_terrain() over every cluster.  After depth message `reload_at` the node saves its
// state and loads it back.
// Usage: viewpoint_terrain_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive voxel nx ny nz
//                               max_views max_range enabled reload_at in.bin out.bin out_prefix
//   enabled = 0: no terrain, frontiers, reach or viewpoints (the known field is requested and not dumped).
//   out.bin: after every depth message: when enabled, int32 rc (of viewpoints_terrain(), or of the call before it that
//            failed), int32 unknown_blocks (the message count % 2), float max_range (voxel * (10 + 5 (count % 3))), int32
//            eye (1 + count % 3), int32 origin[3], the state grid (int32 n + n bytes) of the field distance_field()
//            handed out, the clusters of frontiers(1) (int32 n + n dsm_frontier_cluster_t) and its voxel list (int32 n +
//            n int32), the reach start (3 doubles; radius 0.1 and approach 1; with_reach = count % 2 decides whether
//            viewpoints_terrain() uses it), the rotations (int32 n + n doubles: eight yaws level and four pitched up, in
//            the y-down frame of up -2), the named clusters (int32 n + n int32: every table entry and two past it),
//            dsm_viewpoint_params_t's first eight int32 and its float radius, dsm_viewpoint_info_t, the cluster records
//            (int32 n + n dsm_viewpoint_cluster_t) and the slots (int32 n + n dsm_viewpoint_t), int32 the rc of
//            viewpoints_terrain() before terrain() on that frame, and int32 the rc of viewpoints_terrain() right after
//            load_state at message reload_at (1 at every other message); then, always, int32 rc and the clouds of
//            active_points() and inactive_points() (each int32 n + n points); at the end: local_surfels (int32 n +
//            records), and the node's save_mesh and save_cloud go to <out_prefix>.ply / <out_prefix>.pcd.
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "driver_io.hpp"

#include <cmath>

int main(int argc, char **argv)
{
    if (argc != 24) return 2;
    const NodeArgs args(argv, true);
    const FieldArgs field(argv);
    const int reload_at = atoi(argv[20]);
    const bool on = atoi(argv[19]) != 0;
    DriverNode node(args);
    if (const int e = setup_code(node.last_error())) return e;
    if (const int e = field.enable(node)) return e;
    if (on && (node.enable_terrain(-2) != DSM_OK || node.enable_frontiers(64, 1 << 16) != DSM_OK ||
               node.enable_reach(8, 1 << 12, 4096) != DSM_OK || node.enable_viewpoints(66, 1 << 16) != DSM_OK))
        return 4;
    if (!open_io(argv[21], argv[22])) return 5;
    const std::string prefix = argv[23];
    std::vector<dsm_frontier_cluster_t> clusters;
    std::vector<int32_t> voxels, path, named;
    std::vector<dsm_reach_target_t> targets;
    std::vector<dsm_viewpoint_cluster_t> records;
    std::vector<dsm_viewpoint_t> slots;
    std::vector<int16_t> level;
    std::vector<uint8_t> status, step;
    std::vector<float> clearance;
    std::vector<double> rotations;
    for (int k = 0; k < 12; k++)
    { // up is -y: forward f in the x-z plane (pitched up toward -y), right r = (-up) x f_horizontal, down d = f x r
        const double a = 0.25 * M_PI * (k % 8), p = k < 8 ? 0.0 : 0.3;
        const double f[3] = {std::cos(p) * std::cos(a), -std::sin(p), std::cos(p) * std::sin(a)}, r[3] = {std::sin(a), 0.0, -std::cos(a)};
        const double d[3] = {f[1] * r[2] - f[2] * r[1], f[2] * r[0] - f[0] * r[2], f[0] * r[1] - f[1] * r[0]};
        for (int i = 0; i < 3; i++) rotations.push_back(r[i]), rotations.push_back(d[i]), rotations.push_back(f[i]); // row i: (r_i, d_i, f_i)
    }
    int depth_msgs = 0;
    const int e = feed_script(node, args.W, args.H, [&]() -> int {
        const int ub = depth_msgs % 2, with_reach = depth_msgs % 2, eye = 1 + depth_msgs % 3;
        const float max_range = field.voxel * (float)(10 + 5 * (depth_msgs % 3));
        dsm_viewpoint_params_t prm = {1, 5, 0, 1 + depth_msgs % 2, 64, 1, 4, with_reach, 0.1f, 0};
        dsm_frontier_counts_t counts = dsm_frontier_counts_t();
        dsm_terrain_info_t tinfo = dsm_terrain_info_t();
        dsm_reach_info_t rinfo = dsm_reach_info_t();
        dsm_viewpoint_info_t info = dsm_viewpoint_info_t();
        const FieldHandout h(node, true);
        double start[3];
        field.middle(h.origin, start);
        int before_terrain = 1, rt = DSM_OK, rf = DSM_OK, rr = DSM_OK, rv = DSM_OK;
        if (on && h.ok())
        {
            named.clear();
            before_terrain = node.viewpoints_terrain(prm, eye, rotations.data(), 12, max_range, ub, named, with_reach, info, records, slots);
            rt = node.terrain(3, 1, tinfo, level, status, step, clearance);
            rf = node.frontiers(1, clusters, voxels, counts);
            for (int k = 0; k < (int)clusters.size() + 2; k++) named.push_back(k);
            if (rt == DSM_OK && rf == DSM_OK) rr = node.reach_terrain(start, prm.radius, 1, std::vector<double>(), false, rinfo, targets, path);
            if (rt == DSM_OK && rf == DSM_OK && rr == DSM_OK)
                rv = node.viewpoints_terrain(prm, eye, rotations.data(), 12, max_range, ub, named, with_reach, info, records, slots);
        }
        if (on)
        {
            put(first_error({h.rc, h.rs, rt, rf, rr, rv}));
            put(ub);
            put(max_range);
            put(eye);
            h.put_origin();
            h.put_state(field);
            put_list(clusters);
            put_list(voxels);
            for (double s : start) put(s);
            put_list(rotations);
            put_list(named);
            put(prm.r_min), put(prm.r_max), put(prm.dz_max), put(prm.stride), put(prm.max_samples), put(prm.min_seen), put(prm.top_k);
            put(prm.with_reach), put(prm.radius);
            put(info);
            put_list(records);
            put_list(slots);
            put(before_terrain);
        }
        int after_load = 1;
        if (++depth_msgs == reload_at)
        {
            if (!reload(node, prefix)) return 6;
            if (on) after_load = node.viewpoints_terrain(prm, eye, rotations.data(), 12, max_range, ub, named, 0, info, records, slots);
        }
        if (on) put(after_load);
        put_clouds(node);
        return 0;
    });
    return e ? e : end_drive(node, prefix);
}
