// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with known space, with or without enable_frontiers() and enable_view_gain(), and dumps the gains of every fused frame
// with the grid, frontiers and poses they were scored on, and the node's clouds.  After depth message `reload_at` the
// node saves its state and loads it back.
// Usage: gain_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive voxel nx ny nz max_views
//                  max_range max_gain_views reload_at in.bin out.bin out_prefix
//   max_gain_views = 0: no frontiers and no gains (the known field is requested and not dumped).
//   out.bin: after every depth message: with gains, int32 rc (of view_gain(), or of the reader before it that failed),
//            int32 unknown_blocks (the message count % 2), float max_range (voxel * (10 + 5 (count % 3))), int32
//            origin[3], the state grid (int32 n + n bytes) of the field distance_field() handed out, the clusters of
//            frontiers(1) (int32 n + n dsm_frontier_cluster_t) and its voxel list (int32 n + n int32), the poses (int32
//            n + n doubles: eight yaws about the world z axis at the centre of the field's middle voxel), the cluster
//            per view (int32 n + n int32), dsm_gain_info_t and the gains (int32 n + n dsm_view_gain_t) of view_gain()
//            with those clusters, int32 the rc of view_gain(clusters) before frontiers() on that frame, and int32 the rc
//            of view_gain() right after load_state at message reload_at (1 at every other message); then, always, int32
//            rc and the clouds of active_points() and inactive_points() (each int32 n + n points); at the end:
//            local_surfels (int32 n + records), and the node's save_mesh and save_cloud go to <out_prefix>.ply /
//            <out_prefix>.pcd.
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "driver_io.hpp"

#include <cmath>

int main(int argc, char **argv)
{
    if (argc != 24) return 2;
    const NodeArgs args(argv, true);
    const FieldArgs field(argv);
    const int max_gain_views = atoi(argv[19]), reload_at = atoi(argv[20]);
    const bool gain = max_gain_views > 0;
    DriverNode node(args);
    if (const int e = setup_code(node.last_error())) return e;
    if (const int e = field.enable(node)) return e;
    if (gain && (node.enable_frontiers(64, 1 << 16) != DSM_OK || node.enable_view_gain(max_gain_views) != DSM_OK)) return 4;
    if (!open_io(argv[21], argv[22])) return 5;
    const std::string prefix = argv[23];
    std::vector<dsm_frontier_cluster_t> clusters;
    std::vector<int32_t> voxels;
    std::vector<dsm_view_gain_t> gains;
    const int n_yaws = 8;
    std::vector<double> poses(12 * n_yaws, 0.0);
    std::vector<int32_t> named(n_yaws, -1);
    int depth_msgs = 0;
    const int e = feed_script(node, args.W, args.H, [&]() -> int {
        const int ub = depth_msgs % 2;
        const float max_range = field.voxel * (float)(10 + 5 * (depth_msgs % 3));
        dsm_frontier_counts_t counts = dsm_frontier_counts_t();
        dsm_gain_info_t info = dsm_gain_info_t();
        int before = 1, rg = DSM_OK;
        // the jobs are enqueued behind the field request of the frame just fused, before that field is handed out
        if (gain) before = node.view_gain(poses.data(), n_yaws, max_range, ub, named, info, gains);
        const int rf = gain ? node.frontiers(1, clusters, voxels, counts) : DSM_OK;
        const FieldHandout h(node, true);
        double centre[3];
        field.middle(h.origin, centre);
        for (int k = 0; k < n_yaws; k++)
        {
            const double a = 0.25 * M_PI * k, f[3] = {std::cos(a), std::sin(a), 0.0}, r[3] = {std::sin(a), -std::cos(a), 0.0},
                         d[3] = {0.0, 0.0, -1.0};
            for (int i = 0; i < 3; i++)
            {
                double *row = &poses[12 * k + 4 * i];
                row[0] = r[i], row[1] = d[i], row[2] = f[i];
                row[3] = centre[i];
            }
            named[k] = k % ((int)clusters.size() + 2) - 1;
        }
        if (gain && h.ok() && rf == DSM_OK) rg = node.view_gain(poses.data(), n_yaws, max_range, ub, named, info, gains);
        if (gain)
        {
            put(first_error({h.rc, h.rs, rf, rg}));
            put(ub);
            put(max_range);
            h.put_origin();
            h.put_state(field);
            put_list(clusters);
            put_list(voxels);
            put_list(poses);
            put_list(named);
            put(info);
            put_list(gains);
            put(before);
        }
        int after_load = 1;
        if (++depth_msgs == reload_at)
        {
            if (!reload(node, prefix)) return 6;
            if (gain) after_load = node.view_gain(poses.data(), n_yaws, max_range, ub, std::vector<int32_t>(), info, gains);
        }
        if (gain) put(after_load);
        put_clouds(node);
        return 0;
    });
    return e ? e : end_drive(node, prefix);
}
