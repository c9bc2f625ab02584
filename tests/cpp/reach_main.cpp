// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with known space, with or without enable_frontiers() and enable_reach(), and dumps the paths of every fused frame with
// the grids and frontiers they were found on, and the node's clouds.  After depth message `reload_at` the node saves its
// state and loads it back.
// Usage: reach_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive voxel nx ny nz max_views
//                   max_range max_targets max_path_voxels max_rounds reload_at in.bin out.bin out_prefix
//   max_targets = max_path_voxels = max_rounds = 0: no frontiers and no paths (the known field is requested and not
//   dumped).
//   out.bin: after every depth message: with paths, int32 rc (of reach(), or of the reader before it that failed),
//            int32 approach (the message count % 5), double start[3] (the centre of the field's middle voxel), float
//            radius (voxel * (count % 3) / 2), int32 origin[3], the state grid (int32 n + n bytes) and the distance grid
//            (int32 n + n floats) of the field distance_field() handed out, the clusters of frontiers(1) (int32 n + n
//            dsm_frontier_cluster_t) and its voxel list (int32 n + n int32), dsm_reach_info_t, the targets (int32 n + n
//            dsm_reach_target_t) and the path list (int32 n + n int32) of reach(with_frontiers) to those clusters, int32
//            the rc of reach(with_frontiers) before frontiers() on that frame, and int32 the rc of reach() right after
//            load_state at message reload_at (1 at every other message); then, always, int32 rc and the clouds of
//            active_points() and inactive_points() (each int32 n + n points); at the end: local_surfels (int32 n +
//            records), and the node's save_mesh and save_cloud go to <out_prefix>.ply / <out_prefix>.pcd.
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "driver_io.hpp"

int main(int argc, char **argv)
{
    if (argc != 26) return 2;
    const NodeArgs args(argv, true);
    const FieldArgs field(argv);
    const int max_targets = atoi(argv[19]), max_path = atoi(argv[20]), max_rounds = atoi(argv[21]), reload_at = atoi(argv[22]);
    const bool paths = max_targets > 0 || max_path > 0 || max_rounds > 0;
    DriverNode node(args);
    if (const int e = setup_code(node.last_error())) return e;
    if (const int e = field.enable(node)) return e;
    if (paths && (node.enable_frontiers(max_targets, 1 << 16) != DSM_OK || node.enable_reach(max_targets, max_path, max_rounds) != DSM_OK))
        return 4;
    if (!open_io(argv[23], argv[24])) return 5;
    const std::string prefix = argv[25];
    std::vector<dsm_frontier_cluster_t> clusters;
    std::vector<int32_t> voxels, path;
    std::vector<dsm_reach_target_t> targets;
    const std::vector<double> no_goals;
    int depth_msgs = 0;
    const int e = feed_script(node, args.W, args.H, [&]() -> int {
        const int k = depth_msgs % 5;
        const float radius = field.voxel * (float)(depth_msgs % 3) / 2.f;
        dsm_frontier_counts_t counts = dsm_frontier_counts_t();
        dsm_reach_info_t info = dsm_reach_info_t();
        double start[3] = {0.0, 0.0, 0.0};
        int before = 1, rr = DSM_OK;
        // the jobs are enqueued behind the field request of the frame just fused, before that field is handed out
        if (paths) before = node.reach(start, radius, k, no_goals, true, info, targets, path);
        const int rf = paths ? node.frontiers(1, clusters, voxels, counts) : DSM_OK;
        const FieldHandout h(node, true);
        field.middle(h.origin, start);
        if (paths && h.ok() && rf == DSM_OK) rr = node.reach(start, radius, k, no_goals, true, info, targets, path);
        if (paths)
        {
            put(first_error({h.rc, h.rs, rf, rr}));
            put(k);
            put(start[0]), put(start[1]), put(start[2]);
            put(radius);
            h.put_origin();
            h.put_state(field);
            h.put_dist(field);
            put_list(clusters);
            put_list(voxels);
            put(info);
            put_list(targets);
            put_list(path);
            put(before);
        }
        int after_load = 1;
        if (++depth_msgs == reload_at)
        {
            if (!reload(node, prefix)) return 6;
            if (paths) after_load = node.reach(start, radius, k, no_goals, false, info, targets, path);
        }
        if (paths) put(after_load);
        put_clouds(node);
        return 0;
    });
    return e ? e : end_drive(node, prefix);
}
