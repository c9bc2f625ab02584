// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with known space, with or without enable_frontiers(), and dumps the frontiers of every fused frame with the state grid
// they were found on, and the node's clouds.  After depth message `reload_at` the node saves its state and loads it back.
// Usage: frontier_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive voxel nx ny nz
//                      max_views max_range max_clusters max_voxels reload_at in.bin out.bin out_prefix
//   max_clusters = max_voxels = 0: no frontiers (the known field is requested and not dumped).
//   out.bin: after every depth message: with frontiers, int32 rc (of frontiers(), or of the reader before it that
//            failed), int32 min_voxels (1, 2, 50 by message), int32 origin[3] and the state grid (int32 n + n bytes) of
//            the field distance_field() handed out, the clusters (int32 n + n dsm_frontier_cluster_t), the voxel list
//            (int32 n + n int32), dsm_frontier_counts_t, and int32 the rc of frontiers() right after load_state at
//            message reload_at (1 at every other message); then, always, int32 rc and the clouds of active_points() and
//            inactive_points() (each int32 n + n points); at the end: local_surfels (int32 n + records), and the node's
//            save_mesh and save_cloud go to <out_prefix>.ply / <out_prefix>.pcd.
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "driver_io.hpp"

int main(int argc, char **argv)
{
    if (argc != 25) return 2;
    const NodeArgs args(argv, true);
    const FieldArgs field(argv);
    const int max_clusters = atoi(argv[19]), max_voxels = atoi(argv[20]), reload_at = atoi(argv[21]);
    const bool frontiers = max_clusters > 0 || max_voxels > 0;
    DriverNode node(args);
    if (const int e = setup_code(node.last_error())) return e;
    if (const int e = field.enable(node)) return e;
    if (frontiers && node.enable_frontiers(max_clusters, max_voxels) != DSM_OK) return 4;
    if (!open_io(argv[22], argv[23])) return 5;
    const std::string prefix = argv[24];
    const int ms[3] = {1, 2, 50};
    std::vector<dsm_frontier_cluster_t> clusters;
    std::vector<int32_t> voxels;
    int depth_msgs = 0;
    const int e = feed_script(node, args.W, args.H, [&]() -> int {
        const int m = ms[depth_msgs % 3];
        dsm_frontier_counts_t counts = dsm_frontier_counts_t();
        // the job is enqueued behind the field request of the frame just fused, before that field is handed out
        const int rf = frontiers ? node.frontiers(m, clusters, voxels, counts) : DSM_OK;
        const FieldHandout h(node, true);
        if (frontiers)
        {
            put(first_error({h.rc, h.rs, rf}));
            put(m);
            h.put_origin();
            h.put_state(field);
            put_list(clusters);
            put_list(voxels);
            put(counts);
        }
        int after_load = 1;
        if (++depth_msgs == reload_at)
        {
            if (!reload(node, prefix)) return 6;
            if (frontiers) after_load = node.frontiers(1, clusters, voxels, counts);
        }
        if (frontiers) put(after_load);
        put_clouds(node);
        return 0;
    });
    return e ? e : end_drive(node, prefix);
}
