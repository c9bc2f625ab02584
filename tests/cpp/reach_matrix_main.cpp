// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with known space, with or without enable_reach_matrix(), and dumps the travel-cost matrix of every fused frame with the
// grids and points it was found on, and the node's clouds.  A planner's chain: frontiers(), reach(with_frontiers) from
// the field's centre, then reach_matrix over that point and the reached viewpoints' centres.  After depth message
// `reload_at` the node saves its state and loads it back.
// Usage: reach_matrix_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive voxel nx ny nz
//                          max_views max_range max_sites max_tiles max_rounds reload_at in.bin out.bin out_prefix
//   max_sites = max_tiles = max_rounds = 0: no frontiers, paths or matrices (the known field is requested and not
//   dumped).
//   out.bin: after every depth message: with matrices, int32 rc (of reach_matrix(), or of the reader before it that
//            failed), int32 approach (the message count % 5), float radius (voxel * (count % 3) / 2), int32 origin[3],
//            the state grid (int32 n + n bytes) and the distance grid (int32 n + n floats) of the field
//            distance_field() handed out, the points (int32 n + n doubles, xyz each), dsm_reach_matrix_info_t, the
//            sites (int32 n + n dsm_reach_site_t) and the matrix (int32 n + n uint32), and int32 the rc of
//            reach_matrix() right after load_state at message reload_at (1 at every other message); then, always,
//            int32 rc and the clouds of active_points() and inactive_points() (each int32 n + n points); at the end:
//            local_surfels (int32 n + records), and the node's save_mesh and save_cloud go to <out_prefix>.ply /
//            <out_prefix>.pcd.
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "driver_io.hpp"

int main(int argc, char **argv)
{
    if (argc != 26) return 2;
    const NodeArgs args(argv, true);
    const float voxel = (float)atof(argv[13]);
    const int nx = atoi(argv[14]), ny = atoi(argv[15]), nz = atoi(argv[16]);
    const int max_views = atoi(argv[17]), max_sites = atoi(argv[19]), max_tiles = atoi(argv[20]), max_rounds = atoi(argv[21]);
    const int reload_at = atoi(argv[22]);
    const bool matrices = max_sites > 0 || max_tiles > 0 || max_rounds > 0;
    DriverNode node(args);
    if (const int e = setup_code(node.last_error())) return e;
    if (node.enable_distance_field(voxel, nx, ny, nz) != DSM_OK) return 4;
    if (node.enable_known_space(max_views, (float)atof(argv[18])) != DSM_OK) return 4;
    if (matrices && (node.enable_frontiers(64, 1 << 16) != DSM_OK || node.enable_reach(max_sites - 1, 1 << 16, max_rounds) != DSM_OK ||
                     node.enable_reach_matrix(max_sites, max_tiles, max_rounds) != DSM_OK))
        return 4;
    if (!open_io(argv[23], argv[24])) return 5;
    const std::string prefix = argv[25];
    std::vector<dsm_frontier_cluster_t> clusters;
    std::vector<int32_t> voxels, path;
    std::vector<dsm_reach_target_t> targets;
    std::vector<dsm_reach_site_t> sites;
    std::vector<uint32_t> matrix;
    std::vector<double> points;
    const std::vector<double> no_goals;
    int depth_msgs = 0;
    const int e = feed_script(node, args.W, args.H, [&]() -> int {
        const int k = depth_msgs % 5;
        const float radius = voxel * (float)(depth_msgs % 3) / 2.f;
        dsm_frontier_counts_t counts = dsm_frontier_counts_t();
        dsm_reach_info_t rinfo = dsm_reach_info_t();
        dsm_reach_matrix_info_t info = dsm_reach_matrix_info_t();
        // the jobs are enqueued behind the field request of the frame just fused, before that field is handed out
        const int rf = matrices ? node.frontiers(1, clusters, voxels, counts) : DSM_OK;
        const float *dist = nullptr;
        int32_t origin[3] = {0, 0, 0};
        int n_occ = 0;
        const int rc = node.distance_field(dist, origin, n_occ);
        const uint8_t *state = nullptr;
        int n_free = 0;
        const int rs = rc == DSM_OK ? node.known_space(state, n_free) : rc;
        const int n[3] = {nx, ny, nz};
        double start[3];
        for (int a = 0; a < 3; a++) start[a] = ((double)(origin[a] + n[a] / 2) + 0.5) * (double)voxel;
        int rr = DSM_OK, rm = DSM_OK;
        points.assign(start, start + 3);
        if (matrices && rc == DSM_OK && rs == DSM_OK && rf == DSM_OK)
        {
            rr = node.reach(start, radius, k, no_goals, true, rinfo, targets, path);
            for (const dsm_reach_target_t &t : targets)
                if (t.status == 0)
                {
                    const int v = t.viewpoint, c[3] = {v % nx, v / nx % ny, v / (nx * ny)};
                    for (int a = 0; a < 3; a++) points.push_back(((double)(origin[a] + c[a]) + 0.5) * (double)voxel);
                }
            if (rr == DSM_OK) rm = node.reach_matrix(points, radius, k, info, sites, matrix);
        }
        if (matrices)
        {
            const bool ok = rc == DSM_OK && rs == DSM_OK;
            put(rc != DSM_OK ? rc : rs != DSM_OK ? rs : rf != DSM_OK ? rf : rr != DSM_OK ? rr : rm);
            put(k);
            put(radius);
            put(origin[0]), put(origin[1]), put(origin[2]);
            put_n(state, ok ? nx * ny * nz : 0);
            put_n(dist, ok ? nx * ny * nz : 0);
            put_list(points);
            put(info);
            put_list(sites);
            put_list(matrix);
        }
        int after_load = 1;
        if (++depth_msgs == reload_at)
        {
            if (node.save_state(prefix + ".state") != DSM_OK || node.load_state(prefix + ".state") != DSM_OK) return 6;
            if (matrices) after_load = node.reach_matrix(points, radius, k, info, sites, matrix);
        }
        if (matrices) put(after_load);
        put_clouds(node);
        return 0;
    });
    if (e) return e;
    std::vector<dsm_surfel_t> local;
    if (node.local_surfels(local) != DSM_OK) return 6;
    put_list(local);
    if (!save_files(node, prefix)) return 6;
    return close_io();
}
