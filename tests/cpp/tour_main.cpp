// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with known space and dumps, for every fused frame, the exploration tour over the travel-cost matrix of a planner's
// chain: frontiers(), reach(with_frontiers) from the field's centre, reach_matrix over that point and the reached
// viewpoints' centres, then tour() over that matrix as it stands.
// Usage: tour_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive voxel nx ny nz max_views
//                  max_range max_sites max_tiles max_rounds n_starts max_passes in.bin out.bin
//   out.bin: after every depth message: int32 rc (of tour(), or of the reader before it that failed), int32 open (the
//            message count % 2), uint64 seed (the message count), the matrix (int32 n*n + n*n uint32),
//            dsm_tour_info_t, the starts (int32 n + n dsm_tour_start_t) and the order (int32 n + n int32).
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "driver_io.hpp"

int main(int argc, char **argv)
{
    if (argc != 26) return 2;
    const NodeArgs args(argv, true);
    const float voxel = (float)atof(argv[13]);
    const int nx = atoi(argv[14]), ny = atoi(argv[15]), nz = atoi(argv[16]);
    const int max_views = atoi(argv[17]), max_sites = atoi(argv[19]), max_tiles = atoi(argv[20]), max_rounds = atoi(argv[21]);
    const int n_starts = atoi(argv[22]), max_passes = atoi(argv[23]);
    DriverNode node(args);
    if (const int e = setup_code(node.last_error())) return e;
    if (node.enable_distance_field(voxel, nx, ny, nz) != DSM_OK) return 4;
    if (node.enable_known_space(max_views, (float)atof(argv[18])) != DSM_OK) return 4;
    if (node.enable_frontiers(64, 1 << 16) != DSM_OK || node.enable_reach(max_sites - 1, 1 << 16, max_rounds) != DSM_OK ||
        node.enable_reach_matrix(max_sites, max_tiles, max_rounds) != DSM_OK || node.enable_tour(max_sites, n_starts) != DSM_OK)
        return 4;
    if (!open_io(argv[24], argv[25])) return 5;
    std::vector<dsm_frontier_cluster_t> clusters;
    std::vector<int32_t> voxels, path, order;
    std::vector<dsm_reach_target_t> targets;
    std::vector<dsm_reach_site_t> sites;
    std::vector<uint32_t> matrix;
    std::vector<dsm_tour_start_t> starts;
    std::vector<double> points;
    const std::vector<double> no_goals;
    int depth_msgs = 0;
    const int e = feed_script(node, args.W, args.H, [&]() -> int {
        const int open = depth_msgs % 2;
        const uint64_t seed = (uint64_t)depth_msgs++;
        dsm_frontier_counts_t counts = dsm_frontier_counts_t();
        dsm_reach_info_t rinfo = dsm_reach_info_t();
        dsm_reach_matrix_info_t minfo = dsm_reach_matrix_info_t();
        dsm_tour_info_t info = dsm_tour_info_t();
        // the jobs are enqueued behind the field request of the frame just fused, before that field is handed out
        int rc = node.frontiers(1, clusters, voxels, counts);
        const float *dist = nullptr;
        int32_t origin[3] = {0, 0, 0};
        int n_occ = 0;
        if (rc == DSM_OK) rc = node.distance_field(dist, origin, n_occ);
        const int n[3] = {nx, ny, nz};
        points.clear();
        for (int a = 0; a < 3; a++) points.push_back(((double)(origin[a] + n[a] / 2) + 0.5) * (double)voxel);
        if (rc == DSM_OK) rc = node.reach(points.data(), 0.f, 1, no_goals, true, rinfo, targets, path);
        if (rc == DSM_OK)
        {
            for (const dsm_reach_target_t &t : targets)
                if (t.status == 0)
                {
                    const int v = t.viewpoint, c[3] = {v % nx, v / nx % ny, v / (nx * ny)};
                    for (int a = 0; a < 3; a++) points.push_back(((double)(origin[a] + c[a]) + 0.5) * (double)voxel);
                }
            rc = node.reach_matrix(points, 0.f, 1, minfo, sites, matrix);
        }
        if (rc == DSM_OK) rc = node.tour(matrix, minfo.n_sites, open, n_starts, max_passes, seed, info, starts, order);
        put(rc);
        put(open);
        put(seed);
        put_list(matrix);
        put(info);
        put_list(starts);
        put_list(order);
        return 0;
    });
    if (e) return e;
    return close_io();
}
