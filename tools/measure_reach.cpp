// Timing harness of tools/measure_reach.py: drives dsm::SurfelMapNode (include/dsm_surfel_node.hpp) through the message
// script of tools/measure_node.py with a host-copy known field every frame, read right after every fuse, and times the
// whole drive on the host clock, the device synchronised once at the end (and wherever the node waits).
// Usage: measure_reach W H fx fy cx cy far near drift_free_poses frames.bin script.bin mode voxel nx ny nz max_views
//                      max_range max_rounds
//   frames.bin / script.bin: as tools/measure_node.cpp (the script's per-frame publish flag is ignored)
//   mode  f: frontiers (enable_frontiers(4096, 1 << 20)); frontiers(1) every frame before the field is read
//         r: paths as well (enable_reach(4096, 1 << 18, max_rounds)); reach(with_frontiers) from the centre of the
//            field's middle voxel (the camera's), radius one voxel, approach 2, right after frontiers(1)
// Prints one JSON object: "reached" sums the reached targets, "converged" counts the converged jobs and "most_rounds" is
// the most rounds a job ran.
#include "measure_drive.hpp"

int main(int argc, char **argv)
{
    if (argc != 20) return 2;
    const int W = atoi(argv[1]);
    const char mode = argv[12][0];
    const float voxel = (float)atof(argv[13]);
    const int nx = atoi(argv[14]), ny = atoi(argv[15]), nz = atoi(argv[16]), max_views = atoi(argv[17]);
    const float max_range = (float)atof(argv[18]);
    const int max_rounds = atoi(argv[19]);
    if (mode != 'f' && mode != 'r') return 2;
    Drive d;
    if (!d.load(argv)) return 5;
    const int T = (int)d.msgs.size();
    DriveNode node(argv);
    if (const int e = node.setup_code()) return e;
    if (node.enable_distance_field(voxel, nx, ny, nz) != DSM_OK) return 4;
    if (node.enable_known_space(max_views, max_range) != DSM_OK) return 4;
    if (node.enable_frontiers(4096, 1 << 20) != DSM_OK) return 4;
    if (mode == 'r' && node.enable_reach(4096, 1 << 18, max_rounds) != DSM_OK) return 4;
    const float *dist = nullptr;
    const uint8_t *state = nullptr;
    int32_t origin[3] = {0, 0, 0};
    int n_occ = 0, n_free = 0, rc = DSM_OK;
    long long reached = 0, converged = 0, most_rounds = 0;
    std::vector<dsm_frontier_cluster_t> table;
    std::vector<int32_t> voxels, path;
    std::vector<dsm_reach_target_t> targets;
    const std::vector<double> no_goals;
    dsm_frontier_counts_t counts;
    dsm_reach_info_t info;
    dsm_sync(node.context());
    const clk::time_point t0 = clk::now();
    for (int t = 0; t < T && rc == DSM_OK; t++)
    {
        const DriveMsg &m = d.msgs[(size_t)t];
        rc = m.orb(node);
        if (rc == DSM_OK) rc = d.images(node, m, W);
        if (rc == DSM_OK) rc = node.frontiers(1, table, voxels, counts);
        if (rc == DSM_OK && mode == 'r')
        { // the previous field's origin locates this one's middle voxel to within the camera's motion of one frame
            const double start[3] = {((double)(origin[0] + nx / 2) + 0.5) * (double)voxel, ((double)(origin[1] + ny / 2) + 0.5) * (double)voxel,
                                     ((double)(origin[2] + nz / 2) + 0.5) * (double)voxel};
            rc = node.reach(start, voxel, 2, no_goals, true, info, targets, path);
            for (size_t i = 0; i < targets.size(); i++) reached += targets[i].status == 0;
            converged += info.converged;
            most_rounds = std::max(most_rounds, (long long)info.rounds);
        }
        if (rc == DSM_OK) rc = node.distance_field(dist, origin, n_occ);
        if (rc == DSM_OK) rc = node.known_space(state, n_free);
    }
    if (rc != DSM_OK) return 6;
    dsm_sync(node.context());
    const double total = ms(t0, clk::now());
    std::printf("{\"mode\": \"%c\", \"frames\": %d, \"total_ms\": %.3f, \"ms_per_frame\": %.4f, \"reached\": %lld, \"converged\": %lld, "
                "\"most_rounds\": %lld}\n",
                mode, T, total, total / (T ? T : 1), reached, converged, most_rounds);
    return 0;
}
