// Timing harness of tools/measure_gain.py: drives dsm::SurfelMapNode (include/dsm_surfel_node.hpp) through the message
// script of tools/measure_node.py with a host-copy known field every frame, read right after every fuse, and times the
// whole drive on the host clock, the device synchronised once at the end (and wherever the node waits).
// Usage: measure_gain W H fx fy cx cy far near drift_free_poses frames.bin script.bin mode voxel nx ny nz max_views
//                     max_range gain_range
//   frames.bin / script.bin: as tools/measure_node.cpp (the script's per-frame publish flag is ignored)
//   mode  r: frontiers(1) and reach(with_frontiers) from the centre of the field's middle voxel (the camera's), radius
//            one voxel, approach 2, every frame before the field is read (enable_frontiers(4096, 1 << 20),
//            enable_reach(4096, 1 << 18, 64))
//         g: view_gain() as well (enable_view_gain(512)): eight yaws about the world z axis at each of the first 64
//            reached viewpoints, each naming its cluster, out to gain_range, unknown voxels blocking
// Prints one JSON object: "views" sums the scored views.
#include "measure_drive.hpp"

#include <cmath>

int main(int argc, char **argv)
{
    if (argc != 20) return 2;
    const int W = atoi(argv[1]);
    const char mode = argv[12][0];
    const float voxel = (float)atof(argv[13]);
    const int nx = atoi(argv[14]), ny = atoi(argv[15]), nz = atoi(argv[16]), max_views = atoi(argv[17]);
    const float max_range = (float)atof(argv[18]), gain_range = (float)atof(argv[19]);
    if (mode != 'r' && mode != 'g') return 2;
    Drive d;
    if (!d.load(argv)) return 5;
    const int T = (int)d.msgs.size();
    DriveNode node(argv);
    if (const int e = node.setup_code()) return e;
    if (node.enable_distance_field(voxel, nx, ny, nz) != DSM_OK) return 4;
    if (node.enable_known_space(max_views, max_range) != DSM_OK) return 4;
    if (node.enable_frontiers(4096, 1 << 20) != DSM_OK || node.enable_reach(4096, 1 << 18, 64) != DSM_OK) return 4;
    if (mode == 'g' && node.enable_view_gain(512) != DSM_OK) return 4;
    const float *dist = nullptr;
    const uint8_t *state = nullptr;
    int32_t origin[3] = {0, 0, 0};
    int n_occ = 0, n_free = 0, rc = DSM_OK;
    long long views = 0;
    std::vector<dsm_frontier_cluster_t> table;
    std::vector<int32_t> voxels, path, named;
    std::vector<dsm_reach_target_t> targets;
    std::vector<dsm_view_gain_t> gains;
    std::vector<double> poses;
    const std::vector<double> no_goals;
    dsm_frontier_counts_t counts;
    dsm_reach_info_t info;
    dsm_gain_info_t ginfo;
    dsm_sync(node.context());
    const clk::time_point t0 = clk::now();
    for (int t = 0; t < T && rc == DSM_OK; t++)
    {
        const DriveMsg &m = d.msgs[(size_t)t];
        rc = m.orb(node);
        if (rc == DSM_OK) rc = d.images(node, m, W);
        if (rc == DSM_OK) rc = node.frontiers(1, table, voxels, counts);
        if (rc == DSM_OK)
        { // the previous field's origin locates this one's middle voxel to within the camera's motion of one frame
            const double start[3] = {((double)(origin[0] + nx / 2) + 0.5) * (double)voxel, ((double)(origin[1] + ny / 2) + 0.5) * (double)voxel,
                                     ((double)(origin[2] + nz / 2) + 0.5) * (double)voxel};
            rc = node.reach(start, voxel, 2, no_goals, true, info, targets, path);
        }
        if (rc == DSM_OK && mode == 'g')
        {
            poses.clear();
            named.clear();
            for (size_t i = 0; i < targets.size() && named.size() < 512; i++)
            {
                if (targets[i].status != 0) continue;
                const int u = targets[i].viewpoint;
                const int g[3] = {u % nx, u / nx % ny, u / (nx * ny)};
                for (int k = 0; k < 8; k++)
                {
                    const double a = 0.25 * M_PI * k, f[3] = {std::cos(a), std::sin(a), 0.0}, r[3] = {std::sin(a), -std::cos(a), 0.0},
                                 dn[3] = {0.0, 0.0, -1.0};
                    for (int j = 0; j < 3; j++)
                    {
                        const double row[4] = {r[j], dn[j], f[j], ((double)(info.origin[j] + g[j]) + 0.5) * (double)voxel};
                        poses.insert(poses.end(), row, row + 4);
                    }
                    named.push_back((int32_t)i - info.n_goals);
                }
            }
            rc = node.view_gain(poses.data(), (int)named.size(), gain_range, 1, named, ginfo, gains);
            views += (long long)named.size();
        }
        if (rc == DSM_OK) rc = node.distance_field(dist, origin, n_occ);
        if (rc == DSM_OK) rc = node.known_space(state, n_free);
    }
    if (rc != DSM_OK) return 6;
    dsm_sync(node.context());
    const double total = ms(t0, clk::now());
    std::printf("{\"mode\": \"%c\", \"frames\": %d, \"total_ms\": %.3f, \"ms_per_frame\": %.4f, \"views\": %lld}\n", mode, T, total,
                total / (T ? T : 1), views);
    return 0;
}
