// Timing harness of tools/measure_field_known.py: drives dsm::SurfelMapNode (include/dsm_surfel_node.hpp) through the
// message script of tools/measure_node.py with a host-copy distance field every frame, read right after every fuse, and
// times the whole drive on the host clock, the device synchronised once at the end (and wherever the node waits).
// Usage: measure_field_known W H fx fy cx cy far near drift_free_poses frames.bin script.bin mode voxel nx ny nz max_views
//                            max_range
//   frames.bin / script.bin: as tools/measure_node.cpp (the script's per-frame publish flag is ignored)
//   mode  p: the plain field (enable_distance_field only)
//         k: known space as well (enable_known_space(max_views, max_range)); known_space() is read with every field
// Prints one JSON object: "occupied" and "free" are summed over the drive's fields, "views" is the slot count of the
// last field.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "dsm_surfel_node.hpp"

typedef std::chrono::steady_clock clk;
static double ms(clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); }

int main(int argc, char **argv)
{
    if (argc != 19) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]);
    const char mode = argv[12][0];
    const float voxel = (float)atof(argv[13]);
    const int nx = atoi(argv[14]), ny = atoi(argv[15]), nz = atoi(argv[16]), max_views = atoi(argv[17]);
    const float max_range = (float)atof(argv[18]);
    if (mode != 'p' && mode != 'k') return 2;
    FILE *ff = fopen(argv[10], "rb"), *fs = fopen(argv[11], "rb");
    if (!ff || !fs) return 5;
    int K = 0, T = 0;
    if (fread(&K, 4, 1, ff) != 1 || fread(&T, 4, 1, fs) != 1) return 5;
    std::vector<std::vector<uint8_t> > gray((size_t)K, std::vector<uint8_t>((size_t)W * H));
    std::vector<std::vector<float> > depth((size_t)K, std::vector<float>((size_t)W * H));
    for (int k = 0; k < K; k++)
        if (fread(gray[k].data(), 1, gray[k].size(), ff) != gray[k].size() || fread(depth[k].data(), 4, depth[k].size(), ff) != depth[k].size())
            return 5;
    dsm::SurfelMapNode node(W, H, atof(argv[3]), atof(argv[4]), atof(argv[5]), atof(argv[6]), atof(argv[7]), atof(argv[8]), atoi(argv[9]), 0);
    if (node.last_error() != DSM_OK) return node.last_error() == DSM_E_NODEVICE ? 3 : 4;
    if (node.enable_distance_field(voxel, nx, ny, nz) != DSM_OK) return 4;
    if (mode == 'k' && node.enable_known_space(max_views, max_range) != DSM_OK) return 4;
    struct Msg
    {
        double stamp, pose[7];
        int kf, ref, k;
        std::vector<double> path;
    };
    std::vector<Msg> msgs((size_t)T);
    for (int t = 0; t < T; t++)
    {
        Msg &m = msgs[(size_t)t];
        int n_path = 0, n_loops = 0, publish = 0;
        if (fread(&m.stamp, 8, 1, fs) != 1 || fread(&m.kf, 4, 1, fs) != 1 || fread(&m.ref, 4, 1, fs) != 1 || fread(&m.k, 4, 1, fs) != 1 ||
            fread(m.pose, 8, 7, fs) != 7 || fread(&n_path, 4, 1, fs) != 1)
            return 5;
        m.path.resize((size_t)7 * n_path + 1);
        if (fread(m.path.data(), 8, (size_t)7 * n_path, fs) != (size_t)7 * n_path || fread(&n_loops, 4, 1, fs) != 1 || n_loops != 0 ||
            fread(&publish, 4, 1, fs) != 1)
            return 5;
    }
    const float *dist = nullptr;
    const uint8_t *state = nullptr;
    int32_t origin[3];
    int n_occ = 0, n_free = 0, rc = DSM_OK, fields = 0, views = 0;
    long long occupied = 0, free_voxels = 0;
    std::vector<int32_t> slots;
    std::vector<double> poses;
    dsm_sync(node.context());
    const clk::time_point t0 = clk::now();
    for (int t = 0; t < T && rc == DSM_OK; t++)
    {
        const Msg &m = msgs[(size_t)t];
        rc = node.orb_results_input(m.stamp, nullptr, 0, m.path.data(), (int)(m.path.size() / 7), m.pose, m.kf != 0, m.ref);
        if (rc == DSM_OK) rc = node.image_input(m.stamp, gray[(size_t)m.k].data(), (size_t)W);
        if (rc == DSM_OK) rc = node.depth_input(m.stamp, depth[(size_t)m.k].data(), (size_t)W * 4);
        if (rc == DSM_OK) rc = node.distance_field(dist, origin, n_occ);
        if (rc == DSM_OK && mode == 'k') rc = node.known_space(state, n_free);
        occupied += n_occ, free_voxels += n_free, fields++;
    }
    if (rc != DSM_OK) return 6;
    dsm_sync(node.context());
    const double total = ms(t0, clk::now());
    if (mode == 'k') views = (int)(node.known_views(slots, poses), slots.size());
    std::printf("{\"mode\": \"%c\", \"frames\": %d, \"total_ms\": %.3f, \"ms_per_frame\": %.4f, \"fields\": %d, \"occupied\": %lld, "
                "\"free\": %lld, \"views\": %d}\n",
                mode, T, total, total / (T ? T : 1), fields, occupied, free_voxels, views);
    return 0;
}
