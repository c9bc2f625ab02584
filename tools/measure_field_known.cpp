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
#include "measure_drive.hpp"

int main(int argc, char **argv)
{
    if (argc != 19) return 2;
    const int W = atoi(argv[1]);
    const char mode = argv[12][0];
    const float voxel = (float)atof(argv[13]);
    const int nx = atoi(argv[14]), ny = atoi(argv[15]), nz = atoi(argv[16]), max_views = atoi(argv[17]);
    const float max_range = (float)atof(argv[18]);
    if (mode != 'p' && mode != 'k') return 2;
    Drive d;
    if (!d.load(argv)) return 5;
    const int T = (int)d.msgs.size();
    DriveNode node(argv);
    if (const int e = node.setup_code()) return e;
    if (node.enable_distance_field(voxel, nx, ny, nz) != DSM_OK) return 4;
    if (mode == 'k' && node.enable_known_space(max_views, max_range) != DSM_OK) return 4;
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
        const DriveMsg &m = d.msgs[(size_t)t];
        rc = m.orb(node);
        if (rc == DSM_OK) rc = d.images(node, m, W);
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
