// Timing harness of tools/measure_field.py: drives dsm::SurfelMapNode (include/dsm_surfel_node.hpp) through the message
// script of tools/measure_node.py with or without the distance field and times the whole drive on the host clock, the
// device synchronised once at the end (and wherever the mode itself waits).
// Usage: measure_field W H fx fy cx cy far near drift_free_poses frames.bin script.bin mode voxel nx ny nz
//   frames.bin / script.bin: as tools/measure_node.cpp (the script's per-frame publish flag is ignored)
//   mode  a: no field
//         f: distance_field() of frame t-1 at the start of frame t's callbacks (the last one after the drive)
//         g: distance_field() right after every frame's fuse
// Prints one JSON object; "occupied" is the sum of n_occupied over the fields handed out.
#include "measure_drive.hpp"

int main(int argc, char **argv)
{
    if (argc != 17) return 2;
    const int W = atoi(argv[1]);
    const char mode = argv[12][0];
    const float voxel = (float)atof(argv[13]);
    const int nx = atoi(argv[14]), ny = atoi(argv[15]), nz = atoi(argv[16]);
    if (mode != 'a' && mode != 'f' && mode != 'g') return 2;
    Drive d;
    if (!d.load(argv)) return 5;
    const int T = (int)d.msgs.size();
    DriveNode node(argv);
    if (const int e = node.setup_code()) return e;
    if (mode != 'a' && node.enable_distance_field(voxel, nx, ny, nz) != DSM_OK) return 4;
    const float *dist = nullptr;
    int32_t origin[3];
    int n_occ = 0, rc = DSM_OK, fields = 0;
    long long occupied = 0;
    dsm_sync(node.context());
    const clk::time_point t0 = clk::now();
    for (int t = 0; t < T && rc == DSM_OK; t++)
    {
        const DriveMsg &m = d.msgs[(size_t)t];
        if (mode == 'f' && t > 0)
        {
            rc = node.distance_field(dist, origin, n_occ);
            occupied += n_occ, fields++;
        }
        if (rc == DSM_OK) rc = m.orb(node);
        if (rc == DSM_OK) rc = d.images(node, m, W);
        if (rc != DSM_OK) break;
        if (mode == 'g')
        {
            rc = node.distance_field(dist, origin, n_occ);
            occupied += n_occ, fields++;
        }
    }
    if (rc == DSM_OK && mode == 'f')
    {
        rc = node.distance_field(dist, origin, n_occ);
        occupied += n_occ, fields++;
    }
    if (rc != DSM_OK) return 6;
    dsm_sync(node.context());
    const double total = ms(t0, clk::now());
    int n_store = 0, n_pool = 0;
    if (dsm_inactive_size(node.context(), &n_store, nullptr) != DSM_OK || dsm_pool_size(node.context(), &n_pool) != DSM_OK) return 6;
    std::printf("{\"mode\": \"%c\", \"frames\": %d, \"total_ms\": %.3f, \"ms_per_frame\": %.4f, \"store_surfels\": %d, \"pool_surfels\": %d, "
                "\"fields\": %d, \"occupied\": %lld}\n",
                mode, T, total, total / (T ? T : 1), n_store, n_pool, fields, occupied);
    return 0;
}
