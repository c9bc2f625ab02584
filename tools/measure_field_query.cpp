// Timing harness of tools/measure_field_query.py: drives dsm::SurfelMapNode (include/dsm_surfel_node.hpp) through the
// message script of tools/measure_node.py with a distance field every frame and times the whole drive on the host clock,
// the device synchronised once at the end (and wherever the mode itself waits).
// Usage: measure_field_query W H fx fy cx cy far near drift_free_poses frames.bin script.bin mode voxel nx ny nz
//   frames.bin / script.bin: as tools/measure_node.cpp (the script's per-frame publish flag is ignored)
//   mode  h: host-copy field, distance_field() read right after every frame's fuse
//         q: resident field, one trajectory_clearance() of 4096 trajectories of 32 waypoints (step voxel / 2,
//            radius 2 voxels) right after every frame's fuse, then distance_field() for its origin
// The trajectories are fixed offsets (drawn before the clock, within 12 m of the origin) added to the frame's camera.
// Prints one JSON object; "hits" is the number of trajectories with a first_hit over the drive.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "dsm_surfel_node.hpp"

typedef std::chrono::steady_clock clk;
static double ms(clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); }

int main(int argc, char **argv)
{
    if (argc != 17) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]);
    const char mode = argv[12][0];
    const float voxel = (float)atof(argv[13]);
    const int nx = atoi(argv[14]), ny = atoi(argv[15]), nz = atoi(argv[16]);
    const int n_traj = 4096, per_traj = 32;
    if (mode != 'h' && mode != 'q') return 2;
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
    if (node.enable_distance_field(voxel, nx, ny, nz, mode == 'h') != DSM_OK) return 4;
    if (mode == 'q' && node.enable_field_queries(0, n_traj, n_traj * per_traj) != DSM_OK) return 4;
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
    // trajectories: a random walk of 31 steps of up to 0.4 m per axis from a start within 10 m of the origin
    std::vector<double> rel((size_t)3 * n_traj * per_traj), wp(rel.size());
    std::vector<int32_t> offsets((size_t)n_traj + 1);
    srand(7);
    for (int j = 0; j < n_traj; j++)
    {
        double p[3];
        for (int k = 0; k < 3; k++) p[k] = (rand() / (double)RAND_MAX - 0.5) * (k == 2 ? 2.0 : 20.0);
        for (int i = 0; i < per_traj; i++)
            for (int k = 0; k < 3; k++)
            {
                rel[(size_t)3 * (j * per_traj + i) + k] = p[k];
                p[k] += (rand() / (double)RAND_MAX - 0.5) * 0.8;
            }
        offsets[(size_t)j] = j * per_traj;
    }
    offsets[(size_t)n_traj] = n_traj * per_traj;
    std::vector<dsm_clearance_t> clearance;
    const float *dist = nullptr;
    int32_t origin[3];
    int n_occ = 0, rc = DSM_OK, fields = 0;
    long long occupied = 0, hits = 0;
    dsm_sync(node.context());
    const clk::time_point t0 = clk::now();
    for (int t = 0; t < T && rc == DSM_OK; t++)
    {
        const Msg &m = msgs[(size_t)t];
        rc = node.orb_results_input(m.stamp, nullptr, 0, m.path.data(), (int)(m.path.size() / 7), m.pose, m.kf != 0, m.ref);
        if (rc == DSM_OK) rc = node.image_input(m.stamp, gray[(size_t)m.k].data(), (size_t)W);
        if (rc == DSM_OK) rc = node.depth_input(m.stamp, depth[(size_t)m.k].data(), (size_t)W * 4);
        if (rc != DSM_OK) break;
        if (mode == 'q')
        {
            const dsm::Pose c = node.pose_graph().camera;
            for (size_t i = 0; i < rel.size(); i += 3) wp[i] = rel[i] + c.x, wp[i + 1] = rel[i + 1] + c.y, wp[i + 2] = rel[i + 2] + c.z;
            rc = node.trajectory_clearance(wp.data(), offsets.data(), n_traj, voxel / 2, 2 * voxel, clearance);
            for (size_t j = 0; j < clearance.size(); j++) hits += clearance[j].first_hit >= 0;
        }
        if (rc == DSM_OK) rc = node.distance_field(dist, origin, n_occ);
        occupied += n_occ, fields++;
    }
    if (rc != DSM_OK) return 6;
    dsm_sync(node.context());
    const double total = ms(t0, clk::now());
    std::printf("{\"mode\": \"%c\", \"frames\": %d, \"total_ms\": %.3f, \"ms_per_frame\": %.4f, \"fields\": %d, \"occupied\": %lld, "
                "\"hits\": %lld}\n",
                mode, T, total, total / (T ? T : 1), fields, occupied, hits);
    return 0;
}
