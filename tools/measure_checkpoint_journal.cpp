// Node-drive harness of tools/measure_checkpoint_journal.py: drives dsm::SurfelMapNode through measure_node.cpp's message
// script as a node does, without synchronising per frame, and checkpoints once `every` frames have passed, skipping a
// due save while the previous one is still written (the policy of INTEGRATION.md section 4).
// Usage: measure_checkpoint_journal W H fx fy cx cy far near drift_free_poses frames.bin script.bin mode every dir
//   frames.bin, script.bin: as measure_node.cpp (the publish field is ignored)
//   mode 0: no checkpoint.  mode 1: save_state_async (a whole file each time).  mode 2: save_state_incremental.
// Prints one JSON object: the wall time of the drive (one synchronisation at its end) per frame, the saves, the saves
// put off, and for every finished save the bytes it wrote (the file for a whole file or a base, the record otherwise)
// and whether it was a base.
#include <sys/stat.h>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>
#include "dsm_surfel_node.hpp"

typedef std::chrono::steady_clock clk;
static double ms(clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); }
static long long size_of(const std::string &p)
{
    struct stat st;
    return stat(p.c_str(), &st) == 0 ? (long long)st.st_size : -1;
}

int main(int argc, char **argv)
{
    if (argc != 15) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]), mode = atoi(argv[12]), every = atoi(argv[13]);
    const std::string dir = argv[14], path = dir + "/node_journal.dsm";
    FILE *ff = fopen(argv[10], "rb"), *fs = fopen(argv[11], "rb");
    if (!ff || !fs || every < 1) return 5;
    int K = 0, T = 0;
    if (fread(&K, 4, 1, ff) != 1 || fread(&T, 4, 1, fs) != 1) return 5;
    std::vector<std::vector<uint8_t> > gray((size_t)K, std::vector<uint8_t>((size_t)W * H));
    std::vector<std::vector<float> > depth((size_t)K, std::vector<float>((size_t)W * H));
    for (int k = 0; k < K; k++)
        if (fread(gray[k].data(), 1, gray[k].size(), ff) != gray[k].size() || fread(depth[k].data(), 4, depth[k].size(), ff) != depth[k].size())
            return 5;
    dsm::SurfelMapNode node(W, H, atof(argv[3]), atof(argv[4]), atof(argv[5]), atof(argv[6]), atof(argv[7]), atof(argv[8]), atoi(argv[9]), 0);
    if (node.last_error() != DSM_OK) return node.last_error() == DSM_E_NODEVICE ? 3 : 4;
    if (mode != 0 && node.enable_checkpoints() != DSM_OK) return 6;
    int saves = 0, skipped = 0, in_flight = 0, since = 0;
    long long journal = 0;
    std::vector<long long> bytes;
    std::vector<int> base;
    auto finished = [&]() { // the save just retired: what it wrote
        const long long j = size_of(path + ".journal");
        const bool b = mode == 1 || j < journal || j == 32;
        bytes.push_back(b ? size_of(path) : j - journal);
        base.push_back(b ? 1 : 0);
        journal = j;
    };
    const clk::time_point t0 = clk::now();
    for (int t = 0; t < T; t++)
    {
        double stamp, pose[7];
        int kf, ref, k, n_path, n_loops, publish;
        std::vector<double> pth;
        std::vector<int> pairs;
        if (fread(&stamp, 8, 1, fs) != 1 || fread(&kf, 4, 1, fs) != 1 || fread(&ref, 4, 1, fs) != 1 || fread(&k, 4, 1, fs) != 1 ||
            fread(pose, 8, 7, fs) != 7 || fread(&n_path, 4, 1, fs) != 1)
            return 5;
        pth.resize((size_t)7 * n_path + 1);
        if (fread(pth.data(), 8, (size_t)7 * n_path, fs) != (size_t)7 * n_path || fread(&n_loops, 4, 1, fs) != 1) return 5;
        pairs.resize((size_t)2 * n_loops + 1);
        if (fread(pairs.data(), 4, (size_t)2 * n_loops, fs) != (size_t)2 * n_loops || fread(&publish, 4, 1, fs) != 1) return 5;
        if (in_flight)
        { // the poll of the next call
            bool fin = false;
            if (node.wait_state_saved(false, &fin) != DSM_OK) return 6;
            in_flight = !fin;
            if (fin) finished();
        }
        int rc = node.orb_results_input(stamp, pairs.data(), n_loops, pth.data(), n_path, pose, kf != 0, ref);
        if (rc == DSM_OK) rc = node.image_input(stamp, gray[(size_t)k].data(), (size_t)W);
        if (rc == DSM_OK) rc = node.depth_input(stamp, depth[(size_t)k].data(), (size_t)W * 4);
        if (rc != DSM_OK) return 6;
        if (mode != 0 && ++since >= every)
        {
            if (in_flight)
            {
                skipped++; // still due on the next frame
                continue;
            }
            rc = mode == 1 ? node.save_state_async(path) : node.save_state_incremental(path);
            if (rc != DSM_OK) return 6;
            in_flight = 1;
            saves++;
            since = 0;
        }
    }
    dsm_sync(node.context());
    const double total = ms(t0, clk::now());
    if (in_flight)
    {
        if (node.wait_state_saved(true, nullptr) != DSM_OK) return 6;
        finished();
    }
    std::printf("{\"frames\": %d, \"total_ms\": %.3f, \"ms_per_frame\": %.4f, \"saves\": %d, \"skipped\": %d, \"bytes\": [", T, total,
                total / (T ? T : 1), saves, skipped);
    for (size_t i = 0; i < bytes.size(); i++) std::printf("%s%lld", i ? ", " : "", bytes[i]);
    std::printf("], \"base\": [");
    for (size_t i = 0; i < base.size(); i++) std::printf("%s%d", i ? ", " : "", base[i]);
    std::printf("]}\n");
    return 0;
}
