// Node-drive harness of tools/measure_checkpoint_async.py: drives dsm::SurfelMapNode through measure_node.cpp's message
// script as a node does, without synchronising per frame, and checkpoints every `every` frames.
// Usage: measure_checkpoint_async W H fx fy cx cy far near drift_free_poses frames.bin script.bin mode every dir
//   frames.bin, script.bin: as measure_node.cpp (the publish field is ignored)
//   mode 0: no checkpoint.
//   mode 1: save_state_async when `every` frames have passed since the last save, polled with wait_state_saved(false)
//           before each frame's callbacks; a save that falls due while the previous one is still written is skipped
//           (the policy of INTEGRATION.md section 4: the node never waits).
//   mode 2: the blocking save_state every `every` frames.
//   mode 3: save_state_async every `every` frames, waiting (wait_state_saved(true)) for a previous one still in flight.
// Prints one JSON object: the wall time of the whole drive (one synchronisation at its end), per frame, the checkpoints
// written, the frames on which a due save was put off because the previous one was still written (mode 1) and the
// host time spent in blocking waits (mode 3), and the host time inside the save calls themselves.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>
#include "dsm_surfel_node.hpp"

typedef std::chrono::steady_clock clk;
static double ms(clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); }

int main(int argc, char **argv)
{
    if (argc != 15) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]), mode = atoi(argv[12]), every = atoi(argv[13]);
    const std::string dir = argv[14];
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
    if ((mode == 1 || mode == 3) && node.enable_checkpoints() != DSM_OK) return 6;
    int saves = 0, skipped = 0, in_flight = 0, since = 0;
    double wait_ms = 0, call_ms = 0;
    const clk::time_point t0 = clk::now();
    for (int t = 0; t < T; t++)
    {
        double stamp, pose[7];
        int kf, ref, k, n_path, n_loops, publish;
        std::vector<double> path;
        std::vector<int> pairs;
        if (fread(&stamp, 8, 1, fs) != 1 || fread(&kf, 4, 1, fs) != 1 || fread(&ref, 4, 1, fs) != 1 || fread(&k, 4, 1, fs) != 1 ||
            fread(pose, 8, 7, fs) != 7 || fread(&n_path, 4, 1, fs) != 1)
            return 5;
        path.resize((size_t)7 * n_path + 1);
        if (fread(path.data(), 8, (size_t)7 * n_path, fs) != (size_t)7 * n_path || fread(&n_loops, 4, 1, fs) != 1) return 5;
        pairs.resize((size_t)2 * n_loops + 1);
        if (fread(pairs.data(), 4, (size_t)2 * n_loops, fs) != (size_t)2 * n_loops || fread(&publish, 4, 1, fs) != 1) return 5;
        if (in_flight)
        { // the poll of the next call
            bool fin = false;
            if (node.wait_state_saved(false, &fin) != DSM_OK) return 6;
            in_flight = !fin;
        }
        int rc = node.orb_results_input(stamp, pairs.data(), n_loops, path.data(), n_path, pose, kf != 0, ref);
        if (rc == DSM_OK) rc = node.image_input(stamp, gray[(size_t)k].data(), (size_t)W);
        if (rc == DSM_OK) rc = node.depth_input(stamp, depth[(size_t)k].data(), (size_t)W * 4);
        if (rc != DSM_OK) return 6;
        if (mode != 0 && ++since >= every)
        {
            const std::string p = dir + "/node" + std::to_string(saves % 2) + ".dsm";
            if (mode == 1 && in_flight)
            {
                skipped++; // still due on the next frame
                continue;
            }
            if (mode == 3 && in_flight)
            {
                const clk::time_point w = clk::now();
                if (node.wait_state_saved(true, nullptr) != DSM_OK) return 6;
                wait_ms += ms(w, clk::now());
            }
            const clk::time_point c = clk::now();
            rc = mode == 2 ? node.save_state(p) : node.save_state_async(p);
            call_ms += ms(c, clk::now());
            in_flight = mode != 2;
            if (rc != DSM_OK) return 6;
            saves++;
            since = 0;
        }
    }
    dsm_sync(node.context());
    const double total = ms(t0, clk::now());
    // the last checkpoint's write finishes outside the timed drive, as it would behind the node's next frames
    if (in_flight && node.wait_state_saved(true, nullptr) != DSM_OK) return 6;
    int n_store = 0;
    if (dsm_inactive_size(node.context(), &n_store, nullptr) != DSM_OK) return 6;
    std::printf("{\"frames\": %d, \"total_ms\": %.3f, \"ms_per_frame\": %.4f, \"saves\": %d, \"skipped\": %d, \"wait_ms\": %.3f, "
                "\"save_call_ms\": %.3f, \"store_surfels\": %d}\n",
                T, total, total / (T ? T : 1), saves, skipped, wait_ms, call_ms, n_store);
    return 0;
}
