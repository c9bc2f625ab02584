// Timing harness of tools/measure_node.py: drives dsm::SurfelMapNode (include/dsm_surfel_node.hpp) through a message
// script and times it on the host clock, with device synchronisation where a number needs it.
// Usage: measure_node W H fx fy cx cy far near drift_free_poses frames.bin script.bin
//   frames.bin: int32 K, K x { uint8 gray[H*W], float depth[H*W] }
//   script.bin: int32 T, T x { double stamp, int32 is_keyframe, int32 reference, int32 frame (of K), double pose7[7],
//               int32 n_path, double path7[n_path][7], int32 n_loops, int32 pairs[2 n_loops], int32 publish }
//   publish = 1: the frame also builds the active and inactive clouds, as the reference node publishes them per frame.
// Prints one JSON object.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "dsm_surfel_node.hpp"

typedef std::chrono::steady_clock clk;
static double ms(clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); }

int main(int argc, char **argv)
{
    if (argc != 12) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]);
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
    std::vector<dsm_point_t> active, inactive;
    double frames_ms = 0, publish_ms = 0, loop_ms = 0;
    int n_frames = 0, n_publish = 0, n_loops_ev = 0, transforms = 0;
    const clk::time_point t_all = clk::now();
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
        dsm_sync(node.context());
        const clk::time_point a = clk::now();
        int rc = node.orb_results_input(stamp, pairs.data(), n_loops, path.data(), n_path, pose, kf != 0, ref);
        if (!node.last_warp().empty())
        { // a loop closure: the orb callback and the transforms it enqueued
            dsm_sync(node.context());
            loop_ms += ms(a, clk::now());
            n_loops_ev++;
            transforms += (int)node.last_warp().size();
        }
        const clk::time_point b = clk::now();
        if (rc == DSM_OK) rc = node.image_input(stamp, gray[(size_t)k].data(), (size_t)W);
        if (rc == DSM_OK) rc = node.depth_input(stamp, depth[(size_t)k].data(), (size_t)W * 4);
        dsm_sync(node.context());
        frames_ms += ms(node.last_warp().empty() ? a : b, clk::now()); // the frame alone: pose, images, fuse
        if (rc == DSM_OK && publish)
        {
            const clk::time_point c = clk::now();
            rc = node.active_points(active);
            if (rc == DSM_OK) rc = node.inactive_points(inactive);
            publish_ms += ms(c, clk::now());
            n_publish++;
        }
        if (rc != DSM_OK) return 6;
        n_frames++;
    }
    int n_store = 0;
    if (dsm_inactive_size(node.context(), &n_store, nullptr) != DSM_OK) return 6; // also reports a deferred capacity error
    const double total_ms = ms(t_all, clk::now());
    const int reps = 20;
    const clk::time_point c = clk::now();
    for (int r = 0; r < reps; r++)
        if (node.inactive_points(inactive) != DSM_OK) return 6;
    const double inactive_ms = ms(c, clk::now()) / reps;
    std::printf("{\"frames\": %d, \"total_ms\": %.3f, \"frame_ms\": %.4f, \"publish_frames\": %d, \"publish_ms_per_frame\": %.4f, "
                "\"loop_events\": %d, \"loop_ms_per_event\": %.4f, \"transforms\": %d, \"store_surfels\": %d, "
                "\"inactive_points_ms\": %.4f}\n",
                n_frames, total_ms, frames_ms / (n_frames ? n_frames : 1), n_publish, publish_ms / (n_publish ? n_publish : 1), n_loops_ev,
                loop_ms / (n_loops_ev ? n_loops_ev : 1), transforms, n_store, inactive_ms);
    return 0;
}
