// Shared by the timing harnesses tools/measure_*.cpp: the drive they read, written by tools/measure_drive.py, the node
// built from their argument prefix, and the host clock.  Every harness takes W H fx fy cx cy far near drift_free_poses
// frames.bin script.bin as argv[1..11]:
//   frames.bin: int32 K, K x { uint8 gray[H*W], float depth[H*W] }
//   script.bin: int32 T, T x { double stamp, int32 is_keyframe, int32 reference, int32 frame (of K), double pose7[7],
//               int32 n_path, double path7[n_path][7], int32 n_loops, int32 pairs[2 n_loops], int32 publish }
// The whole drive is read before a harness starts its clock.
#pragma once
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "dsm_surfel_node.hpp"

typedef std::chrono::steady_clock clk;
static inline double ms(clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); }

struct DriveMsg
{
    double stamp, pose[7];
    int kf, ref, k, n_path, n_loops, publish;
    std::vector<double> path;
    std::vector<int> pairs;
    int orb(dsm::SurfelMapNode &node) const
    {
        return node.orb_results_input(stamp, pairs.data(), n_loops, path.data(), n_path, pose, kf != 0, ref);
    }
};

struct Drive
{
    std::vector<std::vector<uint8_t> > gray; // per frame of frames.bin
    std::vector<std::vector<float> > depth;
    std::vector<DriveMsg> msgs; // per message of script.bin
    // argv[10] and argv[11]; false (exit code 5) when either file is missing or short
    bool load(char **argv)
    {
        const size_t n = (size_t)atoi(argv[1]) * atoi(argv[2]);
        FILE *ff = fopen(argv[10], "rb"), *fs = fopen(argv[11], "rb");
        const bool ok = ff && fs && load_frames(ff, n) && load_script(fs);
        if (ff) fclose(ff);
        if (fs) fclose(fs);
        return ok;
    }
    // the image and depth callbacks of message m's frame
    int images(dsm::SurfelMapNode &node, const DriveMsg &m, int W) const
    {
        int rc = node.image_input(m.stamp, gray[(size_t)m.k].data(), (size_t)W);
        if (rc == DSM_OK) rc = node.depth_input(m.stamp, depth[(size_t)m.k].data(), (size_t)W * 4);
        return rc;
    }

  private:
    bool load_frames(FILE *f, size_t n)
    {
        int K = 0;
        if (fread(&K, 4, 1, f) != 1 || K < 0) return false;
        gray.assign((size_t)K, std::vector<uint8_t>(n));
        depth.assign((size_t)K, std::vector<float>(n));
        for (int k = 0; k < K; k++)
            if (fread(gray[k].data(), 1, n, f) != n || fread(depth[k].data(), 4, n, f) != n) return false;
        return true;
    }
    bool load_script(FILE *f)
    {
        int T = 0;
        if (fread(&T, 4, 1, f) != 1 || T < 0) return false;
        msgs.resize((size_t)T);
        for (int t = 0; t < T; t++)
        {
            DriveMsg &m = msgs[(size_t)t];
            if (fread(&m.stamp, 8, 1, f) != 1 || fread(&m.kf, 4, 1, f) != 1 || fread(&m.ref, 4, 1, f) != 1 || fread(&m.k, 4, 1, f) != 1 ||
                fread(m.pose, 8, 7, f) != 7 || fread(&m.n_path, 4, 1, f) != 1 || m.n_path < 0)
                return false;
            m.path.resize((size_t)7 * m.n_path + 1);
            if (fread(m.path.data(), 8, (size_t)7 * m.n_path, f) != (size_t)7 * m.n_path || fread(&m.n_loops, 4, 1, f) != 1 || m.n_loops < 0)
                return false;
            m.pairs.resize((size_t)2 * m.n_loops + 1);
            if (fread(m.pairs.data(), 4, (size_t)2 * m.n_loops, f) != (size_t)2 * m.n_loops || fread(&m.publish, 4, 1, f) != 1) return false;
            if (m.k < 0 || m.k >= (int)gray.size()) return false;
        }
        return true;
    }
};

// a node on device 0 of the argument prefix W H fx fy cx cy far near drift_free_poses (argv[1..9])
struct DriveNode : dsm::SurfelMapNode
{
    explicit DriveNode(char **argv)
        : dsm::SurfelMapNode(atoi(argv[1]), atoi(argv[2]), atof(argv[3]), atof(argv[4]), atof(argv[5]), atof(argv[6]), atof(argv[7]),
                             atof(argv[8]), atoi(argv[9]), 0)
    {
    }
    // 0 when the node is ready, else the exit code: 3 without a usable GPU (the library has no CPU fallback), 4 for any other
    int setup_code() { return last_error() == DSM_OK ? 0 : last_error() == DSM_E_NODEVICE ? 3 : 4; }
};
