// Shared by the C++ test drivers of this directory: the reference's caller types, the binary I/O of a driver's in.bin
// and out.bin, the frame record of the fuse_map drivers and the message reader of the node drivers.  Every record is
// read and written in the layout the driver's header comment gives.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <opencv2/opencv.hpp> // oracle/shim

struct SurfelElement // reference elements.h:22-31
{
    float px, py, pz, nx, ny, nz, size, color, weight;
    int update_times, last_update;
};
struct PointXYZI // the four named fields of pcl::PointXYZI
{
    float x, y, z, intensity;
};
struct Pose4f // Eigen::Matrix4f: a column-major .data()
{
    float m[16];
    float *data() { return m; }
};

static FILE *in_f, *out_f; // the driver's in.bin and out.bin

template <class T>
static bool get(T &v)
{
    return fread(&v, sizeof(T), 1, in_f) == 1;
}
template <class T>
static bool get_n(std::vector<T> &v, int n)
{
    if (n < 0) return false;
    v.resize((size_t)n);
    return n == 0 || fread(v.data(), sizeof(T), (size_t)n, in_f) == (size_t)n;
}
template <class T>
static void put(const T &v)
{
    fwrite(&v, sizeof(T), 1, out_f);
}
// int32 n, then n records
template <class T>
static void put_n(const T *p, int n)
{
    put(n);
    if (n > 0) fwrite(p, sizeof(T), (size_t)n, out_f);
}
template <class T>
static void put_list(const std::vector<T> &v)
{
    put_n(v.data(), (int)v.size());
}

// one frame of the fuse_map drivers: int32 ref_idx, float pose[16], then (after what the driver reads in between)
// uint8 gray[H*W], float depth[H*W]; image() and depth_map() are cv::Mat views of the two planes
struct FrameRecord
{
    int W, H, ref;
    Pose4f pose;
    std::vector<unsigned char> gray;
    std::vector<float> depth;
    FrameRecord(int w, int h) : W(w), H(h), ref(0) {}
    bool get_head() { return get(ref) && get(pose); }
    bool get_images() { return get_n(gray, W * H) && get_n(depth, W * H); }
    cv::Mat image() { return cv::Mat(H, W, CV_8UC1, gray.data(), (size_t)W); }
    cv::Mat depth_map() { return cv::Mat(H, W, CV_32FC1, depth.data(), (size_t)W * 4); }
};

// The orb / image / depth messages of the node drivers' script (node_main.cpp), each handed to the node as it is read:
//   0 orb    double stamp, int32 is_keyframe, int32 reference_index, double pose7[7], int32 n_path, double path7[n_path][7],
//            int32 n_loops, int32 pairs[2 n_loops]
//   1 image  double stamp, uint8 gray[H*W]
//   2 depth  double stamp, float depth[H*W]
struct NodeMessages
{
    std::vector<uint8_t> gray;
    std::vector<float> depth;
    std::vector<double> path;
    std::vector<int> pairs;
    // false for a malformed message or another type; else rc is the node's code
    template <class Node>
    bool feed(Node &node, int type, int W, int H, int &rc)
    {
        double stamp = 0;
        if (type == 0)
        {
            int kf = 0, ref = 0, n_path = 0, n_loops = 0;
            double pose[7];
            if (!get(stamp) || !get(kf) || !get(ref) || fread(pose, 8, 7, in_f) != 7 || !get(n_path) || !get_n(path, 7 * n_path) ||
                !get(n_loops) || !get_n(pairs, 2 * n_loops))
                return false;
            rc = node.orb_results_input(stamp, pairs.data(), n_loops, path.data(), n_path, pose, kf != 0, ref);
        }
        else if (type == 1)
        {
            if (!get(stamp) || !get_n(gray, W * H)) return false;
            rc = node.image_input(stamp, gray.data(), (size_t)W);
        }
        else if (type == 2)
        {
            if (!get(stamp) || !get_n(depth, W * H)) return false;
            rc = node.depth_input(stamp, depth.data(), (size_t)W * 4);
        }
        else
            return false;
        return true;
    }
};
