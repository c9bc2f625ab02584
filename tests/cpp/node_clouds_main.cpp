// Drives the two cloud publishers of include/dsm_surfel_map.hpp that need the device-resident inactive store and the
// fused frame: a short stream through fuse_map, two keyframes retired into the store, then neighbor_points() over a
// BFS-shaped pose list and raw_points() of the last frame.  Caller types are the oracle's cv::Mat stand-in and PODs.
// Usage: node_clouds_main W H fx fy cx cy far near in.bin out.bin
//   in.bin : int32 T, then T x { int32 ref_idx, float pose[16], uint8 gray[H*W], float depth[H*W] },
//            int32 retire[2], int32 n_list, int32 list[n_list], double pose7[7]
//   out.bin: int32 n, point neighbor[n]; int32 n, point active1[n]; int32 n, point inactive[n]; int32 n_first_retired;
//            int32 n, point raw[n]
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <opencv2/opencv.hpp> // oracle/shim
#include "dsm_surfel_map.hpp"

struct PointXYZI // the four named fields of pcl::PointXYZI
{
    float x, y, z, intensity;
};
struct Pose4f
{
    float m[16];
    float *data() { return m; }
};
struct RosPose // the members of geometry_msgs::Pose that raw_points reads
{
    struct
    {
        double x, y, z;
    } position;
    struct
    {
        double x, y, z, w;
    } orientation;
};

static void put(FILE *f, const std::vector<PointXYZI> &v)
{
    const int n = (int)v.size();
    fwrite(&n, 4, 1, f);
    if (n) fwrite(v.data(), sizeof(PointXYZI), (size_t)n, f);
}

int main(int argc, char **argv)
{
    if (argc != 11) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]);
    dsm::ResidentSurfelPool map;
    map.set_device(0, 200000);
    if (map.initialize(W, H, (float)atof(argv[3]), (float)atof(argv[4]), (float)atof(argv[5]), (float)atof(argv[6]), (float)atof(argv[7]),
                       (float)atof(argv[8])) != DSM_OK)
        return map.last_error() == DSM_E_NODEVICE ? 3 : 4;
    if (map.reserve_inactive(200000) != DSM_OK) return 4;
    FILE *f = fopen(argv[9], "rb");
    if (!f) return 5;
    int T = 0;
    if (fread(&T, 4, 1, f) != 1) return 5;
    std::vector<unsigned char> gray((size_t)W * H);
    std::vector<float> depth((size_t)W * H);
    for (int t = 0; t < T; t++)
    {
        int ref = 0;
        Pose4f pose;
        if (fread(&ref, 4, 1, f) != 1 || fread(pose.m, 4, 16, f) != 16) return 5;
        if (fread(gray.data(), 1, gray.size(), f) != gray.size() || fread(depth.data(), 4, depth.size(), f) != depth.size()) return 5;
        cv::Mat image(H, W, CV_8UC1, gray.data(), (size_t)W), dmap(H, W, CV_32FC1, depth.data(), (size_t)W * 4);
        if (map.fuse_map(image, dmap, pose, ref) != DSM_OK) return 6;
    }
    int retire[2] = {0, 0}, n_list = 0;
    if (fread(retire, 4, 2, f) != 2 || fread(&n_list, 4, 1, f) != 1 || n_list < 0) return 5;
    std::vector<int> list((size_t)n_list);
    double p7[7];
    if ((n_list && fread(list.data(), 4, (size_t)n_list, f) != (size_t)n_list) || fread(p7, 8, 7, f) != 7) return 5;
    fclose(f);
    RosPose pose;
    pose.position.x = p7[0], pose.position.y = p7[1], pose.position.z = p7[2];
    pose.orientation.x = p7[3], pose.orientation.y = p7[4], pose.orientation.z = p7[5], pose.orientation.w = p7[6];
    const int n_first = map.retire_surfels_resident(retire[0]);
    if (n_first < 0 || map.retire_surfels_resident(retire[1]) < 0) return 7;
    std::vector<PointXYZI> neighbor, active1, inactive, raw;
    if (map.neighbor_points(neighbor, list) != DSM_OK) return 8;
    if (map.active_points(active1, 1) != DSM_OK) return 9;
    if (map.inactive_points(inactive) != DSM_OK) return 10;
    if (map.raw_points(raw, pose) != DSM_OK) return 11;
    f = fopen(argv[10], "wb");
    if (!f) return 5;
    put(f, neighbor);
    put(f, active1);
    put(f, inactive);
    fwrite(&n_first, 4, 1, f);
    put(f, raw);
    fclose(f);
    return 0;
}
