// Drives the two cloud publishers of include/dsm_surfel_map.hpp that need the device-resident inactive store and the
// fused frame: a short stream through fuse_map, two keyframes retired into the store, then neighbor_points() over a
// BFS-shaped pose list and raw_points() of the last frame.  Caller types are the oracle's cv::Mat stand-in and PODs.
// Usage: node_clouds_main W H fx fy cx cy far near in.bin out.bin
//   in.bin : int32 T, then T x { int32 ref_idx, float pose[16], uint8 gray[H*W], float depth[H*W] },
//            int32 retire[2], int32 n_list, int32 list[n_list], double pose7[7]
//   out.bin: int32 n, point neighbor[n]; int32 n, point active1[n]; int32 n, point inactive[n]; int32 n_first_retired;
//            int32 n, point raw[n]
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "dsm_surfel_map.hpp"
#include "driver_io.hpp"

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
    in_f = fopen(argv[9], "rb");
    if (!in_f) return 5;
    int T = 0;
    if (!get(T)) return 5;
    FrameRecord fr(W, H);
    for (int t = 0; t < T; t++)
    {
        if (!fr.get_head() || !fr.get_images()) return 5;
        cv::Mat image = fr.image(), dmap = fr.depth_map();
        if (map.fuse_map(image, dmap, fr.pose, fr.ref) != DSM_OK) return 6;
    }
    int retire[2] = {0, 0}, n_list = 0;
    std::vector<int> list;
    double p7[7];
    if (!get(retire) || !get(n_list) || !get_n(list, n_list) || !get(p7)) return 5;
    fclose(in_f);
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
    out_f = fopen(argv[10], "wb");
    if (!out_f) return 5;
    put_list(neighbor);
    put_list(active1);
    put_list(inactive);
    put(n_first);
    put_list(raw);
    fclose(out_f);
    return 0;
}
