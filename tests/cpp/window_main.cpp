// Drives the windowed fuse_map of include/dsm_surfel_map.hpp the way the node's synchronize_msgs would
// (surfel_map.cpp:154-161): per frame, move_add_surfels with the node's two lists, then fuse_map, with no host
// synchronisation in between; the map is read back once at the end.
// Usage: window_main W H fx fy cx cy far near in.bin out.bin
//   in.bin : int32 T, then T x { int32 ref_idx, float pose[16], int32 n_remove, int32 remove[], int32 n_add, int32 add[],
//            uint8 gray[H*W], float depth[H*W] }
//   out.bin: int32 n_pool, surfel pool[], int32 n_stored, surfel store[] (every pose's attached surfels, store order),
//            int32 n_points, point inactive_points[]
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <opencv2/opencv.hpp> // oracle/shim
#include "dsm_surfel_map.hpp"

struct SurfelElement // reference elements.h:22-31
{
    float px, py, pz, nx, ny, nz, size, color, weight;
    int update_times, last_update;
};
struct PointXYZI // the four named fields of pcl::PointXYZI
{
    float x, y, z, intensity;
};
struct Pose4f
{
    float m[16];
    float *data() { return m; }
};

template <class T>
static void put(FILE *f, const std::vector<T> &v)
{
    const int n = (int)v.size();
    fwrite(&n, 4, 1, f);
    if (n) fwrite(v.data(), sizeof(T), (size_t)n, f);
}
static bool get_list(FILE *f, std::vector<int> &v)
{
    int n = 0;
    if (fread(&n, 4, 1, f) != 1 || n < 0) return false;
    v.resize((size_t)n);
    return n == 0 || fread(v.data(), 4, (size_t)n, f) == (size_t)n;
}

int main(int argc, char **argv)
{
    if (argc != 11) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]);
    dsm::ResidentSurfelPool map;
    map.set_device(0, 400000);
    if (map.initialize(W, H, (float)atof(argv[3]), (float)atof(argv[4]), (float)atof(argv[5]), (float)atof(argv[6]), (float)atof(argv[7]),
                       (float)atof(argv[8])) != DSM_OK)
        return map.last_error() == DSM_E_NODEVICE ? 3 : 4;
    if (map.reserve_inactive(400000) != DSM_OK) return 4;
    FILE *f = fopen(argv[9], "rb");
    if (!f) return 5;
    int T = 0;
    if (fread(&T, 4, 1, f) != 1) return 5;
    std::vector<unsigned char> gray((size_t)W * H);
    std::vector<float> depth((size_t)W * H);
    std::vector<int> remove, add;
    for (int t = 0; t < T; t++)
    {
        int ref = 0;
        Pose4f pose;
        if (fread(&ref, 4, 1, f) != 1 || fread(pose.m, 4, 16, f) != 16 || !get_list(f, remove) || !get_list(f, add)) return 5;
        if (fread(gray.data(), 1, gray.size(), f) != gray.size() || fread(depth.data(), 4, depth.size(), f) != depth.size()) return 5;
        cv::Mat image(H, W, CV_8UC1, gray.data(), (size_t)W), dmap(H, W, CV_32FC1, depth.data(), (size_t)W * 4);
        if (map.fuse_map(image, dmap, pose, ref, remove, add) != DSM_OK) return 6;
    }
    fclose(f);
    std::vector<SurfelElement> pool, store;
    std::vector<PointXYZI> points;
    if (map.download(pool) != DSM_OK) return 7;
    int n = 0, got = 0;
    if (dsm_inactive_size(map.context(), &n, nullptr) != DSM_OK) return 8;
    store.resize((size_t)n);
    if (dsm_inactive_download(map.context(), -1, reinterpret_cast<dsm_surfel_t *>(store.data()), n, &got) != DSM_OK) return 8;
    if (map.inactive_points(points) != DSM_OK) return 9;
    f = fopen(argv[10], "wb");
    if (!f) return 5;
    put(f, pool);
    put(f, store);
    put(f, points);
    fclose(f);
    return 0;
}
