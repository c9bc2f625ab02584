// Drives the windowed fuse_map of include/dsm_surfel_map.hpp the way the node's synchronize_msgs would
// (surfel_map.cpp:154-161): per frame, move_add_surfels with the node's two lists, then fuse_map, with no host
// synchronisation in between; the map is read back once at the end.
// Usage: window_main W H fx fy cx cy far near in.bin out.bin
//   in.bin : int32 T, then T x { int32 ref_idx, float pose[16], int32 n_remove, int32 remove[], int32 n_add, int32 add[],
//            uint8 gray[H*W], float depth[H*W] }
//   out.bin: int32 n_pool, surfel pool[], int32 n_stored, surfel store[] (every pose's attached surfels, store order),
//            int32 n_points, point inactive_points[]
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "dsm_surfel_map.hpp"
#include "driver_io.hpp"

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
    in_f = fopen(argv[9], "rb");
    if (!in_f) return 5;
    int T = 0, n = 0;
    if (!get(T)) return 5;
    FrameRecord fr(W, H);
    std::vector<int> remove, add;
    for (int t = 0; t < T; t++)
    {
        if (!fr.get_head() || !get(n) || !get_n(remove, n) || !get(n) || !get_n(add, n) || !fr.get_images()) return 5;
        cv::Mat image = fr.image(), dmap = fr.depth_map();
        if (map.fuse_map(image, dmap, fr.pose, fr.ref, remove, add) != DSM_OK) return 6;
    }
    fclose(in_f);
    std::vector<SurfelElement> pool, store;
    std::vector<PointXYZI> points;
    if (map.download(pool) != DSM_OK) return 7;
    if (map.attached_surfels(-1, store) != DSM_OK) return 8;
    if (map.inactive_points(points) != DSM_OK) return 9;
    out_f = fopen(argv[10], "wb");
    if (!out_f) return 5;
    put_list(pool);
    put_list(store);
    put_list(points);
    fclose(out_f);
    return 0;
}
