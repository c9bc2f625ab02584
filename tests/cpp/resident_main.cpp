// Drives include/dsm_surfel_map.hpp the way a SurfelMap with a GPU-resident local_surfels would (INTEGRATION.md §4):
// a short stream through fuse_map, then the loop-closure warp, one move_add_surfels round trip, the cloud export
// and the two save files.  Caller types are the oracle's cv::Mat stand-in and plain PODs.
// Usage: resident_main W H fx fy cx cy far near in.bin out.bin cloud.pcd mesh.ply
//   in.bin : int32 T, then T x { int32 ref_idx, float pose[16], uint8 gray[H*W], float depth[H*W] },
//            float warp[16], int32 retire_keyframe
//   out.bin: int32 n_pool_after_stream, surfel pool[], int32 n_retired, surfel retired[], int32 n_final, surfel final[],
//            int32 n_points, point points[]
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "dsm_surfel_map.hpp"
#include "driver_io.hpp"

int main(int argc, char **argv)
{
    if (argc != 13) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]);
    dsm::ResidentSurfelPool map;
    map.set_device(0, 200000);
    if (map.initialize(W, H, (float)atof(argv[3]), (float)atof(argv[4]), (float)atof(argv[5]), (float)atof(argv[6]), (float)atof(argv[7]),
                       (float)atof(argv[8])) != DSM_OK)
        return map.last_error() == DSM_E_NODEVICE ? 3 : 4;
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
    Pose4f warp;
    int retire_kf = 0;
    if (!get(warp) || !get(retire_kf)) return 5;
    fclose(in_f);
    std::vector<SurfelElement> pool, retired, final_pool;
    std::vector<PointXYZI> points, no_inactive;
    if (map.download(pool) != DSM_OK) return 7;
    if (map.warp_active_surfels(warp) != DSM_OK) return 8;
    if (map.retire_surfels(retire_kf, retired) != DSM_OK) return 9;
    if (map.add_surfels(retired) != DSM_OK) return 10; // the pose comes straight back into the drift-free set
    if (map.active_points(points, 5) != DSM_OK) return 11;
    if (map.save_cloud(argv[11], no_inactive) != DSM_OK) return 12;
    if (map.save_mesh(argv[12], retired) != DSM_OK) return 13;
    if (map.download(final_pool) != DSM_OK) return 14;
    out_f = fopen(argv[10], "wb");
    if (!out_f) return 5;
    put_list(pool);
    put_list(retired);
    put_list(final_pool);
    put_list(points);
    fclose(out_f);
    return 0;
}
