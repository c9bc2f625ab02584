// Drives the superpixel normal image (FusionFunctions::debug_show, fusion_functions.cpp:977-1006) through both C++
// helpers: dsm::ResidentSurfelPool::superpixel_image after each frame of a short fuse_map stream, and
// dsm::FusionFunctions::superpixel_image after fuse_initialize_map of the last frame.  Caller images are the oracle's
// cv::Mat stand-in: the resident pool writes into a Mat view with a padded row pitch, the adapter into an owned CV_8UC3.
// Usage: superpixel_image_main W H fx fy cx cy far near in.bin out.bin
//   in.bin : int32 T, then T x { int32 ref_idx, float pose[16], uint8 gray[H*W], float depth[H*W] }
//   out.bin: T x uint8 resident[H][W*3 + 5] (pitched, the 5 padding bytes of each row as the caller filled them),
//            uint8 adapter[H][W*3]
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "dsm_fusion_functions.hpp"
#include "dsm_surfel_map.hpp"
#include "driver_io.hpp"

int main(int argc, char **argv)
{
    if (argc != 11) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]);
    const float fx = (float)atof(argv[3]), fy = (float)atof(argv[4]), cx = (float)atof(argv[5]), cy = (float)atof(argv[6]);
    const float fa = (float)atof(argv[7]), ne = (float)atof(argv[8]);
    dsm::ResidentSurfelPool map;
    map.set_device(0, 200000);
    if (map.initialize(W, H, fx, fy, cx, cy, fa, ne) != DSM_OK) return map.last_error() == DSM_E_NODEVICE ? 3 : 4;
    in_f = fopen(argv[9], "rb");
    if (!in_f) return 5;
    int T = 0;
    if (!get(T) || T < 1) return 5;
    const size_t pitch = (size_t)W * 3 + 5;
    out_f = fopen(argv[10], "wb");
    if (!out_f) return 5;
    std::vector<unsigned char> shown(pitch * H);
    FrameRecord fr(W, H);
    for (int t = 0; t < T; t++)
    {
        if (!fr.get_head() || !fr.get_images()) return 5;
        cv::Mat image = fr.image(), dmap = fr.depth_map();
        if (map.fuse_map(image, dmap, fr.pose, fr.ref) != DSM_OK) return 6;
        for (size_t i = 0; i < shown.size(); i++) shown[i] = (unsigned char)(0xA5 ^ (i * 7));
        cv::Mat sp(H, W, CV_8UC3, shown.data(), pitch);
        if (map.superpixel_image(sp) != DSM_OK) return 7;
        fwrite(shown.data(), 1, shown.size(), out_f);
    }
    fclose(in_f);
    dsm::FusionFunctions ff;
    ff.set_device(0, 1 << 16);
    ff.initialize(W, H, fx, fy, cx, cy, fa, ne);
    if (ff.last_error() != DSM_OK) return 8;
    cv::Mat image = fr.image(), dmap = fr.depth_map();
    std::vector<SurfelElement> local, fresh;
    ff.fuse_initialize_map(fr.ref, image, dmap, fr.pose, local, fresh);
    if (ff.last_error() != DSM_OK) return 8;
    cv::Mat out(H, W, CV_8UC3);
    if (ff.superpixel_image(out) != DSM_OK) return 9;
    fwrite(out.data, 1, out.step * (size_t)H, out_f);
    fclose(out_f);
    return 0;
}
