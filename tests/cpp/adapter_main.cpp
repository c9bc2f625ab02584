// Drives the library exactly the way the reference's SurfelMap does (surfel_map.cpp:53, :1066-1073),
// through include/dsm_fusion_functions.hpp, with the oracle's cv::Mat / Eigen stand-ins as the caller's
// types.  Usage: adapter_main W H fx fy cx cy far near in.bin out.bin
//   in.bin : int32 ref_idx, float pose[16], int32 n_local, uint8 gray[H*W], float depth[H*W], surfel local[n_local]
//   out.bin: int32 n_local, surfel local[n_local], int32 n_new, surfel new[n_new]
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include <Eigen/Eigen> // oracle/shim
#include "dsm_fusion_functions.hpp"
#include "driver_io.hpp"

int main(int argc, char **argv)
{
    if (argc != 11) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]);
    dsm::FusionFunctions fusion_functions;
    fusion_functions.initialize(W, H, (float)atof(argv[3]), (float)atof(argv[4]), (float)atof(argv[5]), (float)atof(argv[6]),
                                (float)atof(argv[7]), (float)atof(argv[8]));
    if (fusion_functions.last_error() != DSM_OK) return fusion_functions.last_error() == DSM_E_NODEVICE ? 3 : 4;
    in_f = fopen(argv[9], "rb");
    if (!in_f) return 5;
    FrameRecord fr(W, H);
    int n_local = 0;
    std::vector<SurfelElement> local_surfels, new_surfels;
    if (!fr.get_head() || !get(n_local) || !fr.get_images() || !get_n(local_surfels, n_local)) return 5;
    fclose(in_f);
    cv::Mat image = fr.image(), dmap = fr.depth_map();
    fusion_functions.fuse_initialize_map(fr.ref, image, dmap, fr.pose, local_surfels, new_surfels);
    if (fusion_functions.last_error() != DSM_OK) return 6;
    out_f = fopen(argv[10], "wb");
    put_list(local_surfels);
    put_list(new_surfels);
    fclose(out_f);
    return 0;
}
