// dsm_fusion_functions.hpp — header-only C++ adapter that gives the H100 library the public surface
// of the reference's `class FusionFunctions` (surfel_fusion/src/fusion_functions.h:84-94), so that
// `SurfelMap` (surfel_fusion/src/surfel_map.h:118, surfel_map.cpp:53 and :1066-1073) can hold a
// `dsm::FusionFunctions` instead and call it unchanged:
//
//     fusion_functions.initialize(cam_width, cam_height, cam_fx, cam_fy, cam_cx, cam_cy, far_dist, near_dist);
//     fusion_functions.fuse_initialize_map(reference_index, image, depth, pose_input, local_surfels, new_surfels);
//
// The two methods are templates over the image / pose types so the header needs neither OpenCV nor
// Eigen: any `Mat` with `.data`, `.step` (bytes per row), `.rows`, `.cols` (cv::Mat) and any 4x4 float
// matrix with a column-major `.data()` (Eigen::Matrix4f) work.  `SurfelElement` is the reference's
// own struct (elements.h:22-31); it is layout-compatible with dsm_surfel_t and checked below.
//
// Error behaviour: the reference's methods return void and never throw; a CUDA failure here cannot be
// ignored silently, so it is reported on stderr and `last_error()` keeps the code (0 = OK).  There is
// no CPU fallback.
#pragma once
#include <vector>
#include "dsm_context.hpp"

namespace dsm
{
class FusionFunctions
{
  public:
    FusionFunctions() : ctx_("dsm::FusionFunctions"), device_(0), capacity_(1 << 21) {}

    // optional, before initialize(): CUDA ordinal and the largest local_surfels.size() to expect
    void set_device(int device, int max_local_surfels = 1 << 21)
    {
        device_ = device;
        capacity_ = max_local_surfels;
    }

    // reference: FusionFunctions::initialize (fusion_functions.cpp:7-28)
    void initialize(int _width, int _height, float _fx, float _fy, float _cx, float _cy, float _fuse_far, float _fuse_near)
    {
        const dsm_params p = detail::Context::params(_width, _height, _fx, _fy, _cx, _cy, _fuse_far, _fuse_near, 1, capacity_);
        ctx_.open("initialize", p, device_, false, nullptr, nullptr);
    }

    // reference: FusionFunctions::fuse_initialize_map (fusion_functions.cpp:30-83).
    // image: CV_8UC1, depth: CV_32FC1 (metres), pose: T_world<-cam; local_surfels updated in place and
    // never resized; new_surfels cleared and filled in seed-index order.
    template <class Mat, class Mat4f, class Surfel>
    void fuse_initialize_map(int reference_frame_index, Mat &input_image, Mat &input_depth, Mat4f &pose,
                             std::vector<Surfel> &local_surfels, std::vector<Surfel> &new_surfels)
    {
        static_assert(sizeof(Surfel) == sizeof(dsm_surfel_t), "SurfelElement must be the 44-byte reference POD");
        new_surfels.clear();
        if (!ctx_.ready("fuse_initialize_map")) return;
        const int S = dsm_num_seeds(ctx_.ctx);
        new_surfels.resize((size_t)S);
        int n_new = 0;
        const int rc = dsm_fuse_frame(ctx_.ctx, reference_frame_index,
                                      reinterpret_cast<const uint8_t *>(input_image.data), (size_t)input_image.step,
                                      reinterpret_cast<const float *>(input_depth.data), (size_t)input_depth.step,
                                      pose.data(),
                                      reinterpret_cast<dsm_surfel_t *>(local_surfels.data()), (int)local_surfels.size(),
                                      reinterpret_cast<dsm_surfel_t *>(new_surfels.data()), S, &n_new);
        if (ctx_.done(rc, "fuse_initialize_map") != DSM_OK) n_new = 0;
        new_surfels.resize((size_t)n_new);
    }

    // reference: FusionFunctions::debug_show (fusion_functions.cpp:977-1006) of the frame of the last
    // fuse_initialize_map, written into `image` instead of cv::imshow: height rows of width x 3 bytes at the
    // image's row pitch.  Mat: any type with .data and .step, allocated by the caller (cv::Mat of CV_8UC3).
    // Returns the C ABI code (also kept in last_error()).
    template <class Mat>
    int superpixel_image(Mat &image)
    {
        return ctx_.run("superpixel_image", [&] { return detail::superpixel_image(ctx_, image); });
    }

    int last_error() const { return ctx_.err; }
    dsm_ctx *context() { return ctx_.ctx; }

  private:
    detail::Context ctx_;
    int device_;
    int capacity_;
};
} // namespace dsm
