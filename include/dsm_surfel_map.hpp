// dsm_surfel_map.hpp — header-only C++ helper for the SECOND integration step of INTEGRATION.md §4: the
// `local_surfels` of the reference's SurfelMap kept on the GPU between frames.  Each method has the name and
// the role of the SurfelMap member whose `local_surfels` part it replaces (surfel_fusion/src/surfel_map.cpp);
// everything else in those members (pose graph, drift-free BFS, ROS publishing, and the inactive cloud unless the
// device-resident store below is used) stays in SurfelMap unchanged.  Like dsm_fusion_functions.hpp it needs neither
// OpenCV, Eigen, PCL nor ROS: images are any type with .data / .step (cv::Mat), matrices any type with a column-major
// .data() (Eigen::Matrix4f), poses any type with position.{x,y,z} / orientation.{x,y,z,w} (geometry_msgs::Pose), points
// any 16-byte {x, y, z, intensity} POD or pcl::PointXYZI (converted field by field).
//
//   SurfelMap member (file:line)                          here
//   ----------------------------------------------------  -----------------------------------------------
//   ctor: fusion_functions.initialize(...)     (:53)      initialize(w, h, fx, fy, cx, cy, far, near)
//   fuse_map(image, depth, pose, ref)     (:1060-1113)    fuse_map(image, depth, pose, reference_index)
//   warp_surfels(), active part            (:805-819)     warp_active_surfels(warp_pose)
//   move_add_surfels(), removal loop      (:1479-1497)    retire_surfels(inactive_index, attached_surfels)
//   move_add_surfels(), insertion         (:1583-1587)    add_surfels(attached_surfels)
//   publish_active/all_pointcloud, local  (:1398-1454)    active_points(points, 5)
//   publish_neighbor_pointcloud           (:1283-1383)    neighbor_points(points, neighbor_indexs)
//   publish_raw_pointcloud                (:1115-1151)    raw_points(points, pose)
//   FusionFunctions::debug_show (fusion_functions.cpp:977-1006)   superpixel_image(image)
//   save_cloud                            (:1153-1173)    save_cloud(name, inactive_points)
//   save_mesh                             (:1229-1280)    save_mesh(name, attached_surfels_of_all_poses)
//   local_surfels.size()                                  size()
//
// Errors: the reference's members return void; here every method returns the C ABI code (0 = OK) and keeps it
// in last_error().  There is no CPU fallback.
#pragma once
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "dsm.h"

namespace dsm
{
class ResidentSurfelPool
{
  public:
    ResidentSurfelPool() : ctx_(nullptr), err_(0), device_(0), capacity_(1 << 21), width_(0), height_(0) {}
    ~ResidentSurfelPool() { dsm_destroy(ctx_); }
    ResidentSurfelPool(const ResidentSurfelPool &) = delete;
    ResidentSurfelPool &operator=(const ResidentSurfelPool &) = delete;

    void set_device(int device, int max_local_surfels = 1 << 21)
    {
        device_ = device;
        capacity_ = max_local_surfels;
    }

    int initialize(int width, int height, float fx, float fy, float cx, float cy, float fuse_far, float fuse_near)
    {
        dsm_destroy(ctx_);
        ctx_ = nullptr;
        dsm_params p;
        std::memset(&p, 0, sizeof(p));
        p.width = width, p.height = height;
        p.fx = fx, p.fy = fy, p.cx = cx, p.cy = cy;
        p.fuse_far = fuse_far, p.fuse_near = fuse_near;
        p.max_batch = 2; // two frame slots: the copy of frame t+1 overlaps the kernels of frame t
        p.max_local_surfels = capacity_;
        width_ = width, height_ = height;
        err_ = dsm_create(&p, device_, nullptr, &ctx_);
        if (err_ == DSM_OK) err_ = dsm_pool_upload(ctx_, nullptr, 0); // local_surfels starts empty
        return report("initialize");
    }

    // SurfelMap::fuse_map: the hot-path call plus the post-step (slot recycling as the reference), all on the device.
    // Returns as soon as the images have been copied; the kernels overlap the caller's next steps.
    template <class Mat, class Mat4f>
    int fuse_map(Mat &image, Mat &depth, Mat4f &pose, int reference_index)
    {
        if (!ready("fuse_map")) return err_;
        err_ = dsm_fuse_frame_resident(ctx_, reference_index, reinterpret_cast<const uint8_t *>(image.data), (size_t)image.step,
                                       reinterpret_cast<const float *>(depth.data), (size_t)depth.step, pose.data(), nullptr);
        return report("fuse_map");
    }

    // synchronize_msgs (surfel_map.cpp:154-161) in one call: move_add_surfels with the lists get_add_remove_poses hands
    // it (poses_to_remove, then poses_to_add), then fuse_map -- all on the device, and the call never synchronises (a
    // frame that does not fit the pool or the inactive store is reported by the next call that reads the map, see
    // dsm_fuse_stream_window).  Non-empty lists need reserve_inactive().
    template <class Mat, class Mat4f>
    int fuse_map(Mat &image, Mat &depth, Mat4f &pose, int reference_index, const std::vector<int> &poses_to_remove,
                 const std::vector<int> &poses_to_add)
    {
        if (!ready("fuse_map")) return err_;
        const uint8_t *g = reinterpret_cast<const uint8_t *>(image.data);
        const float *d = reinterpret_cast<const float *>(depth.data);
        if ((size_t)image.step != (size_t)width_ || (size_t)depth.step != (size_t)width_ * 4)
        { // the stream entry point takes tightly packed images
            packed_gray_.resize((size_t)width_ * height_);
            packed_depth_.resize((size_t)width_ * height_);
            for (int y = 0; y < height_; y++)
            {
                std::memcpy(&packed_gray_[(size_t)y * width_], g + (size_t)y * image.step, (size_t)width_);
                std::memcpy(&packed_depth_[(size_t)y * width_], reinterpret_cast<const uint8_t *>(d) + (size_t)y * depth.step,
                            (size_t)width_ * 4);
            }
            g = packed_gray_.data(), d = packed_depth_.data();
        }
        const std::vector<int32_t> rk(poses_to_remove.begin(), poses_to_remove.end()), ak(poses_to_add.begin(), poses_to_add.end());
        const int32_t ro[2] = {0, (int32_t)rk.size()}, ao[2] = {0, (int32_t)ak.size()};
        const int32_t ref = reference_index;
        err_ = dsm_fuse_stream_window(ctx_, 1, &ref, g, d, pose.data(), rk.data(), ro, ak.data(), ao, nullptr);
        return report("fuse_map");
    }

    // warp_surfels(): p <- W p, n <- R_W n for every local surfel; W = T_loop * T_cam^-1 as float, column-major
    template <class Mat4f>
    int warp_active_surfels(Mat4f &warp_pose)
    {
        if (!ready("warp_active_surfels")) return err_;
        err_ = dsm_pool_transform(ctx_, warp_pose.data());
        return report("warp_active_surfels");
    }

    // move_add_surfels(), removal: the live surfels last updated by keyframe `inactive_index` leave the pool
    // (in pool order) and become that pose's attached_surfels
    template <class Surfel>
    int retire_surfels(int inactive_index, std::vector<Surfel> &attached_surfels)
    {
        static_assert(sizeof(Surfel) == sizeof(dsm_surfel_t), "SurfelElement must be the 44-byte reference POD");
        attached_surfels.clear();
        if (!ready("retire_surfels")) return err_;
        int n = 0;
        err_ = dsm_pool_size(ctx_, &n);
        if (err_ == DSM_OK)
        {
            attached_surfels.resize((size_t)n);
            int got = 0;
            err_ = dsm_pool_retire(ctx_, inactive_index, reinterpret_cast<dsm_surfel_t *>(attached_surfels.data()), n, &got);
            attached_surfels.resize(err_ == DSM_OK ? (size_t)got : 0);
        }
        return report("retire_surfels");
    }

    // move_add_surfels(), insertion: a pose re-enters the drift-free set
    template <class Surfel>
    int add_surfels(const std::vector<Surfel> &attached_surfels)
    {
        static_assert(sizeof(Surfel) == sizeof(dsm_surfel_t), "SurfelElement must be the 44-byte reference POD");
        if (!ready("add_surfels")) return err_;
        err_ = dsm_pool_append(ctx_, reinterpret_cast<const dsm_surfel_t *>(attached_surfels.data()), (int)attached_surfels.size());
        return report("add_surfels");
    }

    // the local_surfels loop of the cloud publishers: points with update_times >= min_update_times, pool order.
    // Point: any type with float members x, y, z, intensity (pcl::PointXYZI) -- appended to `points`.
    template <class Point>
    int active_points(std::vector<Point> &points, int min_update_times = 5)
    {
        if (!ready("active_points")) return err_;
        int n = 0;
        err_ = dsm_pool_size(ctx_, &n);
        if (err_ != DSM_OK) return report("active_points");
        scratch_.resize((size_t)(n > 0 ? n : 1));
        int got = 0;
        err_ = dsm_pool_export_cloud(ctx_, min_update_times, scratch_.data(), n, &got);
        if (err_ != DSM_OK) return report("active_points");
        append(points, got);
        return DSM_OK;
    }

    // save_cloud: active points (update_times >= 5) followed by the caller's inactive cloud, PCD v0.7 ASCII
    template <class Point>
    int save_cloud(const std::string &save_path_name, const std::vector<Point> &inactive_points)
    {
        std::vector<dsm_point_t> all;
        if (active_points(all, 5) != DSM_OK) return err_;
        all.reserve(all.size() + inactive_points.size());
        for (size_t i = 0; i < inactive_points.size(); i++)
        {
            dsm_point_t q;
            q.x = inactive_points[i].x, q.y = inactive_points[i].y, q.z = inactive_points[i].z;
            q.intensity = inactive_points[i].intensity;
            all.push_back(q);
        }
        err_ = dsm_write_pcd(save_path_name.c_str(), all.data(), all.size(), 0);
        return report("save_cloud");
    }

    // save_mesh: the attached surfels of every pose (no filter) followed by the local surfels with
    // update_times >= 5, one hexagon each, ASCII PLY
    template <class Surfel>
    int save_mesh(const std::string &save_path_name, const std::vector<Surfel> &attached_surfels_of_all_poses)
    {
        static_assert(sizeof(Surfel) == sizeof(dsm_surfel_t), "SurfelElement must be the 44-byte reference POD");
        if (!ready("save_mesh")) return err_;
        int n = 0;
        err_ = dsm_pool_size(ctx_, &n);
        if (err_ != DSM_OK) return report("save_mesh");
        const size_t na = attached_surfels_of_all_poses.size();
        std::vector<dsm_surfel_t> all(na + (size_t)(n > 0 ? n : 1));
        if (na) std::memcpy(all.data(), attached_surfels_of_all_poses.data(), na * sizeof(dsm_surfel_t));
        int got = 0;
        err_ = dsm_pool_export_surfels(ctx_, 5, all.data() + na, n, &got);
        if (err_ == DSM_OK) err_ = dsm_write_ply_mesh(save_path_name.c_str(), all.data(), na + (size_t)got);
        return report("save_mesh");
    }

    // ---- device-resident attached_surfels / inactive_pointcloud (see include/dsm.h "inactive store") ----
    // Call reserve_inactive() once after initialize(); then the removal / insertion halves of move_add_surfels and the
    // per-pose inactive warp never move surfels across PCIe.
    int reserve_inactive(int max_inactive_surfels)
    {
        if (!ready("reserve_inactive")) return err_;
        err_ = dsm_inactive_reserve(ctx_, max_inactive_surfels);
        return report("reserve_inactive");
    }
    // move_add_surfels(), removal (surfel_map.cpp:1479-1497) without the host copy; returns the surfel count or -1
    int retire_surfels_resident(int inactive_index)
    {
        if (!ready("retire_surfels_resident")) return -1;
        int n = 0;
        err_ = dsm_inactive_retire(ctx_, inactive_index, &n);
        return report("retire_surfels_resident") == DSM_OK ? n : -1;
    }
    // move_add_surfels(), insertion (surfel_map.cpp:1583-1587)
    int add_surfels_resident(int pose_index)
    {
        if (!ready("add_surfels_resident")) return -1;
        int n = 0;
        err_ = dsm_inactive_reactivate(ctx_, pose_index, &n);
        return report("add_surfels_resident") == DSM_OK ? n : -1;
    }
    // warp_inactive_surfels_cpu_kernel for one pose (surfel_map.cpp:704-733): warp_matrix = (after * pre^-1).cast<float>()
    template <class Mat4f>
    int warp_inactive_surfels(int pose_index, Mat4f &warp_matrix)
    {
        if (!ready("warp_inactive_surfels")) return err_;
        err_ = dsm_inactive_transform(ctx_, pose_index, warp_matrix.data());
        return report("warp_inactive_surfels");
    }
    // inactive_pointcloud appended to `points` (publish_inactive_pointcloud / publish_all_pointcloud / save_cloud)
    template <class Point>
    int inactive_points(std::vector<Point> &points)
    {
        if (!ready("inactive_points")) return err_;
        int n = 0;
        err_ = dsm_inactive_size(ctx_, &n, nullptr);
        if (err_ != DSM_OK) return report("inactive_points");
        scratch_.resize((size_t)(n > 0 ? n : 1));
        int got = 0;
        err_ = dsm_inactive_export_cloud(ctx_, scratch_.data(), n, &got);
        if (err_ != DSM_OK) return report("inactive_points");
        append(points, got);
        return DSM_OK;
    }

    // publish_neighbor_pointcloud (surfel_map.cpp:1283-1383): the live local points (update_times != 0) followed by the
    // stored points of the poses in neighbor_indexs, in list order -- pass get_driftfree_poses(reference_index, ...,
    // 2*drift_free_poses) unchanged (local poses and poses with nothing stored contribute nothing).  Appended to `points`.
    template <class Point>
    int neighbor_points(std::vector<Point> &points, const std::vector<int> &neighbor_indexs)
    {
        if (active_points(points, 1) != DSM_OK) return err_;
        int n = 0;
        err_ = dsm_inactive_size(ctx_, &n, nullptr);
        if (err_ != DSM_OK) return report("neighbor_points");
        scratch_.resize((size_t)(n > 0 ? n : 1));
        std::vector<int32_t> kf(neighbor_indexs.begin(), neighbor_indexs.end());
        int got = 0;
        err_ = dsm_inactive_export_poses(ctx_, kf.data(), (int)kf.size(), scratch_.data(), n, &got);
        if (err_ != DSM_OK) return report("neighbor_points");
        append(points, got);
        return DSM_OK;
    }

    // publish_raw_pointcloud (surfel_map.cpp:1115-1151) of the frame of the last fuse_map: every pixel in the world frame,
    // column-major, holes included.  Pose: any type with position.{x,y,z} and orientation.{x,y,z,w}
    // (geometry_msgs::Pose).  Appended to `points`.
    template <class Point, class Pose>
    int raw_points(std::vector<Point> &points, const Pose &pose)
    {
        if (!ready("raw_points")) return err_;
        const double p7[7] = {pose.position.x, pose.position.y, pose.position.z, pose.orientation.x, pose.orientation.y,
                              pose.orientation.z, pose.orientation.w};
        scratch_.resize((size_t)width_ * (size_t)height_);
        int got = 0;
        err_ = dsm_frame_raw_cloud(ctx_, 0, p7, scratch_.data(), (int)scratch_.size(), &got);
        if (err_ != DSM_OK) return report("raw_points");
        append(points, got);
        return DSM_OK;
    }

    // FusionFunctions::debug_show (fusion_functions.cpp:977-1006) of the frame of the last fuse_map: the superpixel normal
    // image, height rows of width x 3 bytes written at the image's row pitch (bytes past 3*width untouched).  Mat: any
    // type with .data and .step, allocated by the caller (a cv::Mat(height, width, CV_8UC3)).
    template <class Mat>
    int superpixel_image(Mat &image)
    {
        if (!ready("superpixel_image")) return err_;
        err_ = dsm_frame_superpixel_image(ctx_, 0, reinterpret_cast<uint8_t *>(image.data), (size_t)image.step);
        return report("superpixel_image");
    }

    // local_surfels as a host vector (debugging, or a caller that still wants the whole pool)
    template <class Surfel>
    int download(std::vector<Surfel> &local_surfels)
    {
        static_assert(sizeof(Surfel) == sizeof(dsm_surfel_t), "SurfelElement must be the 44-byte reference POD");
        local_surfels.clear();
        if (!ready("download")) return err_;
        int n = 0;
        err_ = dsm_pool_size(ctx_, &n);
        if (err_ == DSM_OK)
        {
            local_surfels.resize((size_t)n);
            int got = 0;
            err_ = dsm_pool_download(ctx_, reinterpret_cast<dsm_surfel_t *>(local_surfels.data()), n, &got);
        }
        return report("download");
    }

    int size()
    {
        int n = 0;
        if (!ctx_ || dsm_pool_size(ctx_, &n) != DSM_OK) return 0;
        return n;
    }
    int last_error() const { return err_; }
    dsm_ctx *context() { return ctx_; }

  private:
    bool ready(const char *what)
    {
        if (ctx_) return true;
        err_ = DSM_E_STATE;
        std::fprintf(stderr, "dsm::ResidentSurfelPool::%s: initialize() has not succeeded\n", what);
        return false;
    }
    // the first `got` points of scratch_, converted field by field, appended to `points`
    template <class Point>
    void append(std::vector<Point> &points, int got)
    {
        points.reserve(points.size() + (size_t)got);
        for (int i = 0; i < got; i++)
        {
            Point p;
            p.x = scratch_[(size_t)i].x, p.y = scratch_[(size_t)i].y, p.z = scratch_[(size_t)i].z;
            p.intensity = scratch_[(size_t)i].intensity;
            points.push_back(p);
        }
    }
    int report(const char *what)
    {
        if (err_ != DSM_OK)
            std::fprintf(stderr, "dsm::ResidentSurfelPool::%s failed: %s (%s)\n", what, dsm_strerror(err_), ctx_ ? dsm_last_error(ctx_) : "no context");
        return err_;
    }
    dsm_ctx *ctx_;
    int err_;
    int device_;
    int capacity_;
    int width_, height_;
    std::vector<dsm_point_t> scratch_;
    std::vector<uint8_t> packed_gray_;
    std::vector<float> packed_depth_;
};
} // namespace dsm
