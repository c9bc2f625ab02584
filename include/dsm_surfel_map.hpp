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
//
// The map operations themselves are the functions of dsm::detail below, one per operation; dsm::SurfelMapNode
// (dsm_surfel_node.hpp) is built on the same ones.
#pragma once
#include <cstring>
#include <string>
#include <vector>
#include "dsm_context.hpp"

namespace dsm
{
namespace detail
{
// Each operation needs a context (Context::ready), returns the C ABI code and appends to the caller's vector, which a
// failure leaves as it was.

inline int pool_size(Context &c, int &n)
{
    n = 0;
    return dsm_pool_size(c.ctx, &n);
}
// the size-then-read of the pool and of the inactive store (read_records)
template <class Rec, class T, class Read>
int read_pool(Context &c, std::vector<T> &out, Read read)
{
    int n = 0;
    const int rc = pool_size(c, n);
    return rc != DSM_OK ? rc : read_records<Rec>(out, n, read);
}
template <class Rec, class T, class Read>
int read_store(Context &c, std::vector<T> &out, Read read)
{
    int n = 0;
    const int rc = dsm_inactive_size(c.ctx, &n, nullptr);
    return rc != DSM_OK ? rc : read_records<Rec>(out, n, read);
}

// the local_surfels loop of the cloud publishers: points with update_times >= min_update_times, pool order
template <class Point>
int pool_cloud(Context &c, int min_update_times, std::vector<Point> &points)
{
    return read_pool<dsm_point_t>(c, points, [&](dsm_point_t *o, int cap, int *got) { return dsm_pool_export_cloud(c.ctx, min_update_times, o, cap, got); });
}
// the local surfels with update_times >= min_update_times, pool order
inline int pool_surfels(Context &c, int min_update_times, std::vector<dsm_surfel_t> &surfels)
{
    return read_pool<dsm_surfel_t>(c, surfels, [&](dsm_surfel_t *o, int cap, int *got) { return dsm_pool_export_surfels(c.ctx, min_update_times, o, cap, got); });
}
// local_surfels, pool order
template <class Surfel>
int whole_pool(Context &c, std::vector<Surfel> &surfels)
{
    return read_pool<dsm_surfel_t>(c, surfels, [&](dsm_surfel_t *o, int cap, int *got) { return dsm_pool_download(c.ctx, o, cap, got); });
}
// move_add_surfels(), removal: the live surfels last updated by `keyframe` leave the pool, in pool order
template <class Surfel>
int retire(Context &c, int keyframe, std::vector<Surfel> &surfels)
{
    return read_pool<dsm_surfel_t>(c, surfels, [&](dsm_surfel_t *o, int cap, int *got) { return dsm_pool_retire(c.ctx, keyframe, o, cap, got); });
}
// inactive_pointcloud: the inactive store, store order
template <class Point>
int inactive_cloud(Context &c, std::vector<Point> &points)
{
    return read_store<dsm_point_t>(c, points, [&](dsm_point_t *o, int cap, int *got) { return dsm_inactive_export_cloud(c.ctx, o, cap, got); });
}
// publish_neighbor_pointcloud (surfel_map.cpp:1283-1383): the live local points (update_times != 0), then the stored
// points of `keyframes` in list order
template <class Point>
int neighbourhood(Context &c, const std::vector<int> &keyframes, std::vector<Point> &points)
{
    const std::vector<int32_t> kf(keyframes.begin(), keyframes.end());
    const int rc = pool_cloud(c, 1, points);
    return rc != DSM_OK ? rc : read_store<dsm_point_t>(c, points, [&](dsm_point_t *o, int cap, int *got) {
        return dsm_inactive_export_poses(c.ctx, kf.data(), (int)kf.size(), o, cap, got);
    });
}
// PoseElement::attached_surfels of one keyframe, or the whole store in store order for keyframe -1
template <class Surfel>
int attached(Context &c, int keyframe, std::vector<Surfel> &surfels)
{
    int n = 0;
    const int rc = dsm_inactive_download(c.ctx, keyframe, nullptr, 0, &n);
    return rc != DSM_OK ? rc : read_records<dsm_surfel_t>(surfels, n, [&](dsm_surfel_t *o, int cap, int *got) {
        return dsm_inactive_download(c.ctx, keyframe, o, cap, got);
    });
}
// publish_raw_pointcloud (surfel_map.cpp:1115-1151) of the last fused frame: every pixel (n_pixels = width * height) in
// the world frame at pose7 = {px, py, pz, qx, qy, qz, qw}, column-major, holes included
template <class Point>
int raw_cloud(Context &c, const double pose7[7], int n_pixels, std::vector<Point> &points)
{
    return read_records<dsm_point_t>(points, n_pixels, [&](dsm_point_t *o, int cap, int *got) { return dsm_frame_raw_cloud(c.ctx, 0, pose7, o, cap, got); });
}

// save_mesh: `surfels` (the attached surfels of every pose) followed by the local surfels with update_times >= 5, one
// hexagon each, ASCII PLY
inline int save_mesh(Context &c, const std::string &name, std::vector<dsm_surfel_t> surfels)
{
    int rc = pool_surfels(c, 5, surfels);
    if (rc == DSM_OK) rc = dsm_write_ply_mesh(name.c_str(), surfels.data(), surfels.size());
    return rc;
}
// save_cloud: the local points with update_times >= 5 followed by the inactive cloud, PCD v0.7 ASCII.  The inactive
// cloud is the caller's `inactive` points, or the device store's when it is null.
template <class Point>
int save_cloud(Context &c, const std::string &name, const std::vector<Point> *inactive)
{
    std::vector<dsm_point_t> points;
    int rc = pool_cloud(c, 5, points);
    if (rc == DSM_OK && !inactive) rc = inactive_cloud(c, points);
    if (rc != DSM_OK) return rc;
    if (inactive) append_points(points, *inactive);
    return dsm_write_pcd(name.c_str(), points.data(), points.size(), 0);
}

// synchronize_msgs (surfel_map.cpp:154-161) for one frame: move_add_surfels with the two lists, then fuse_map, all on
// the device; tightly packed images
inline int fuse_window(Context &c, int reference_index, const uint8_t *gray, const float *depth, const float pose16[16],
                       const std::vector<int> &poses_to_remove, const std::vector<int> &poses_to_add)
{
    const std::vector<int32_t> rk(poses_to_remove.begin(), poses_to_remove.end()), ak(poses_to_add.begin(), poses_to_add.end());
    const int32_t ro[2] = {0, (int32_t)rk.size()}, ao[2] = {0, (int32_t)ak.size()};
    const int32_t ref = reference_index;
    return dsm_fuse_stream_window(c.ctx, 1, &ref, gray, depth, pose16, rk.data(), ro, ak.data(), ao, nullptr);
}

// the checkpoint of the map (dsm_map_save) with the caller's `extra` bytes in it
inline int save_state(Context &c, const std::string &path, const std::vector<uint8_t> &extra)
{
    return dsm_map_save(c.ctx, path.c_str(), extra.data(), extra.size());
}
// the same file, taken in stream order and written by the context's thread (dsm_checkpoint_enqueue)
inline int save_state_async(Context &c, const std::string &path, const std::vector<uint8_t> &extra)
{
    return dsm_checkpoint_enqueue(c.ctx, path.c_str(), extra.data(), extra.size());
}
// dsm_checkpoint_wait with a C++ flag
inline int wait_state_saved(Context &c, bool block, bool *finished)
{
    int fin = 0;
    const int rc = dsm_checkpoint_wait(c.ctx, block ? 1 : 0, &fin);
    if (finished) *finished = fin != 0;
    return rc;
}
// dsm_map_load: the map replaced by the checkpoint's, whose extra bytes replace `extra`; a failure leaves both as they were
inline int load_state(Context &c, const std::string &path, std::vector<uint8_t> &extra)
{
    size_t n = 0;
    std::vector<uint8_t> got;
    int rc = dsm_map_load(c.ctx, path.c_str(), nullptr, 0, &n);
    if (rc == DSM_E_CAPACITY && n > 0)
    { // the size-then-read of the extra section: nothing was loaded by the first call
        got.resize(n);
        rc = dsm_map_load(c.ctx, path.c_str(), got.data(), got.size(), &n);
    }
    if (rc == DSM_OK) extra.swap(got);
    return rc;
}
// save_state_async as one journal record of the changed chunks beside the base at path, or a new base
// (dsm_checkpoint_enqueue_incremental, DESIGN.md §8.6); wait_state_saved retires it
inline int save_state_incremental(Context &c, const std::string &path, const std::vector<uint8_t> &extra)
{
    return dsm_checkpoint_enqueue_incremental(c.ctx, path.c_str(), extra.data(), extra.size());
}
// load_state of the state the base at path and its journal resolve to (dsm_map_load_journal); *records (optional): the
// journal records applied
inline int load_state_incremental(Context &c, const std::string &path, std::vector<uint8_t> &extra, int *records = nullptr)
{
    size_t n = 0;
    int applied = 0;
    std::vector<uint8_t> got;
    int rc = dsm_map_load_journal(c.ctx, path.c_str(), nullptr, 0, &n, &applied);
    if (rc == DSM_E_CAPACITY && n > 0)
    { // the size-then-read of the extra section: nothing was loaded by the first call
        got.resize(n);
        rc = dsm_map_load_journal(c.ctx, path.c_str(), got.data(), got.size(), &n, &applied);
    }
    if (rc == DSM_OK) extra.swap(got);
    if (records) *records = rc == DSM_OK ? applied : 0;
    return rc;
}
} // namespace detail

class ResidentSurfelPool
{
  public:
    ResidentSurfelPool() : ctx_("dsm::ResidentSurfelPool"), device_(0), capacity_(1 << 21), width_(0), height_(0) {}

    void set_device(int device, int max_local_surfels = 1 << 21)
    {
        device_ = device;
        capacity_ = max_local_surfels;
    }

    int initialize(int width, int height, float fx, float fy, float cx, float cy, float fuse_far, float fuse_near)
    {
        width_ = width, height_ = height;
        // two frame slots: the copy of frame t+1 overlaps the kernels of frame t; local_surfels starts empty
        const dsm_params p = detail::Context::params(width, height, fx, fy, cx, cy, fuse_far, fuse_near, 2, capacity_);
        return ctx_.open("initialize", p, device_, true, nullptr, nullptr);
    }

    // SurfelMap::fuse_map: the hot-path call plus the post-step (slot recycling as the reference), all on the device.
    // Returns as soon as the images have been copied; the kernels overlap the caller's next steps.
    template <class Mat, class Mat4f>
    int fuse_map(Mat &image, Mat &depth, Mat4f &pose, int reference_index)
    {
        return ctx_.run("fuse_map", [&] {
            return dsm_fuse_frame_resident(ctx_.ctx, reference_index, reinterpret_cast<const uint8_t *>(image.data), (size_t)image.step,
                                           reinterpret_cast<const float *>(depth.data), (size_t)depth.step, pose.data(), nullptr);
        });
    }

    // synchronize_msgs (surfel_map.cpp:154-161) in one call: move_add_surfels with the lists get_add_remove_poses hands
    // it (poses_to_remove, then poses_to_add), then fuse_map -- all on the device, and the call never synchronises (a
    // frame that does not fit the pool or the inactive store is reported by the next call that reads the map, see
    // dsm_fuse_stream_window).  Non-empty lists need reserve_inactive().
    template <class Mat, class Mat4f>
    int fuse_map(Mat &image, Mat &depth, Mat4f &pose, int reference_index, const std::vector<int> &poses_to_remove,
                 const std::vector<int> &poses_to_add)
    {
        if (!ctx_.ready("fuse_map")) return ctx_.err;
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
        return ctx_.done(detail::fuse_window(ctx_, reference_index, g, d, pose.data(), poses_to_remove, poses_to_add), "fuse_map");
    }

    // warp_surfels(): p <- W p, n <- R_W n for every local surfel; W = T_loop * T_cam^-1 as float, column-major
    template <class Mat4f>
    int warp_active_surfels(Mat4f &warp_pose)
    {
        return ctx_.run("warp_active_surfels", [&] { return dsm_pool_transform(ctx_.ctx, warp_pose.data()); });
    }

    // move_add_surfels(), removal: the live surfels last updated by keyframe `inactive_index` leave the pool
    // (in pool order) and become that pose's attached_surfels
    template <class Surfel>
    int retire_surfels(int inactive_index, std::vector<Surfel> &attached_surfels)
    {
        attached_surfels.clear();
        return ctx_.run("retire_surfels", [&] { return detail::retire(ctx_, inactive_index, attached_surfels); });
    }

    // move_add_surfels(), insertion: a pose re-enters the drift-free set
    template <class Surfel>
    int add_surfels(const std::vector<Surfel> &attached_surfels)
    {
        static_assert(sizeof(Surfel) == sizeof(dsm_surfel_t), "SurfelElement must be the 44-byte reference POD");
        return ctx_.run("add_surfels", [&] {
            return dsm_pool_append(ctx_.ctx, reinterpret_cast<const dsm_surfel_t *>(attached_surfels.data()), (int)attached_surfels.size());
        });
    }

    // the local_surfels loop of the cloud publishers: points with update_times >= min_update_times, pool order.
    // Point: any type with float members x, y, z, intensity (pcl::PointXYZI) -- appended to `points`.
    template <class Point>
    int active_points(std::vector<Point> &points, int min_update_times = 5)
    {
        return ctx_.run("active_points", [&] { return detail::pool_cloud(ctx_, min_update_times, points); });
    }

    // save_cloud: active points (update_times >= 5) followed by the caller's inactive cloud, PCD v0.7 ASCII
    template <class Point>
    int save_cloud(const std::string &save_path_name, const std::vector<Point> &inactive_points)
    {
        return ctx_.run("save_cloud", [&] { return detail::save_cloud(ctx_, save_path_name, &inactive_points); });
    }

    // save_mesh: the attached surfels of every pose (no filter) followed by the local surfels with
    // update_times >= 5, one hexagon each, ASCII PLY
    template <class Surfel>
    int save_mesh(const std::string &save_path_name, const std::vector<Surfel> &attached_surfels_of_all_poses)
    {
        static_assert(sizeof(Surfel) == sizeof(dsm_surfel_t), "SurfelElement must be the 44-byte reference POD");
        if (!ctx_.ready("save_mesh")) return ctx_.err;
        const dsm_surfel_t *a = reinterpret_cast<const dsm_surfel_t *>(attached_surfels_of_all_poses.data());
        return ctx_.done(detail::save_mesh(ctx_, save_path_name, std::vector<dsm_surfel_t>(a, a + attached_surfels_of_all_poses.size())),
                         "save_mesh");
    }

    // ---- device-resident attached_surfels / inactive_pointcloud (see include/dsm.h "inactive store") ----
    // Call reserve_inactive() once after initialize(); then the removal / insertion halves of move_add_surfels and the
    // per-pose inactive warp never move surfels across PCIe.
    int reserve_inactive(int max_inactive_surfels)
    {
        return ctx_.run("reserve_inactive", [&] { return dsm_inactive_reserve(ctx_.ctx, max_inactive_surfels); });
    }
    // move_add_surfels(), removal (surfel_map.cpp:1479-1497) without the host copy; returns the surfel count or -1
    int retire_surfels_resident(int inactive_index)
    {
        int n = 0;
        return ctx_.run("retire_surfels_resident", [&] { return dsm_inactive_retire(ctx_.ctx, inactive_index, &n); }) == DSM_OK ? n : -1;
    }
    // move_add_surfels(), insertion (surfel_map.cpp:1583-1587)
    int add_surfels_resident(int pose_index)
    {
        int n = 0;
        return ctx_.run("add_surfels_resident", [&] { return dsm_inactive_reactivate(ctx_.ctx, pose_index, &n); }) == DSM_OK ? n : -1;
    }
    // warp_inactive_surfels_cpu_kernel for one pose (surfel_map.cpp:704-733): warp_matrix = (after * pre^-1).cast<float>()
    template <class Mat4f>
    int warp_inactive_surfels(int pose_index, Mat4f &warp_matrix)
    {
        return ctx_.run("warp_inactive_surfels", [&] { return dsm_inactive_transform(ctx_.ctx, pose_index, warp_matrix.data()); });
    }
    // PoseElement::attached_surfels of pose_index as stored on the device, or every pose's in store order for -1
    template <class Surfel>
    int attached_surfels(int pose_index, std::vector<Surfel> &out)
    {
        out.clear();
        return ctx_.run("attached_surfels", [&] { return detail::attached(ctx_, pose_index, out); });
    }
    // inactive_pointcloud appended to `points` (publish_inactive_pointcloud / publish_all_pointcloud / save_cloud)
    template <class Point>
    int inactive_points(std::vector<Point> &points)
    {
        return ctx_.run("inactive_points", [&] { return detail::inactive_cloud(ctx_, points); });
    }

    // publish_neighbor_pointcloud (surfel_map.cpp:1283-1383): the live local points (update_times != 0) followed by the
    // stored points of the poses in neighbor_indexs, in list order -- pass get_driftfree_poses(reference_index, ...,
    // 2*drift_free_poses) unchanged (local poses and poses with nothing stored contribute nothing).  Appended to `points`.
    template <class Point>
    int neighbor_points(std::vector<Point> &points, const std::vector<int> &neighbor_indexs)
    {
        return ctx_.run("neighbor_points", [&] { return detail::neighbourhood(ctx_, neighbor_indexs, points); });
    }

    // publish_raw_pointcloud (surfel_map.cpp:1115-1151) of the frame of the last fuse_map: every pixel in the world frame,
    // column-major, holes included.  Pose: any type with position.{x,y,z} and orientation.{x,y,z,w}
    // (geometry_msgs::Pose).  Appended to `points`.
    template <class Point, class Pose>
    int raw_points(std::vector<Point> &points, const Pose &pose)
    {
        if (!ctx_.ready("raw_points")) return ctx_.err;
        const double p7[7] = {pose.position.x, pose.position.y, pose.position.z, pose.orientation.x, pose.orientation.y,
                              pose.orientation.z, pose.orientation.w};
        return ctx_.done(detail::raw_cloud(ctx_, p7, width_ * height_, points), "raw_points");
    }

    // FusionFunctions::debug_show (fusion_functions.cpp:977-1006) of the frame of the last fuse_map: the superpixel normal
    // image, height rows of width x 3 bytes written at the image's row pitch (bytes past 3*width untouched).  Mat: any
    // type with .data and .step, allocated by the caller (a cv::Mat(height, width, CV_8UC3)).
    template <class Mat>
    int superpixel_image(Mat &image)
    {
        return ctx_.run("superpixel_image", [&] { return detail::superpixel_image(ctx_, image); });
    }

    // local_surfels as a host vector (debugging, or a caller that still wants the whole pool)
    template <class Surfel>
    int download(std::vector<Surfel> &local_surfels)
    {
        local_surfels.clear();
        return ctx_.run("download", [&] { return detail::whole_pool(ctx_, local_surfels); });
    }

    // ---- checkpoint and resume (DESIGN.md §8.4) ----
    // local_surfels, the device store and its segment table to one file, with the caller's own state (the pose
    // database of a SurfelMap that keeps it) as `extra`; load_state replaces the map by the file's and returns that
    // `extra`.  The constants must be set before loading; a failed load leaves the map as it was.
    int save_state(const std::string &path, const std::vector<uint8_t> &extra)
    {
        return ctx_.run("save_state", [&] { return detail::save_state(ctx_, path, extra); });
    }
    int load_state(const std::string &path, std::vector<uint8_t> &extra)
    {
        return ctx_.run("load_state", [&] { return detail::load_state(ctx_, path, extra); });
    }
    // The same file without stopping the stream (DESIGN.md §8.5): enable_checkpoints once after initialize;
    // save_state_async enqueues the file save_state would write at this point of the stream and returns at once;
    // wait_state_saved(false, &finished) polls it (finished = false while it is written), wait_state_saved(true, ...)
    // waits, and either returns the write's result once finished.  One checkpoint at a time.
    int enable_checkpoints()
    {
        return ctx_.run("enable_checkpoints", [&] { return dsm_checkpoint_enable(ctx_.ctx); });
    }
    int save_state_async(const std::string &path, const std::vector<uint8_t> &extra)
    {
        return ctx_.run("save_state_async", [&] { return detail::save_state_async(ctx_, path, extra); });
    }
    int wait_state_saved(bool block, bool *finished)
    {
        return ctx_.run("wait_state_saved", [&] { return detail::wait_state_saved(ctx_, block, finished); });
    }
    // Incremental checkpoints (DESIGN.md §8.6): save_state_incremental is save_state_async, written as one record of the
    // changed chunks appended to <path>.journal, or as a new base file at path when a record cannot be (the first save to
    // path, a failed save, the map replaced, the journal larger than its base).  load_state_incremental loads the state
    // base and journal resolve to; *records (optional) receives the records applied.
    int save_state_incremental(const std::string &path, const std::vector<uint8_t> &extra)
    {
        return ctx_.run("save_state_incremental", [&] { return detail::save_state_incremental(ctx_, path, extra); });
    }
    int load_state_incremental(const std::string &path, std::vector<uint8_t> &extra, int *records = nullptr)
    {
        return ctx_.run("load_state_incremental", [&] { return detail::load_state_incremental(ctx_, path, extra, records); });
    }

    int size()
    {
        int n = 0;
        if (!ctx_.ctx || detail::pool_size(ctx_, n) != DSM_OK) return 0;
        return n;
    }
    int last_error() const { return ctx_.err; }
    dsm_ctx *context() { return ctx_.ctx; }

  private:
    detail::Context ctx_;
    int device_;
    int capacity_;
    int width_, height_;
    std::vector<uint8_t> packed_gray_;
    std::vector<float> packed_depth_;
};
} // namespace dsm
