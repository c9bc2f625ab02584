// TEST INFRASTRUCTURE ONLY.  The SurfelMap oracle of ref_map_driver.cpp (the reference's own surfel_map.cpp compiled in
// place) with three more hooks for the node's per-frame window step (move_add_surfels, surfel_map.cpp:1458-1595): the
// lists get_add_remove_poses hands it, the fuse pose synchronize_msgs hands fuse_map, and the image callbacks alone.  Built into
// oracle/_ref/libdsm_refmap_window[_b200].so by oracle/window.mk; every entry point of libdsm_refmap.so is exported too.
#include "ref_map_driver.cpp"

static int copy_list(const std::vector<int> &v, int *out, int cap)
{
    for (size_t i = 0; i < v.size() && (int)i < cap; i++) out[i] = v[i];
    return (int)v.size();
}

extern "C"
{
    // get_add_remove_poses(root, add, remove) (surfel_map.cpp:1597-1641) on the current state; reads only the pose graph
    // and local_surfels_indexs.  Returns the two lengths through n_add / n_remove, writes at most cap entries of each.
    void dsmmap_window_lists(RefMap *r, int root, int *add, int *n_add, int *remove, int *n_remove, int cap)
    {
        std::vector<int> a, rm;
        r->map->get_add_remove_poses(root, a, rm);
        *n_add = copy_list(a, add, cap);
        *n_remove = copy_list(rm, remove, cap);
    }
    // What synchronize_msgs (surfel_map.cpp:143-161) will do with the frame at the front of the pose buffer once its
    // image and depth arrive: the reference index (returned; -1 if the buffer is empty), the pose it hands fuse_map
    // (fuse_pose.cast<float>(), column-major) and the window lists move_add_surfels(reference index) will use.
    int dsmmap_pending_frame(RefMap *r, float *pose16, int *add, int *n_add, int *remove, int *n_remove, int cap)
    {
        SurfelMap *m = r->map;
        if (m->pose_reference_buffer.empty()) return -1;
        geometry_msgs::Pose relative_pose_ros = std::get<1>(m->pose_reference_buffer.front());
        const int relative_index = std::get<2>(m->pose_reference_buffer.front());
        Eigen::Matrix4d reference_pose, fuse_pose, relative_pose;
        m->pose_ros2eigen(m->poses_database[relative_index].cam_pose, reference_pose);
        m->pose_ros2eigen(relative_pose_ros, relative_pose);
        fuse_pose = reference_pose * relative_pose;
        const Eigen::Matrix4f f = fuse_pose.cast<float>();
        for (int i = 0; i < 16; i++) pose16[i] = f.d[i];
        dsmmap_window_lists(r, relative_index, add, n_add, remove, n_remove, cap);
        return relative_index;
    }
}

extern "C"
{
    // the image and depth callbacks alone (ros_node.cpp), after a pose feed through dsmmap_frame(..., gray = NULL, ...):
    // synchronize_msgs then runs move_add_surfels and fuse_map for the pending frame
    void dsmmap_images(RefMap *r, double stamp, const unsigned char *gray, const float *depth)
    {
        const int W = r->map->cam_width, H = r->map->cam_height;
        r->map->image_input(make_image(stamp, W, H, gray, false));
        r->map->depth_input(make_image(stamp, W, H, depth, true));
    }
}
