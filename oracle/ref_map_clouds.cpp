// TEST INFRASTRUCTURE ONLY.  The SurfelMap oracle of ref_map_driver.cpp (the reference's own surfel_map.cpp compiled in
// place) with two more hooks, for the node's two remaining cloud publishers: publish_raw_pointcloud itself, and the
// drift-free BFS (get_driftfree_poses) that publish_neighbor_pointcloud walks.  Built into
// oracle/_ref/libdsm_refmap_clouds.so by oracle/clouds.mk; every entry point of libdsm_refmap.so is exported too.
#include "ref_map_driver.cpp"

extern "C"
{
    // publish_raw_pointcloud(depth, image, pose) (surfel_map.cpp:1115-1151) on a packed [H][W] frame; pose7 =
    // {px, py, pz, qx, qy, qz, qw} as geometry_msgs::Pose carries it.  Read the result back with
    // dsmmap_published_points("raw_pointcloud", ...).
    void dsmmap_publish_raw(RefMap *r, const unsigned char *gray, const float *depth, const double *pose7)
    {
        const int W = r->map->cam_width, H = r->map->cam_height;
        cv::Mat image(H, W, CV_8UC1, (void *)gray, (size_t)W), dm(H, W, CV_32FC1, (void *)depth, (size_t)W * 4);
        geometry_msgs::Pose pose;
        pose.position.x = pose7[0], pose.position.y = pose7[1], pose.position.z = pose7[2];
        pose.orientation.x = pose7[3], pose.orientation.y = pose7[4], pose.orientation.z = pose7[5];
        pose.orientation.w = pose7[6];
        r->map->publish_raw_pointcloud(dm, image, pose);
    }
    // get_driftfree_poses(root, out, range) (surfel_map.cpp:1643-1680): the BFS list; returns its length, writes at most cap
    int dsmmap_driftfree_poses(RefMap *r, int root, int range, int *out, int cap)
    {
        std::vector<int> poses;
        r->map->get_driftfree_poses(root, poses, range);
        for (size_t i = 0; i < poses.size() && (int)i < cap; i++) out[i] = poses[i];
        return (int)poses.size();
    }
}
