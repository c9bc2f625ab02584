// Drives include/dsm_surfel_node.hpp through a binary message script and dumps the node's state where the script asks.
// Usage: node_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive rgbd in.bin out.bin
//   device < 0: pose logic only (no context; images count for their stamps alone, dumps must not ask for the map).  rgbd = 1: DSM_CONSTANTS_RGBD.
//   in.bin : messages until EOF, each int32 type then
//     0 orb    double stamp, int32 is_keyframe, int32 reference_index, double pose7[7], int32 n_path, double path7[n_path][7],
//              int32 n_loops, int32 pairs[2 n_loops]
//     1 image  double stamp, uint8 gray[H*W]
//     2 depth  double stamp, float depth[H*W]
//     3 dump   int32 what (bit 0: poses, bit 1: map), int32 neighbor_reference
//     4 save   int32 n, char mesh_path[n], int32 m, char cloud_path[m]
//   out.bin: per dump, int32 rc (first error code of the messages since the previous dump, 0 if none), then
//     poses: int32 n; n x { double cam[7], double loop[7], int32 n_links, int32 links[] }; int32 n_local, local[];
//            int32 pending_ref, float pending_pose[16], list remove, list add;
//            per pose r: list driftfree_poses(r, drift_free_poses), list remove(r), list add(r);
//            int32 n_warp, n_warp x { int32 pose, float W[16] }; double last_fuse_pose[7] (zeros before the first fuse)
//            (list = int32 n, int32[n])
//     map:   int32 rc, then local surfels, attached surfels of every pose, active, inactive, all and neighbour points,
//            each as int32 n + records
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include <string>
#include "dsm_surfel_node.hpp"
#include "driver_io.hpp"

static void put_pose(const dsm::Pose &p)
{
    const double d[7] = {p.x, p.y, p.z, p.qx, p.qy, p.qz, p.qw};
    fwrite(d, 8, 7, out_f);
}

int main(int argc, char **argv)
{
    if (argc != 16) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]), dfp = atoi(argv[9]), device = atoi(argv[10]);
    const dsm_constants rgbd = DSM_CONSTANTS_RGBD;
    dsm::SurfelMapNode node(W, H, atof(argv[3]), atof(argv[4]), atof(argv[5]), atof(argv[6]), atof(argv[7]), atof(argv[8]), dfp, device,
                            atoi(argv[11]), atoi(argv[12]), atoi(argv[13]) ? &rgbd : nullptr);
    if (node.last_error() != DSM_OK) return node.last_error() == DSM_E_NODEVICE ? 3 : 4;
    in_f = fopen(argv[14], "rb");
    out_f = fopen(argv[15], "wb");
    if (!in_f || !out_f) return 5;
    NodeMessages msg;
    int rc = DSM_OK, type = 0;
    while (get(type))
    {
        int r = DSM_OK;
        if (type <= 2)
        {
            if (!msg.feed(node, type, W, H, r)) return 5;
        }
        else if (type == 3)
        {
            int what = 0, nref = 0;
            if (!get(what) || !get(nref)) return 5;
            put(rc);
            rc = DSM_OK;
            if (what & 1)
            {
                const std::vector<dsm::NodePose> &p = node.poses();
                put((int)p.size());
                for (size_t i = 0; i < p.size(); i++)
                {
                    put_pose(p[i].cam_pose);
                    put_pose(p[i].loop_pose);
                    put_list(p[i].linked_pose_index);
                }
                put_list(std::vector<int>(node.local_surfels_indexs().begin(), node.local_surfels_indexs().end()));
                float pose16[16];
                std::vector<int> rem, add;
                const int pref = node.pending_frame(pose16, rem, add);
                put(pref);
                if (pref < 0) std::fill(pose16, pose16 + 16, 0.f);
                fwrite(pose16, 4, 16, out_f);
                put_list(rem);
                put_list(add);
                for (int root = 0; root < (int)p.size(); root++)
                {
                    put_list(node.driftfree_poses(root, dfp));
                    node.window_lists(root, rem, add);
                    put_list(rem);
                    put_list(add);
                }
                put((int)node.last_warp().size());
                for (size_t i = 0; i < node.last_warp().size(); i++)
                {
                    put(node.last_warp()[i].pose);
                    fwrite(node.last_warp()[i].W, 4, 16, out_f);
                }
                put_pose(node.pose_graph().camera);
            }
            if (what & 2)
            {
                std::vector<dsm_surfel_t> local;
                std::vector<std::vector<dsm_surfel_t> > attached(node.poses().size());
                std::vector<dsm_point_t> clouds[4];
                int mr = node.local_surfels(local);
                for (size_t i = 0; i < attached.size() && mr == DSM_OK; i++) mr = node.attached_surfels((int)i, attached[i]);
                if (mr == DSM_OK) mr = node.active_points(clouds[0]);
                if (mr == DSM_OK) mr = node.inactive_points(clouds[1]);
                if (mr == DSM_OK) mr = node.all_points(clouds[2]);
                if (mr == DSM_OK) mr = node.neighbor_points(nref, clouds[3]);
                put(mr);
                put_list(local);
                for (size_t i = 0; i < attached.size(); i++) put_list(attached[i]);
                for (int c = 0; c < 4; c++) put_list(clouds[c]);
            }
            fflush(out_f);
        }
        else if (type == 4)
        {
            int n = 0;
            std::vector<char> a, b;
            if (!get(n) || !get_n(a, n) || !get(n) || !get_n(b, n)) return 5;
            r = node.save_mesh(std::string(a.begin(), a.end()));
            if (r == DSM_OK) r = node.save_cloud(std::string(b.begin(), b.end()));
        }
        else
            return 5;
        if (rc == DSM_OK) rc = r;
    }
    fclose(in_f);
    fclose(out_f);
    return 0;
}
