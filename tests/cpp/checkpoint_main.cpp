// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only),
// checkpoints node A after message j, resumes node B from the file, and feeds both the remaining messages.
// Usage: checkpoint_main W H fx fy cx cy far near drift_free_poses j ckpt in.bin out.bin dir
//   out.bin: int32 rc of A.save_state, int32 rc of B.load_state, int32 B equals A right after the load;
//            per message after j: int32 rc of A, int32 rc of B, int32 B equals A (1) after it;
//            int32 rc and int32 unchanged (1) of a load into a node whose drift_free_poses differ, and of A loading a
//            file without a node section; int32 rc of the four files A and B write at the end into dir:
//            a.ply, b.ply (save_mesh), a.pcd, b.pcd (save_cloud).
//   "equals": every reader agrees byte for byte: local_surfels, attached_surfels of every pose, poses() (cam_pose,
//   loop_pose, cam_stamp, links), local_surfels_indexs(), pending_frame(), last_warp() and pose_graph().
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include <string>
#include "dsm_surfel_node.hpp"
#include "driver_io.hpp"

template <class T>
static void add(std::vector<uint8_t> &d, const T *p, size_t n)
{
    const uint8_t *b = reinterpret_cast<const uint8_t *>(p);
    d.insert(d.end(), b, b + n * sizeof(T));
}
template <class T>
static void add_list(std::vector<uint8_t> &d, const std::vector<T> &v)
{
    const int n = (int)v.size();
    add(d, &n, 1);
    add(d, v.data(), v.size());
}

// everything the node reads back, as bytes
static std::vector<uint8_t> digest(dsm::SurfelMapNode &node)
{
    std::vector<uint8_t> d;
    std::vector<dsm_surfel_t> s;
    int rc = node.local_surfels(s);
    add(d, &rc, 1);
    add_list(d, s);
    const std::vector<dsm::NodePose> &p = node.poses();
    for (size_t i = 0; i < p.size(); i++)
    {
        rc = node.attached_surfels((int)i, s);
        add(d, &rc, 1);
        add_list(d, s);
        add(d, &p[i].cam_pose, 1);
        add(d, &p[i].loop_pose, 1);
        add(d, &p[i].cam_stamp, 1);
        add_list(d, p[i].linked_pose_index);
    }
    add_list(d, std::vector<int>(node.local_surfels_indexs().begin(), node.local_surfels_indexs().end()));
    float pose16[16] = {0};
    std::vector<int> rem, add_;
    const int pref = node.pending_frame(pose16, rem, add_);
    add(d, &pref, 1);
    add(d, pose16, 16);
    add_list(d, rem);
    add_list(d, add_);
    add_list(d, node.last_warp());
    const dsm::NodePoseGraph g = node.pose_graph();
    add_list(d, g.path);
    add_list(d, g.loop_edges);
    add_list(d, g.driftfree);
    add_list(d, g.drift);
    add(d, &g.camera, 1);
    return d;
}

int main(int argc, char **argv)
{
    if (argc != 15) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]), dfp = atoi(argv[9]), j = atoi(argv[10]);
    const double fx = atof(argv[3]), fy = atof(argv[4]), cx = atof(argv[5]), cy = atof(argv[6]), fr = atof(argv[7]), nr = atof(argv[8]);
    const std::string ckpt = argv[11], dir = argv[14];
    const int max_local = 1 << 20, max_inactive = 1 << 21;
    dsm::SurfelMapNode a(W, H, fx, fy, cx, cy, fr, nr, dfp, 0, max_local, max_inactive);
    if (a.last_error() != DSM_OK) return a.last_error() == DSM_E_NODEVICE ? 3 : 4;
    in_f = fopen(argv[12], "rb");
    out_f = fopen(argv[13], "wb");
    if (!in_f || !out_f) return 5;
    NodeMessages msg;
    int type = 0, r = DSM_OK;
    for (int m = 0; m < j; m++)
    {
        if (!get(type) || !msg.feed(a, type, W, H, r) || r != DSM_OK) return 5;
    }
    put(a.save_state(ckpt));
    dsm::SurfelMapNode b(W, H, fx, fy, cx, cy, fr, nr, dfp, 0, max_local, max_inactive);
    put(b.load_state(ckpt));
    put((int)(digest(a) == digest(b)));
    while (get(type))
    {
        const long at = ftell(in_f);
        int ra = DSM_OK, rb = DSM_OK;
        if (!msg.feed(a, type, W, H, ra)) return 5;
        fseek(in_f, at, SEEK_SET);
        if (!msg.feed(b, type, W, H, rb)) return 5;
        put(ra);
        put(rb);
        put((int)(digest(a) == digest(b)));
    }
    // a node with other parameters, fed the same first j messages: the load is refused and changes nothing
    dsm::SurfelMapNode c(W, H, fx, fy, cx, cy, fr, nr, dfp + 1, 0, max_local, max_inactive);
    fseek(in_f, 0, SEEK_SET);
    for (int m = 0; m < j; m++)
    {
        if (!get(type) || !msg.feed(c, type, W, H, r) || r != DSM_OK) return 5;
    }
    std::vector<uint8_t> before = digest(c);
    put(c.load_state(ckpt));
    put((int)(before == digest(c)));
    // a file without a node section: the map of A saved with no extra bytes, loaded into A
    const std::string bare = ckpt + ".bare";
    if (dsm_map_save(a.context(), bare.c_str(), nullptr, 0) != DSM_OK) return 6;
    before = digest(a);
    put(a.load_state(bare));
    put((int)(before == digest(a)));
    int rs = a.save_mesh(dir + "/a.ply");
    if (rs == DSM_OK) rs = b.save_mesh(dir + "/b.ply");
    if (rs == DSM_OK) rs = a.save_cloud(dir + "/a.pcd");
    if (rs == DSM_OK) rs = b.save_cloud(dir + "/b.pcd");
    put(rs);
    fclose(in_f);
    fclose(out_f);
    return 0;
}
