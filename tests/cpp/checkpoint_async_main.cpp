// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only) and
// checkpoints without stopping the node: node A calls save_state_async after message j and keeps receiving every later
// message while the file is written, polling wait_state_saved(false, ...) after each; twin T calls save_state after
// message j and then waits; node B loads A's file and, with T, receives the messages after j.
// Usage: checkpoint_async_main W H fx fy cx cy far near drift_free_poses j ckpt_async ckpt_twin in.bin out.bin dir
//   out.bin: int32 rc of A.enable_checkpoints, of A.save_state_async, of T.save_state;
//            per message after j: int32 rc of A;
//            int32 rc of the write (the wait that reported it finished), int32 messages A received before it finished;
//            int32 rc of B.load_state, int32 B equals T right after the load;
//            per message after j: int32 rc of B, int32 rc of T, int32 B equals T (1) after it;
//            int32 A equals T (1) at the end; int32 rc of the six files A, B and T write into dir: a.ply, b.ply,
//            t.ply (save_mesh), a.pcd, b.pcd, t.pcd (save_cloud).
//   "equals": every reader agrees byte for byte, as in checkpoint_main.cpp.
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

// everything the node reads back, as bytes (checkpoint_main.cpp's digest)
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
    if (argc != 16) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]), dfp = atoi(argv[9]), j = atoi(argv[10]);
    const double fx = atof(argv[3]), fy = atof(argv[4]), cx = atof(argv[5]), cy = atof(argv[6]), fr = atof(argv[7]), nr = atof(argv[8]);
    const std::string ckpt = argv[11], twin_ckpt = argv[12], dir = argv[15];
    const int max_local = 1 << 20, max_inactive = 1 << 21;
    dsm::SurfelMapNode a(W, H, fx, fy, cx, cy, fr, nr, dfp, 0, max_local, max_inactive);
    if (a.last_error() != DSM_OK) return a.last_error() == DSM_E_NODEVICE ? 3 : 4;
    dsm::SurfelMapNode t(W, H, fx, fy, cx, cy, fr, nr, dfp, 0, max_local, max_inactive);
    in_f = fopen(argv[13], "rb");
    out_f = fopen(argv[14], "wb");
    if (!in_f || !out_f) return 5;
    NodeMessages msg;
    int type = 0, r = DSM_OK;
    for (int m = 0; m < j; m++)
    {
        const long at = ftell(in_f);
        if (!get(type) || !msg.feed(a, type, W, H, r) || r != DSM_OK) return 5;
        fseek(in_f, at, SEEK_SET);
        if (!get(type) || !msg.feed(t, type, W, H, r) || r != DSM_OK) return 5;
    }
    const long at_j = ftell(in_f);
    put(a.enable_checkpoints());
    put(a.save_state_async(ckpt));
    put(t.save_state(twin_ckpt));
    // A goes on while its checkpoint is written
    bool finished = false;
    int wrc = DSM_OK, before_done = 0;
    while (get(type))
    {
        int ra = DSM_OK;
        if (!msg.feed(a, type, W, H, ra)) return 5;
        put(ra);
        if (!finished)
        {
            wrc = a.wait_state_saved(false, &finished);
            if (wrc != DSM_OK && !finished) return 6;
            before_done++;
        }
    }
    if (!finished) wrc = a.wait_state_saved(true, &finished);
    put(wrc);
    put(before_done);
    // B resumes from A's file; T, held at message j, is the uninterrupted node
    dsm::SurfelMapNode b(W, H, fx, fy, cx, cy, fr, nr, dfp, 0, max_local, max_inactive);
    put(b.load_state(ckpt));
    put((int)(digest(b) == digest(t)));
    fseek(in_f, at_j, SEEK_SET);
    while (get(type))
    {
        const long at = ftell(in_f);
        int rb = DSM_OK, rt = DSM_OK;
        if (!msg.feed(b, type, W, H, rb)) return 5;
        fseek(in_f, at, SEEK_SET);
        if (!msg.feed(t, type, W, H, rt)) return 5;
        put(rb);
        put(rt);
        put((int)(digest(b) == digest(t)));
    }
    put((int)(digest(a) == digest(t)));
    int rs = a.save_mesh(dir + "/a.ply");
    if (rs == DSM_OK) rs = b.save_mesh(dir + "/b.ply");
    if (rs == DSM_OK) rs = t.save_mesh(dir + "/t.ply");
    if (rs == DSM_OK) rs = a.save_cloud(dir + "/a.pcd");
    if (rs == DSM_OK) rs = b.save_cloud(dir + "/b.pcd");
    if (rs == DSM_OK) rs = t.save_cloud(dir + "/t.pcd");
    put(rs);
    fclose(in_f);
    fclose(out_f);
    return 0;
}
