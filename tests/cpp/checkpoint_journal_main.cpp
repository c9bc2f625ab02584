// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only) and
// checkpoints incrementally: node A calls save_state_incremental after every `every` messages and after message j,
// feeding the next messages while each save is written and waiting for it right before the next one; twin T receives the
// same messages without saving; node B loads A's base and journal after message j and, with T, receives the rest.
// Usage: checkpoint_journal_main W H fx fy cx cy far near drift_free_poses every j ckpt in.bin out.bin dir
//   out.bin: int32 rc of A.enable_checkpoints, int32 T.last_error();
//            per save: int32 rc of the save (save_state_incremental, then the wait that retired it), int32 journal
//            records the files resolve with after it (dsm_map_peek_journal);
//            int32 rc of B.load_state_incremental, int32 records it applied, int32 B equals T right after the load;
//            per message after j: int32 rc of B, int32 rc of T, int32 B equals T (1) after it;
//            int32 rc of the four files B and T write into dir: b.ply, t.ply (save_mesh), b.pcd, t.pcd (save_cloud).
//   "equals": every reader agrees byte for byte, as in checkpoint_async_main.cpp.
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

// retires A's pending save and reports it with the records the files now resolve with
static void retire(dsm::SurfelMapNode &a, const std::string &ckpt)
{
    bool finished = false;
    put(a.wait_state_saved(true, &finished));
    int records = 0;
    dsm_map_peek_journal(ckpt.c_str(), nullptr, 0, nullptr, nullptr, 0, nullptr, &records);
    put(records);
}

int main(int argc, char **argv)
{
    if (argc != 16) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]), dfp = atoi(argv[9]), every = atoi(argv[10]), j = atoi(argv[11]);
    const double fx = atof(argv[3]), fy = atof(argv[4]), cx = atof(argv[5]), cy = atof(argv[6]), fr = atof(argv[7]), nr = atof(argv[8]);
    const std::string ckpt = argv[12], dir = argv[15];
    if (every < 1) return 2;
    const int max_local = 1 << 20, max_inactive = 1 << 21;
    dsm::SurfelMapNode a(W, H, fx, fy, cx, cy, fr, nr, dfp, 0, max_local, max_inactive);
    if (a.last_error() != DSM_OK) return a.last_error() == DSM_E_NODEVICE ? 3 : 4;
    dsm::SurfelMapNode t(W, H, fx, fy, cx, cy, fr, nr, dfp, 0, max_local, max_inactive);
    in_f = fopen(argv[13], "rb");
    out_f = fopen(argv[14], "wb");
    if (!in_f || !out_f) return 5;
    put(a.enable_checkpoints());
    put(t.last_error());
    NodeMessages msg;
    int type = 0, r = DSM_OK;
    bool pending = false;
    for (int m = 1; m <= j; m++)
    {
        const long at = ftell(in_f);
        if (!get(type) || !msg.feed(a, type, W, H, r) || r != DSM_OK) return 5;
        fseek(in_f, at, SEEK_SET);
        if (!get(type) || !msg.feed(t, type, W, H, r) || r != DSM_OK) return 5;
        if (m % every != 0 && m != j) continue;
        if (pending) retire(a, ckpt);
        const int rc = a.save_state_incremental(ckpt);
        pending = rc == DSM_OK;
        if (!pending)
        {
            put(rc);
            put(0);
        }
    }
    if (pending) retire(a, ckpt);
    // B resumes from A's base and journal; T, held at message j, is the uninterrupted node
    dsm::SurfelMapNode b(W, H, fx, fy, cx, cy, fr, nr, dfp, 0, max_local, max_inactive);
    int records = -1;
    put(b.load_state_incremental(ckpt, &records));
    put(records);
    put((int)(digest(b) == digest(t)));
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
    int rs = b.save_mesh(dir + "/b.ply");
    if (rs == DSM_OK) rs = t.save_mesh(dir + "/t.ply");
    if (rs == DSM_OK) rs = b.save_cloud(dir + "/b.pcd");
    if (rs == DSM_OK) rs = t.save_cloud(dir + "/t.pcd");
    put(rs);
    fclose(in_f);
    fclose(out_f);
    return 0;
}
