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
#include "driver_io.hpp"

int main(int argc, char **argv)
{
    if (argc != 15) return 2;
    const NodeArgs args(argv, false);
    const int W = args.W, H = args.H, j = atoi(argv[10]);
    const std::string ckpt = argv[11], dir = argv[14];
    DriverNode a(args);
    if (const int e = setup_code(a.last_error())) return e;
    if (!open_io(argv[12], argv[13])) return 5;
    NodeMessages msg;
    int type = 0, r = DSM_OK;
    for (int m = 0; m < j; m++)
    {
        if (!get(type) || !msg.feed(a, type, W, H, r) || r != DSM_OK) return 5;
    }
    put(a.save_state(ckpt));
    DriverNode b(args);
    put(b.load_state(ckpt));
    put((int)(digest(a) == digest(b)));
    while (get(type))
    {
        int ra = DSM_OK, rb = DSM_OK;
        if (!msg.feed_both(a, b, type, W, H, ra, rb)) return 5;
        put(ra);
        put(rb);
        put((int)(digest(a) == digest(b)));
    }
    // a node with other parameters, fed the same first j messages: the load is refused and changes nothing
    NodeArgs other = args;
    other.dfp++;
    DriverNode c(other);
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
    return close_io();
}
