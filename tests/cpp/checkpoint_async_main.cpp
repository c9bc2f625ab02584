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
#include "driver_io.hpp"

int main(int argc, char **argv)
{
    if (argc != 16) return 2;
    const NodeArgs args(argv, false);
    const int W = args.W, H = args.H, j = atoi(argv[10]);
    const std::string ckpt = argv[11], twin_ckpt = argv[12], dir = argv[15];
    DriverNode a(args);
    if (const int e = setup_code(a.last_error())) return e;
    DriverNode t(args);
    if (!open_io(argv[13], argv[14])) return 5;
    NodeMessages msg;
    int type = 0, ra = DSM_OK, rt = DSM_OK;
    for (int m = 0; m < j; m++)
    {
        if (!get(type) || !msg.feed_both(a, t, type, W, H, ra, rt) || ra != DSM_OK || rt != DSM_OK) return 5;
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
    DriverNode b(args);
    put(b.load_state(ckpt));
    put((int)(digest(b) == digest(t)));
    fseek(in_f, at_j, SEEK_SET);
    while (get(type))
    {
        int rb = DSM_OK;
        if (!msg.feed_both(b, t, type, W, H, rb, rt)) return 5;
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
    return close_io();
}
