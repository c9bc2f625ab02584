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
#include "driver_io.hpp"

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
    const NodeArgs args(argv, false);
    const int W = args.W, H = args.H, every = atoi(argv[10]), j = atoi(argv[11]);
    const std::string ckpt = argv[12], dir = argv[15];
    if (every < 1) return 2;
    DriverNode a(args);
    if (const int e = setup_code(a.last_error())) return e;
    DriverNode t(args);
    if (!open_io(argv[13], argv[14])) return 5;
    put(a.enable_checkpoints());
    put(t.last_error());
    NodeMessages msg;
    int type = 0, ra = DSM_OK, rt = DSM_OK;
    bool pending = false;
    for (int m = 1; m <= j; m++)
    {
        if (!get(type) || !msg.feed_both(a, t, type, W, H, ra, rt) || ra != DSM_OK || rt != DSM_OK) return 5;
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
    DriverNode b(args);
    int records = -1;
    put(b.load_state_incremental(ckpt, &records));
    put(records);
    put((int)(digest(b) == digest(t)));
    while (get(type))
    {
        int rb = DSM_OK;
        if (!msg.feed_both(b, t, type, W, H, rb, rt)) return 5;
        put(rb);
        put(rt);
        put((int)(digest(b) == digest(t)));
    }
    int rs = b.save_mesh(dir + "/b.ply");
    if (rs == DSM_OK) rs = t.save_mesh(dir + "/t.ply");
    if (rs == DSM_OK) rs = b.save_cloud(dir + "/b.pcd");
    if (rs == DSM_OK) rs = t.save_cloud(dir + "/t.pcd");
    put(rs);
    return close_io();
}
