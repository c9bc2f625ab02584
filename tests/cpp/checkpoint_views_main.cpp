// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with known space and frontiers on node A, which saves its state after depth message `save_at`; node B, built the same
// way, loads that file and from then on receives every message A receives.  Checks that a resumed node is the node that
// saved (DESIGN.md §8.18) when both call enable_view_checkpoints(), and what happens when only one of them does.
// Usage: checkpoint_views_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive voxel nx ny nz
//                              max_views max_range save_at mode a_views b_views in.bin out.bin out_prefix
//   mode 0: save_state; 1: save_state_async, then A receives the messages up to its next depth message before it
//           waits, and B, once loaded, receives those messages too; 2: save_state_incremental after every third depth
//           message and at save_at, each waited for, and B loads with load_state_incremental.
//   a_views / b_views: 1 when the node calls enable_view_checkpoints().
//   out.bin: int32 rc of the save, int32 rc of B's load, then for A and for B: int32 captures and the known views
//            (int32 n + n slots, int32 n + n doubles); after every later depth message, for A and then B: int32 rc (of the
//            field handout or frontiers()), the distance grid and the state grid (each int32 n + n values, empty unless
//            rc is 0), the frontier clusters and voxels (int32 n + n each), and put_clouds; at the end A's and B's
//            local_surfels (int32 n + records), and save_mesh / save_cloud to <out_prefix>a|b.ply / .pcd.  When B's load
//            fails, out.bin ends after the views and B's digest is compared with a fresh node's: int32 1 when equal.
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include <memory>

#include "driver_io.hpp"

namespace
{
int enable_all(DriverNode &node, const FieldArgs &field, bool views)
{
    if (const int e = setup_code(node.last_error())) return e;
    if (const int e = field.enable(node)) return e;
    if (node.enable_frontiers(256, 1 << 18) != DSM_OK || node.enable_checkpoints() != DSM_OK) return 4;
    if (views && node.enable_view_checkpoints() != DSM_OK) return 4;
    return 0;
}

void put_views(dsm::SurfelMapNode &node)
{
    std::vector<int32_t> slots;
    std::vector<double> poses;
    put((int32_t)node.known_views(slots, poses));
    put_list(slots);
    put_list(poses);
}

// the known field of the frame just fused, its frontiers and the clouds
void put_frame(dsm::SurfelMapNode &node, const FieldArgs &field)
{
    static std::vector<dsm_frontier_cluster_t> clusters;
    static std::vector<int32_t> voxels;
    dsm_frontier_counts_t counts = dsm_frontier_counts_t();
    const int rf = node.frontiers(1, clusters, voxels, counts);
    const FieldHandout h(node, true);
    const int rc = first_error({h.rc, h.rs, rf});
    put(rc);
    put_n(h.dist, rc == DSM_OK ? field.cells() : 0);
    h.put_state(field);
    put_list(clusters);
    put_list(voxels);
    put_clouds(node);
}
} // namespace

int main(int argc, char **argv)
{
    if (argc != 26) return 2;
    const NodeArgs args(argv, true);
    const FieldArgs field(argv);
    const int save_at = atoi(argv[19]), mode = atoi(argv[20]);
    const bool a_views = atoi(argv[21]) != 0, b_views = atoi(argv[22]) != 0;
    DriverNode a(args);
    if (const int e = enable_all(a, field, a_views)) return e;
    if (!open_io(argv[23], argv[24])) return 5;
    const std::string prefix = argv[25], state = prefix + ".state";
    std::unique_ptr<DriverNode> b;
    NodeMessages msg;
    int type = 0, ra = DSM_OK, rb = DSM_OK, depth_msgs = 0;
    long replay_from = -1; // save_state_async: where B's catch-up starts
    int rc_save = DSM_OK;
    while (get(type))
    {
        if (b)
        {
            if (!msg.feed_both(a, *b, type, args.W, args.H, ra, rb)) return 5;
            if (ra != DSM_OK || rb != DSM_OK) return 6;
        }
        else
        {
            if (!msg.feed(a, type, args.W, args.H, ra)) return 5;
            if (ra != DSM_OK) return 6;
        }
        if (type != 2) continue;
        ++depth_msgs;
        if (b)
        {
            put_frame(a, field);
            put_frame(*b, field);
            continue;
        }
        if (mode == 2 && (depth_msgs % 3 == 0 || depth_msgs == save_at) && depth_msgs <= save_at)
        {
            rc_save = a.save_state_incremental(state);
            if (rc_save == DSM_OK) rc_save = a.wait_state_saved(true, nullptr);
            if (rc_save != DSM_OK) return 6;
        }
        if (depth_msgs == save_at && mode == 0) rc_save = a.save_state(state);
        if (depth_msgs == save_at && mode == 1)
        {
            rc_save = a.save_state_async(state);
            replay_from = ftell(in_f);
            continue; // A fuses on while the file is written
        }
        const bool load_now = depth_msgs == save_at || (mode == 1 && depth_msgs == save_at + 1);
        if (!load_now) continue;
        if (mode == 1)
        {
            const int rw = a.wait_state_saved(true, nullptr);
            if (rc_save == DSM_OK) rc_save = rw;
        }
        b.reset(new DriverNode(args));
        if (const int e = enable_all(*b, field, b_views)) return e;
        const std::vector<uint8_t> fresh = digest(*b);
        const int rc_load = mode == 2 ? b->load_state_incremental(state) : b->load_state(state);
        put(rc_save), put(rc_load);
        if (mode == 1 && rc_load == DSM_OK)
        { // B catches up with the messages A received while the file was written
            const long at = ftell(in_f);
            fseek(in_f, replay_from, SEEK_SET);
            while (ftell(in_f) < at)
            {
                if (!get(type) || !msg.feed(*b, type, args.W, args.H, rb)) return 5;
                if (rb != DSM_OK) return 6;
            }
        }
        put_views(a);
        put_views(*b);
        if (rc_load != DSM_OK)
        {
            put((int32_t)(digest(*b) == fresh));
            return close_io();
        }
    }
    std::vector<dsm_surfel_t> local;
    if (!b || a.local_surfels(local) != DSM_OK) return 6;
    put_list(local);
    if (!save_files(a, prefix + "a")) return 6;
    return end_drive(*b, prefix + "b");
}
