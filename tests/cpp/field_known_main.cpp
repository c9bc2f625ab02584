// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with a distance field, with or without enable_known_space(), and dumps the known field with the views it carried and
// the node's clouds.  After depth message `reload_at` the node saves its state and loads it back.
// Usage: field_known_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive voxel nx ny nz
//                         max_views max_range reload_at in.bin out.bin out_prefix
//   max_views = 0: no known space (the plain field is requested and not dumped).
//   out.bin: after every depth message: with known space, int32 rc of distance_field, double camera[3] (the fuse pose's
//            position), int32 origin[3], int32 n_occupied, the distance grid (int32 n + n floats), the state grid (int32
//            n + n bytes), int32 n_free, then int32 n_views and per view the seeds of its captured frame (int32 n + n
//            dsm_seed_t) and its pose (12 doubles, row-major [R | t]); then, always, int32 rc and the clouds of
//            active_points() and inactive_points() (each int32 n + n points); at the end: local_surfels (int32 n +
//            records), and the node's save_mesh and save_cloud go to <out_prefix>.ply / <out_prefix>.pcd.
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "driver_io.hpp"

int main(int argc, char **argv)
{
    if (argc != 23) return 2;
    const NodeArgs args(argv, true);
    const FieldArgs field(argv);
    const int max_views = field.max_views, reload_at = atoi(argv[19]);
    DriverNode node(args);
    if (const int e = setup_code(node.last_error())) return e;
    if (const int e = field.enable(node)) return e;
    if (!open_io(argv[20], argv[21])) return 5;
    const std::string prefix = argv[22];
    const int S = dsm_num_seeds(node.context());
    std::vector<std::vector<dsm_seed_t> > seeds((size_t)(max_views > 0 ? max_views : 0)); // per slot, of its captured frame
    std::vector<int32_t> slots;
    std::vector<double> poses;
    int depth_msgs = 0, fused = 0, captures = 0;
    const int e = feed_script(node, args.W, args.H, [&]() -> int {
        const FieldHandout h(node, max_views > 0, true);
        fused += h.rc != DSM_E_STATE; // every fused frame requests a field
        if (max_views > 0)
        {
            const int now = node.known_views(slots, poses);
            if (now != captures)
            { // the frame just fused was captured: its seeds are in the frame slot of the node's latest single-frame
              // call, which alternates between the context's two staging halves (max_batch 2) from the first call on
                std::vector<dsm_seed_t> &s = seeds[(size_t)((now - 1) % max_views)];
                s.resize((size_t)S);
                if (dsm_get_seeds(node.context(), (fused - 1) & 1, s.data()) != DSM_OK) return 6;
                captures = now;
            }
            const dsm::Pose cam = node.pose_graph().camera;
            put(first_error({h.rc, h.rs}));
            put(cam.x), put(cam.y), put(cam.z);
            h.put_origin();
            put(h.n_occ);
            put_n(h.dist, h.rc == DSM_OK ? field.cells() : 0);
            h.put_state(field);
            put(h.n_free);
            put((int32_t)slots.size());
            for (size_t j = 0; j < slots.size(); j++)
            {
                put_list(seeds[(size_t)slots[j]]);
                put_n(poses.data() + 12 * j, 12);
            }
        }
        put_clouds(node);
        if (++depth_msgs == reload_at)
        {
            if (!reload(node, prefix)) return 6;
            captures = 0; // load_state empties the slot table
        }
        return 0;
    });
    return e ? e : end_drive(node, prefix);
}
