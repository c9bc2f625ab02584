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
#include "dsm_surfel_node.hpp"
#include "driver_io.hpp"
#include <string>

int main(int argc, char **argv)
{
    if (argc != 23) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]);
    const float voxel = (float)atof(argv[13]);
    const int nx = atoi(argv[14]), ny = atoi(argv[15]), nz = atoi(argv[16]);
    const int max_views = atoi(argv[17]), reload_at = atoi(argv[19]);
    dsm::SurfelMapNode node(W, H, atof(argv[3]), atof(argv[4]), atof(argv[5]), atof(argv[6]), atof(argv[7]), atof(argv[8]), atoi(argv[9]),
                            atoi(argv[10]), atoi(argv[11]), atoi(argv[12]), nullptr);
    if (node.last_error() != DSM_OK) return node.last_error() == DSM_E_NODEVICE ? 3 : 4;
    if (node.enable_distance_field(voxel, nx, ny, nz) != DSM_OK) return 4;
    if (max_views > 0 && node.enable_known_space(max_views, (float)atof(argv[18])) != DSM_OK) return 4;
    in_f = fopen(argv[20], "rb");
    out_f = fopen(argv[21], "wb");
    if (!in_f || !out_f) return 5;
    const std::string prefix = argv[22];
    const int S = dsm_num_seeds(node.context());
    std::vector<std::vector<dsm_seed_t> > seeds((size_t)(max_views > 0 ? max_views : 0)); // per slot, of its captured frame
    std::vector<int32_t> slots;
    std::vector<double> poses;
    NodeMessages msg;
    std::vector<dsm_point_t> act, inact;
    int type = 0, r = DSM_OK, depth_msgs = 0, fused = 0, captures = 0;
    while (get(type))
    {
        if (!msg.feed(node, type, W, H, r)) return 5;
        if (r != DSM_OK) return 6;
        if (type != 2) continue;
        const float *dist = nullptr;
        int32_t origin[3] = {0, 0, 0};
        int n_occ = 0;
        const int rc = node.distance_field(dist, origin, n_occ);
        fused += rc != DSM_E_STATE; // every fused frame requests a field
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
            const uint8_t *state = nullptr;
            int n_free = 0;
            const int rs = rc == DSM_OK || rc == DSM_E_CAPACITY ? node.known_space(state, n_free) : rc;
            const dsm::Pose cam = node.pose_graph().camera;
            put(rc != DSM_OK ? rc : rs);
            put(cam.x), put(cam.y), put(cam.z);
            put(origin[0]), put(origin[1]), put(origin[2]);
            put(n_occ);
            put_n(dist, rc == DSM_OK ? nx * ny * nz : 0);
            put_n(state, rc == DSM_OK && rs == DSM_OK ? nx * ny * nz : 0);
            put(n_free);
            put((int32_t)slots.size());
            for (size_t j = 0; j < slots.size(); j++)
            {
                put_list(seeds[(size_t)slots[j]]);
                put_n(poses.data() + 12 * j, 12);
            }
        }
        int rr = node.active_points(act);
        if (rr == DSM_OK) rr = node.inactive_points(inact);
        put(rr);
        put_list(act);
        put_list(inact);
        if (++depth_msgs == reload_at)
        {
            if (node.save_state(prefix + ".state") != DSM_OK || node.load_state(prefix + ".state") != DSM_OK) return 6;
            captures = 0; // load_state empties the slot table
        }
    }
    std::vector<dsm_surfel_t> local;
    if (node.local_surfels(local) != DSM_OK) return 6;
    put_list(local);
    if (node.save_mesh(prefix + ".ply") != DSM_OK || node.save_cloud(prefix + ".pcd") != DSM_OK) return 6;
    fclose(in_f);
    fclose(out_f);
    return 0;
}
