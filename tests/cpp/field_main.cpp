// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with or without enable_distance_field(), and dumps the field and the node's clouds.
// Usage: field_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive publish voxel nx ny nz
//                   in.bin out.bin out_prefix
//   voxel = 0: no distance field.  publish = 1: enable_publishing() as well (the field is enqueued behind the snapshot).
//   out.bin: after every depth message: with a field, int32 rc of distance_field, double camera[3] (the fuse pose's
//            position), int32 origin[3], int32 n_occupied, the field (int32 n + n floats; n = 0 unless rc is DSM_OK);
//            with publish, int32 rc of published_clouds and the two published clouds; then, always, int32 rc and the
//            clouds of active_points() and inactive_points() read right after (each cloud as int32 n + n points);
//            at the end: local_surfels (int32 n + records) and inactive_points, and the node's save_mesh and save_cloud
//            go to <out_prefix>.ply / <out_prefix>.pcd.
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "driver_io.hpp"

int main(int argc, char **argv)
{
    if (argc != 21) return 2;
    const NodeArgs args(argv, true);
    const int publish = atoi(argv[13]);
    const float voxel = (float)atof(argv[14]);
    const int nx = atoi(argv[15]), ny = atoi(argv[16]), nz = atoi(argv[17]);
    DriverNode node(args);
    if (const int e = setup_code(node.last_error())) return e;
    if (publish && node.enable_publishing() != DSM_OK) return 4;
    if (voxel > 0.f && node.enable_distance_field(voxel, nx, ny, nz) != DSM_OK) return 4;
    if (!open_io(argv[18], argv[19])) return 5;
    const int e = feed_script(node, args.W, args.H, [&]() -> int {
        if (voxel > 0.f)
        {
            const float *dist = nullptr;
            int32_t origin[3] = {0, 0, 0};
            int n_occ = 0;
            const int rc = node.distance_field(dist, origin, n_occ);
            const dsm::Pose cam = node.pose_graph().camera;
            put(rc);
            put(cam.x), put(cam.y), put(cam.z);
            put(origin[0]), put(origin[1]), put(origin[2]);
            put(n_occ);
            put_n(dist, rc == DSM_OK ? nx * ny * nz : 0);
        }
        if (publish)
        {
            const dsm_point_t *a = nullptr, *b = nullptr;
            int na = 0, nb = 0, from = 0;
            const int rc = node.published_clouds(a, na, b, nb, from);
            put(rc);
            put_n(a, rc == DSM_OK ? na : 0);
            put_n(b, rc == DSM_OK ? nb : 0);
        }
        put_clouds(node);
        return 0;
    });
    if (e) return e;
    if (!put_final(node) || !save_files(node, argv[20])) return 6;
    return close_io();
}
