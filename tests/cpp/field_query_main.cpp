// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with a resident distance field and planner queries after every frame, or without a field, and dumps the queries'
// inputs and results and the node's clouds.
// Usage: field_query_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive queries voxel nx ny nz
//                         in.bin out.bin out_prefix
//   voxel = 0: no distance field.  queries = 1: enable_distance_field(..., host_copy = false) and enable_field_queries.
//   out.bin: after every depth message: with a field, int32 rc of distance_field, double camera[3] (the fuse pose's
//            position), int32 origin[3], int32 n_occupied; with queries, int32 rc of field_samples, the points (int32
//            3n + 3n doubles) and the samples (int32 n + n records), int32 rc of trajectory_clearance, float step,
//            float radius, the waypoints (int32 3w + 3w doubles), the offsets (int32 t + 1 + t + 1 ints) and the
//            clearances (int32 t + t records); then, always, int32 rc and the clouds of active_points() and
//            inactive_points() read right after (each cloud as int32 n + n points);
//            at the end: local_surfels (int32 n + records) and inactive_points, and the node's save_mesh and save_cloud
//            go to <out_prefix>.ply / <out_prefix>.pcd.
// The points and waypoints are drawn from a fixed generator over the grid's box (one voxel beyond it on every side).
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "driver_io.hpp"

static uint64_t rng_state = 0x9e3779b97f4a7c15ull;
static double uniform() // splitmix64, 53 bits
{
    uint64_t z = (rng_state += 0x9e3779b97f4a7c15ull);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return (double)((z ^ (z >> 31)) >> 11) * (1.0 / 9007199254740992.0);
}

int main(int argc, char **argv)
{
    if (argc != 21) return 2;
    const NodeArgs args(argv, true);
    const int queries = atoi(argv[13]);
    const float voxel = (float)atof(argv[14]);
    const int nx = atoi(argv[15]), ny = atoi(argv[16]), nz = atoi(argv[17]);
    const int n_points = 512, n_traj = 16, per_traj = 8;
    const float step = voxel / 2, radius = 4 * voxel;
    DriverNode node(args);
    if (const int e = setup_code(node.last_error())) return e;
    if (voxel > 0.f && node.enable_distance_field(voxel, nx, ny, nz, !queries) != DSM_OK) return 4;
    if (queries && node.enable_field_queries(n_points, n_traj, n_traj * per_traj) != DSM_OK) return 4;
    if (!open_io(argv[18], argv[19])) return 5;
    std::vector<dsm_field_sample_t> samples;
    std::vector<dsm_clearance_t> clearance;
    std::vector<double> points((size_t)3 * n_points), waypoints((size_t)3 * n_traj * per_traj);
    std::vector<int32_t> offsets((size_t)n_traj + 1);
    for (int j = 0; j <= n_traj; j++) offsets[(size_t)j] = j * per_traj;
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
            if (queries)
            {
                if (dist) return 7; // a resident field hands out no grid
                const int n[3] = {nx, ny, nz};
                auto coord = [&](int k) { return ((double)origin[k] - 1.0 + uniform() * (n[k] + 2)) * (double)voxel; };
                for (int i = 0; i < n_points; i++)
                    for (int k = 0; k < 3; k++) points[(size_t)3 * i + k] = coord(k);
                for (int i = 0; i < n_traj * per_traj; i++)
                    for (int k = 0; k < 3; k++) waypoints[(size_t)3 * i + k] = coord(k);
                int rq = node.field_samples(points.data(), n_points, samples);
                put(rq);
                put_list(points);
                put_list(samples);
                rq = node.trajectory_clearance(waypoints.data(), offsets.data(), n_traj, step, radius, clearance);
                put(rq);
                put(step), put(radius);
                put_list(waypoints);
                put_list(offsets);
                put_list(clearance);
            }
        }
        put_clouds(node);
        return 0;
    });
    if (e) return e;
    if (!put_final(node) || !save_files(node, argv[20])) return 6;
    return close_io();
}
