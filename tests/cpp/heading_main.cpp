// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with known space, with or without enable_headings(), and dumps the headings planned after every fused frame with the
// grid and requests they were planned on, and the node's clouds.  After depth message `reload_at` the node saves its
// state and loads it back.
// Usage: heading_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive voxel nx ny nz max_views
//                     max_range headings reload_at in.bin out.bin out_prefix
//   headings = 0: no heading jobs (the known field is requested and not dumped).
//   out.bin: with headings, int32 rc of enable_headings() before enable_known_space, int32 rc of it after and int32 rc
//            of headings() before the first frame; after every depth message: with headings, int32 rc (of headings(),
//            or of the reader before it that failed), int32 unknown_blocks (the message count % 2), float max_range
//            (voxel * (10 + 5 (count % 3))), int32 samples per segment (1 + count % 3), int32 origin[3], the state grid
//            (int32 n + n bytes) of the field distance_field() handed out, the control points (int32 n + n doubles: two
//            trajectories through the field's middle voxel), the offsets (int32 n + n int32), the rotations (int32 n + n
//            doubles: eight yaws about the world z axis), the requests (int32 n + n dsm_heading_request_t),
//            dsm_heading_info_t, the records, samples and counts (each int32 n + n records), and int32 the rc of
//            headings() right after load_state at message reload_at (1 at every other message); then, always, int32 rc
//            and the clouds of active_points() and inactive_points() (each int32 n + n points); at the end:
//            local_surfels (int32 n + records), and the node's save_mesh and save_cloud go to <out_prefix>.ply /
//            <out_prefix>.pcd.
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "driver_io.hpp"

#include <cmath>

int main(int argc, char **argv)
{
    if (argc != 24) return 2;
    const NodeArgs args(argv, true);
    const FieldArgs field(argv);
    const bool heading = atoi(argv[19]) > 0;
    const int reload_at = atoi(argv[20]);
    DriverNode node(args);
    if (const int e = setup_code(node.last_error())) return e;
    if (!open_io(argv[21], argv[22])) return 5;
    if (node.enable_distance_field(field.voxel, field.nx, field.ny, field.nz) != DSM_OK) return 4;
    const int before_known = heading ? node.enable_headings(4, 4096) : DSM_OK;
    if (node.enable_known_space(field.max_views, field.max_range) != DSM_OK) return 4;
    if (heading && node.enable_headings(4, 4096) != DSM_OK) return 4;
    const std::string prefix = argv[23];
    const int n_yaws = 8, n_traj = 2, n_points = 8;
    std::vector<double> rotations(9 * n_yaws), points(3 * n_traj * n_points);
    for (int k = 0; k < n_yaws; k++)
    {
        const double a = 0.25 * M_PI * k, f[3] = {std::cos(a), std::sin(a), 0.0}, r[3] = {std::sin(a), -std::cos(a), 0.0},
                     d[3] = {0.0, 0.0, -1.0};
        for (int i = 0; i < 3; i++) rotations[9 * k + 3 * i] = r[i], rotations[9 * k + 3 * i + 1] = d[i], rotations[9 * k + 3 * i + 2] = f[i];
    }
    const std::vector<int32_t> offsets = {0, n_points, 2 * n_points};
    std::vector<dsm_heading_request_t> requests(n_traj);
    requests[0].start = 0, requests[0].end = -1, requests[0].max_step = 1, requests[0].reserved = 0;
    requests[1].start = 2, requests[1].end = 5, requests[1].max_step = 2, requests[1].reserved = 0;
    dsm_heading_info_t info;
    std::vector<dsm_heading_t> records;
    std::vector<dsm_heading_sample_t> samples;
    std::vector<dsm_heading_count_t> counts;
    if (heading)
    {
        put(before_known);
        put(DSM_OK);
        put(node.headings(points.data(), offsets.data(), n_traj, rotations.data(), n_yaws, 2, requests.data(), field.max_range, 1, 1, 1, info,
                          records, samples, counts)); // no field yet
    }
    int depth_msgs = 0;
    const int e = feed_script(node, args.W, args.H, [&]() -> int {
        const int ub = depth_msgs % 2, K = 1 + depth_msgs % 3;
        const float max_range = field.voxel * (float)(10 + 5 * (depth_msgs % 3));
        info = dsm_heading_info_t();
        int rh = DSM_OK;
        const FieldHandout h(node, true);
        double centre[3];
        field.middle(h.origin, centre);
        // two lines through the middle voxel: along x at its height, and diagonally in x and y, one voxel above
        for (int j = 0; j < n_traj; j++)
            for (int i = 0; i < n_points; i++)
            {
                const double t = ((double)i - 0.5 * (n_points - 1)) * 2.0 * (double)field.voxel;
                double *p = &points[3 * (j * n_points + i)];
                p[0] = centre[0] + t, p[1] = centre[1] + (j ? t : 0.0), p[2] = centre[2] + (j ? (double)field.voxel : 0.0);
            }
        if (heading && h.ok())
            rh = node.headings(points.data(), offsets.data(), n_traj, rotations.data(), n_yaws, K, requests.data(), max_range, ub, 2, 3, info,
                               records, samples, counts);
        if (heading)
        {
            put(first_error({h.rc, h.rs, rh}));
            put(ub);
            put(max_range);
            put(K);
            h.put_origin();
            h.put_state(field);
            put_list(points);
            put_list(offsets);
            put_list(rotations);
            put_list(requests);
            put(info);
            put_list(records);
            put_list(samples);
            put_list(counts);
        }
        int after_load = 1;
        if (++depth_msgs == reload_at)
        {
            if (!reload(node, prefix)) return 6;
            if (heading)
                after_load = node.headings(points.data(), offsets.data(), n_traj, rotations.data(), n_yaws, K, requests.data(), max_range, ub, 2,
                                           3, info, records, samples, counts);
        }
        if (heading) put(after_load);
        put_clouds(node);
        return 0;
    });
    return e ? e : end_drive(node, prefix);
}
