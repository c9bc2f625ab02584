// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with known space, with or without enable_terrain(-2), enable_frontiers(), enable_reach() and enable_reach_matrix(), and
// dumps the driving-cost matrix of every fused frame with the grid and points it was found on, and the node's clouds.  A
// ground planner's chain: terrain(3, 1), frontiers(1), reach_terrain(with_frontiers) from the field's middle, then
// reach_matrix_terrain over that point and the reached viewpoint cells' centres.  After depth message `reload_at` the
// node saves its state and loads it back.
// Usage: reach_matrix_terrain_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive voxel nx ny nz
//                                  max_views max_range max_sites max_tiles max_rounds reload_at in.bin out.bin out_prefix
//   max_sites = max_tiles = max_rounds = 0: no terrain, frontiers, paths or matrices (the known field is requested and
//   not dumped).
//   out.bin: after every depth message: with matrices, int32 rc (of reach_matrix_terrain(), or of the call before it
//            that failed), int32 approach (the message count % 5), float radius (voxel * (count % 3) / 2), int32
//            origin[3], the state grid (int32 n + n bytes) of the field distance_field() handed out, the points (int32 n
//            + n doubles, xyz each), dsm_reach_matrix_info_t, the sites (int32 n + n dsm_reach_site_t) and the matrix
//            (int32 n + n uint32), int32 the rc of reach_matrix_terrain() before terrain() on that frame, and int32 the
//            rc of reach_matrix_terrain() right after load_state at message reload_at (1 at every other message); then,
//            always, int32 rc and the clouds of active_points() and inactive_points() (each int32 n + n points); at the
//            end: local_surfels (int32 n + records), and the node's save_mesh and save_cloud go to <out_prefix>.ply /
//            <out_prefix>.pcd.
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "driver_io.hpp"

int main(int argc, char **argv)
{
    if (argc != 26) return 2;
    const NodeArgs args(argv, true);
    const FieldArgs field(argv);
    const int max_sites = atoi(argv[19]), max_tiles = atoi(argv[20]), max_rounds = atoi(argv[21]), reload_at = atoi(argv[22]);
    const bool matrices = max_sites > 0 || max_tiles > 0 || max_rounds > 0;
    DriverNode node(args);
    if (const int e = setup_code(node.last_error())) return e;
    if (const int e = field.enable(node)) return e;
    if (matrices && (node.enable_terrain(-2) != DSM_OK || node.enable_frontiers(64, 1 << 16) != DSM_OK ||
                     node.enable_reach(max_sites - 1, 1 << 16, max_rounds) != DSM_OK ||
                     node.enable_reach_matrix(max_sites, max_tiles, max_rounds) != DSM_OK))
        return 4;
    if (!open_io(argv[23], argv[24])) return 5;
    const std::string prefix = argv[25];
    std::vector<dsm_frontier_cluster_t> clusters;
    std::vector<int32_t> voxels, path;
    std::vector<dsm_reach_target_t> targets;
    std::vector<dsm_reach_site_t> sites;
    std::vector<uint32_t> matrix;
    std::vector<double> points;
    std::vector<int16_t> level;
    std::vector<uint8_t> status, step;
    std::vector<float> clearance;
    const std::vector<double> no_goals;
    int depth_msgs = 0;
    const int e = feed_script(node, args.W, args.H, [&]() -> int {
        const int k = depth_msgs % 5;
        const float radius = field.voxel * (float)(depth_msgs % 3) / 2.f;
        dsm_frontier_counts_t counts = dsm_frontier_counts_t();
        dsm_terrain_info_t tinfo = dsm_terrain_info_t();
        dsm_reach_info_t rinfo = dsm_reach_info_t();
        dsm_reach_matrix_info_t info = dsm_reach_matrix_info_t();
        const FieldHandout h(node, true);
        double start[3];
        field.middle(h.origin, start);
        points.assign(start, start + 3);
        int before_terrain = 1, rt = DSM_OK, rf = DSM_OK, rr = DSM_OK, rm = DSM_OK;
        if (matrices && h.ok())
        {
            before_terrain = node.reach_matrix_terrain(points, radius, k, info, sites, matrix);
            rt = node.terrain(3, 1, tinfo, level, status, step, clearance);
            rf = node.frontiers(1, clusters, voxels, counts);
            if (rt == DSM_OK && rf == DSM_OK) rr = node.reach_terrain(start, radius, k, no_goals, true, rinfo, targets, path);
            if (rt == DSM_OK && rf == DSM_OK && rr == DSM_OK)
            {
                // a viewpoint cell q P + p of the plane (x, z) of up -2: its centre, at the start's height
                const int P = tinfo.m[0];
                for (const dsm_reach_target_t &t : targets)
                    if (t.status == 0)
                    {
                        points.push_back(((double)(tinfo.origin[0] + t.viewpoint % P) + 0.5) * (double)field.voxel);
                        points.push_back(start[1]);
                        points.push_back(((double)(tinfo.origin[2] + t.viewpoint / P) + 0.5) * (double)field.voxel);
                    }
                rm = node.reach_matrix_terrain(points, radius, k, info, sites, matrix);
            }
        }
        if (matrices)
        {
            put(first_error({h.rc, h.rs, rt, rf, rr, rm}));
            put(k);
            put(radius);
            h.put_origin();
            h.put_state(field);
            put_list(points);
            put(info);
            put_list(sites);
            put_list(matrix);
            put(before_terrain);
        }
        int after_load = 1;
        if (++depth_msgs == reload_at)
        {
            if (!reload(node, prefix)) return 6;
            if (matrices) after_load = node.reach_matrix_terrain(points, radius, k, info, sites, matrix);
        }
        if (matrices) put(after_load);
        put_clouds(node);
        return 0;
    });
    return e ? e : end_drive(node, prefix);
}
