// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with known space, with or without enable_terrain(-2), and dumps the terrain found after every fused frame with the
// grid it was found on, and the node's clouds.  After depth message `reload_at` the node saves its state and loads it
// back.
// Usage: terrain_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive voxel nx ny nz max_views
//                     max_range terrain reload_at in.bin out.bin out_prefix
//   terrain = 0: no terrain jobs (the known field is requested and not dumped).
//   out.bin: with terrain, int32 rc of enable_terrain() before enable_known_space, int32 rc of it after and int32 rc of
//            terrain() before the first frame; after every depth message: with terrain, int32 rc (of terrain(), or of
//            the reader before it that failed), int32 headroom (1 + count % 4), int32 max_step (count % 3), int32
//            origin[3], the state grid (int32 n + n bytes) of the field distance_field() handed out,
//            dsm_terrain_info_t, the level, status, step and clearance planes (each int32 n + n values), and int32 the
//            rc of terrain() right after load_state at message reload_at (1 at every other message); then, always,
//            int32 rc and the clouds of active_points() and inactive_points() (each int32 n + n points); at the end:
//            local_surfels (int32 n + records), and the node's save_mesh and save_cloud go to <out_prefix>.ply /
//            <out_prefix>.pcd.
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "driver_io.hpp"

int main(int argc, char **argv)
{
    if (argc != 24) return 2;
    const NodeArgs args(argv, true);
    const FieldArgs field(argv);
    const bool terrain = atoi(argv[19]) > 0;
    const int reload_at = atoi(argv[20]);
    DriverNode node(args);
    if (const int e = setup_code(node.last_error())) return e;
    if (!open_io(argv[21], argv[22])) return 5;
    if (node.enable_distance_field(field.voxel, field.nx, field.ny, field.nz) != DSM_OK) return 4;
    const int up = -2; // the y-down camera frames of the drive
    const int before_known = terrain ? node.enable_terrain(up) : DSM_OK;
    if (node.enable_known_space(field.max_views, field.max_range) != DSM_OK) return 4;
    if (terrain && node.enable_terrain(up) != DSM_OK) return 4;
    const std::string prefix = argv[23];
    dsm_terrain_info_t info;
    std::vector<int16_t> level;
    std::vector<uint8_t> status, step;
    std::vector<float> clearance;
    if (terrain)
    {
        put(before_known);
        put(DSM_OK);
        put(node.terrain(1, 0, info, level, status, step, clearance)); // no field yet
    }
    int depth_msgs = 0;
    const int e = feed_script(node, args.W, args.H, [&]() -> int {
        const int headroom = 1 + depth_msgs % 4, max_step = depth_msgs % 3;
        info = dsm_terrain_info_t();
        int rt = DSM_OK;
        const FieldHandout h(node, true);
        if (terrain && h.ok()) rt = node.terrain(headroom, max_step, info, level, status, step, clearance);
        if (terrain)
        {
            put(first_error({h.rc, h.rs, rt}));
            put(headroom);
            put(max_step);
            h.put_origin();
            h.put_state(field);
            put(info);
            put_list(level);
            put_list(status);
            put_list(step);
            put_list(clearance);
        }
        int after_load = 1;
        if (++depth_msgs == reload_at)
        {
            if (!reload(node, prefix)) return 6;
            if (terrain) after_load = node.terrain(headroom, max_step, info, level, status, step, clearance);
        }
        if (terrain) put(after_load);
        put_clouds(node);
        return 0;
    });
    return e ? e : end_drive(node, prefix);
}
