// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with a distance field and its signed grid after every frame, optimises trajectories on it with trajectories(), and
// dumps the signed grids, the jobs' inputs and results and the node's clouds.  After depth message `reload_at` the node
// saves its state and loads it back.
// Usage: trajectory_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive voxel nx ny nz
//                        reload_at in.bin out.bin out_prefix
//   out.bin: int32 rc of enable_trajectories before enable_signed_distance, int32 rc of it after, int32 rc of
//            trajectories() before the first frame, the params (dsm_trajectory_params_t);
//            after every depth message: int32 rc of distance_field, double camera[3] (the fuse pose's position), int32
//            origin[3], int32 rc of signed_distance_field and the signed grid (int32 n + n floats), int32 rc of
//            trajectories(), the points (int32 3n + 3n doubles),
//            offsets (int32 t + 1 + t + 1 ints), dt (int32 t + t doubles), the info (dsm_trajectory_info_t), the records
//            (int32 t + t records) and the optimised points (int32 3n + 3n doubles), then int32 rc and the clouds of
//            active_points() and inactive_points() read right after (each int32 n + n points); after message reload_at,
//            int32 rc of trajectories() right after load_state.
// The control points are drawn from a fixed generator over the grid's box (one voxel beyond it on every side).
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "driver_io.hpp"

static uint64_t rng_state = 0x2545f4914f6cdd1dull;
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
    const float voxel = (float)atof(argv[13]);
    const int nx = atoi(argv[14]), ny = atoi(argv[15]), nz = atoi(argv[16]);
    const int reload_at = atoi(argv[17]);
    const size_t voxels = (size_t)nx * ny * nz;
    const int lens[] = {7, 16, 33, 64, 100, 256};
    const int n_traj = 6;
    std::vector<int32_t> offsets(1, 0);
    for (int j = 0; j < n_traj; j++) offsets.push_back(offsets.back() + lens[j]);
    const int n_points = offsets.back();
    std::vector<double> dt;
    for (int j = 0; j < n_traj; j++) dt.push_back(0.25 + 0.125 * j);
    dsm_trajectory_params_t params = dsm_trajectory_params_t();
    params.w_smooth = 1, params.w_clear = 10, params.w_feas = 1, params.margin = 2 * voxel, params.v_max = 2, params.a_max = 4;
    params.g_tol = 1e-6, params.max_iter = 40, params.memory = 6, params.max_ls = 12, params.samples = 5, params.radius = voxel;
    DriverNode node(args);
    if (const int e = setup_code(node.last_error())) return e;
    if (node.enable_distance_field(voxel, nx, ny, nz) != DSM_OK) return 4;
    if (!open_io(argv[18], argv[19])) return 5;
    put(node.enable_trajectories(n_traj, n_points, 8)); // before enable_signed_distance: DSM_E_STATE
    if (node.enable_signed_distance() != DSM_OK) return 4;
    put(node.enable_trajectories(n_traj, n_points, 8));
    std::vector<double> points((size_t)3 * n_points), optimised;
    std::vector<dsm_trajectory_t> records;
    dsm_trajectory_info_t info;
    put(node.trajectories(points.data(), offsets.data(), dt.data(), n_traj, params, info, records, optimised)); // no field yet
    put(params);
    const std::string prefix = argv[20];
    int depth_msgs = 0;
    const int e = feed_script(node, args.W, args.H, [&]() -> int {
        const float *dist = nullptr, *sdist = nullptr;
        int32_t origin[3] = {0, 0, 0};
        int n_occ = 0;
        put(node.distance_field(dist, origin, n_occ));
        const dsm::Pose cam = node.pose_graph().camera;
        put(cam.x), put(cam.y), put(cam.z);
        put(origin[0]), put(origin[1]), put(origin[2]);
        put(node.signed_distance_field(sdist));
        put_list(std::vector<float>(sdist, sdist + (sdist ? voxels : 0)));
        const int n[3] = {nx, ny, nz};
        for (int i = 0; i < n_points; i++)
            for (int k = 0; k < 3; k++) points[(size_t)3 * i + k] = ((double)origin[k] - 1.0 + uniform() * (n[k] + 2)) * (double)voxel;
        put(node.trajectories(points.data(), offsets.data(), dt.data(), n_traj, params, info, records, optimised));
        put_list(points);
        put_list(offsets);
        put_list(dt);
        put(info);
        put_list(records);
        put_list(optimised);
        put_clouds(node);
        if (++depth_msgs == reload_at)
        {
            if (node.save_state(prefix + ".state") != DSM_OK || node.load_state(prefix + ".state") != DSM_OK) return 6;
            put(node.trajectories(points.data(), offsets.data(), dt.data(), n_traj, params, info, records, optimised));
        }
        return 0;
    });
    if (e) return e;
    return close_io();
}
