// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with or without enable_publishing(), and dumps what the node publishes.
// Usage: publish_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive publish in.bin out.bin
//   out.bin: with publish = 1, after every depth message: int32 rc of published_clouds, int32 inactive_changed_from,
//            the published active and inactive clouds, then int32 rc and the clouds of active_points() and
//            inactive_points() read right after (each cloud as int32 n + n points);
//            at the end, for either value of publish: local_surfels (int32 n + records) and inactive_points.
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "driver_io.hpp"

int main(int argc, char **argv)
{
    if (argc != 16) return 2;
    const NodeArgs args(argv, true);
    const int publish = atoi(argv[13]);
    DriverNode node(args);
    if (const int e = setup_code(node.last_error())) return e;
    if (publish && node.enable_publishing() != DSM_OK) return 4;
    if (!open_io(argv[14], argv[15])) return 5;
    const int e = feed_script(node, args.W, args.H, [&]() -> int {
        if (!publish) return 0;
        const dsm_point_t *a = nullptr, *b = nullptr;
        int na = 0, nb = 0, from = 0;
        const int rc = node.published_clouds(a, na, b, nb, from);
        put(rc);
        put(from);
        put_n(a, rc == DSM_OK ? na : 0);
        put_n(b, rc == DSM_OK ? nb : 0);
        put_clouds(node);
        return 0;
    });
    if (e) return e;
    if (!put_final(node)) return 6;
    return close_io();
}
