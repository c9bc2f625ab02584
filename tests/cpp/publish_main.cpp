// Drives include/dsm_surfel_node.hpp through the message script of node_main.cpp (orb / image / depth messages only)
// with or without enable_publishing(), and dumps what the node publishes.
// Usage: publish_main W H fx fy cx cy far near drift_free_poses device max_local max_inactive publish in.bin out.bin
//   out.bin: with publish = 1, after every depth message: int32 rc of published_clouds, int32 inactive_changed_from,
//            the published active and inactive clouds, then int32 rc and the clouds of active_points() and
//            inactive_points() read right after (each cloud as int32 n + n points);
//            at the end, for either value of publish: local_surfels (int32 n + records) and inactive_points.
// exit code 3 when no usable GPU (the library has no CPU fallback).
#include "dsm_surfel_node.hpp"
#include "driver_io.hpp"

int main(int argc, char **argv)
{
    if (argc != 16) return 2;
    const int W = atoi(argv[1]), H = atoi(argv[2]), publish = atoi(argv[13]);
    dsm::SurfelMapNode node(W, H, atof(argv[3]), atof(argv[4]), atof(argv[5]), atof(argv[6]), atof(argv[7]), atof(argv[8]), atoi(argv[9]),
                            atoi(argv[10]), atoi(argv[11]), atoi(argv[12]), nullptr);
    if (node.last_error() != DSM_OK) return node.last_error() == DSM_E_NODEVICE ? 3 : 4;
    if (publish && node.enable_publishing() != DSM_OK) return 4;
    in_f = fopen(argv[14], "rb");
    out_f = fopen(argv[15], "wb");
    if (!in_f || !out_f) return 5;
    NodeMessages msg;
    std::vector<dsm_point_t> act, inact;
    int type = 0, r = DSM_OK;
    while (get(type))
    {
        if (!msg.feed(node, type, W, H, r)) return 5;
        if (r != DSM_OK) return 6;
        if (type != 2 || !publish) continue;
        const dsm_point_t *a = nullptr, *b = nullptr;
        int na = 0, nb = 0, from = 0;
        const int rc = node.published_clouds(a, na, b, nb, from);
        put(rc);
        put(from);
        put_n(a, rc == DSM_OK ? na : 0);
        put_n(b, rc == DSM_OK ? nb : 0);
        int rr = node.active_points(act);
        if (rr == DSM_OK) rr = node.inactive_points(inact);
        put(rr);
        put_list(act);
        put_list(inact);
    }
    std::vector<dsm_surfel_t> local;
    if (node.local_surfels(local) != DSM_OK || node.inactive_points(inact) != DSM_OK) return 6;
    put_list(local);
    put_list(inact);
    fclose(in_f);
    fclose(out_f);
    return 0;
}
