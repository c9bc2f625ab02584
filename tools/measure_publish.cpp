// Timing harness of tools/measure_publish.py: drives dsm::SurfelMapNode (include/dsm_surfel_node.hpp) through the
// message script of tools/measure_node.py in one of four publishing modes and times the whole drive on the host clock,
// the device synchronised once at the end (and wherever the mode itself waits).
// Usage: measure_publish W H fx fy cx cy far near drift_free_poses frames.bin script.bin mode check
//   frames.bin / script.bin: as tools/measure_node.cpp (the script's per-frame publish flag is ignored)
//   mode  a: no publishing            b: active_points() + inactive_points() after every frame
//         c: published_clouds() right after every frame's fuse
//         d: published_clouds() of frame t-1 at the start of frame t's callbacks (the last one after the drive)
//   check 1: every frame's two clouds are folded into a 64-bit FNV-1a hash (sizes and bytes), printed as "hash"; modes
//            b, c and d must print the same value.  Hashing reads every byte on the host, so timings are taken with 0.
// Prints one JSON object.
#include "measure_drive.hpp"

static uint64_t g_hash = 1469598103934665603ull;
static void fold(const void *p, size_t n)
{
    const unsigned char *b = static_cast<const unsigned char *>(p);
    for (size_t i = 0; i < n; i++) g_hash = (g_hash ^ b[i]) * 1099511628211ull;
}
static void fold_clouds(const dsm_point_t *a, int na, const dsm_point_t *b, int nb)
{
    fold(&na, sizeof(na));
    fold(a, (size_t)na * sizeof(dsm_point_t));
    fold(&nb, sizeof(nb));
    fold(b, (size_t)nb * sizeof(dsm_point_t));
}

int main(int argc, char **argv)
{
    if (argc != 14) return 2;
    const int W = atoi(argv[1]);
    const char mode = argv[12][0];
    const bool check = atoi(argv[13]) != 0;
    if (mode < 'a' || mode > 'd') return 2;
    Drive d;
    if (!d.load(argv)) return 5;
    const int T = (int)d.msgs.size();
    DriveNode node(argv);
    if (const int e = node.setup_code()) return e;
    if ((mode == 'c' || mode == 'd') && node.enable_publishing() != DSM_OK) return 4;
    std::vector<dsm_point_t> active, inactive;
    const dsm_point_t *pa = nullptr, *pi = nullptr;
    int na = 0, ni = 0, from = 0, rc = DSM_OK;
    long long changed_points = 0;
    dsm_sync(node.context());
    const clk::time_point t0 = clk::now();
    for (int t = 0; t < T && rc == DSM_OK; t++)
    {
        const DriveMsg &m = d.msgs[(size_t)t];
        if (mode == 'd' && t > 0)
        {
            rc = node.published_clouds(pa, na, pi, ni, from);
            changed_points += ni - from;
            if (check && rc == DSM_OK) fold_clouds(pa, na, pi, ni);
        }
        if (rc == DSM_OK) rc = m.orb(node);
        if (rc == DSM_OK) rc = d.images(node, m, W);
        if (rc != DSM_OK) break;
        if (mode == 'b')
        {
            rc = node.active_points(active);
            if (rc == DSM_OK) rc = node.inactive_points(inactive);
            if (check && rc == DSM_OK) fold_clouds(active.data(), (int)active.size(), inactive.data(), (int)inactive.size());
        }
        else if (mode == 'c')
        {
            rc = node.published_clouds(pa, na, pi, ni, from);
            changed_points += ni - from;
            if (check && rc == DSM_OK) fold_clouds(pa, na, pi, ni);
        }
    }
    if (rc == DSM_OK && mode == 'd')
    {
        rc = node.published_clouds(pa, na, pi, ni, from);
        changed_points += ni - from;
        if (check && rc == DSM_OK) fold_clouds(pa, na, pi, ni);
    }
    if (rc != DSM_OK) return 6;
    dsm_sync(node.context());
    const double total = ms(t0, clk::now());
    int n_store = 0, n_pool = 0;
    if (dsm_inactive_size(node.context(), &n_store, nullptr) != DSM_OK || dsm_pool_size(node.context(), &n_pool) != DSM_OK) return 6;
    std::printf("{\"mode\": \"%c\", \"frames\": %d, \"total_ms\": %.3f, \"ms_per_frame\": %.4f, \"store_surfels\": %d, \"pool_surfels\": %d, "
                "\"inactive_points_from_changed_from\": %lld, \"hash\": \"%016llx\"}\n",
                mode, T, total, total / (T ? T : 1), n_store, n_pool, changed_points, check ? (unsigned long long)g_hash : 0ull);
    return 0;
}
