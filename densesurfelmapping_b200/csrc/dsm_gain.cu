// View gain (dsm_gain_*, DESIGN.md §8.12): per candidate camera pose, the frustum voxels of the latest known field and
// the free, unknown, occupied, frontier and cluster voxels it would see through the known grid.
//
//   k_gain_slots   one thread per entry of the frontier list (with clusters only): slot[list[j]] = the table entry that
//                  lists j, over a slot grid the launcher set to -1.
//   k_gain_init    one thread per view: the record's zero counts, its status and n_cluster (0, or -1 without a countable
//                  cluster); thread 0 writes the header and copies the field's error words.
//   k_gain_views   one 8x8x4 brick of a view's box per CTA of 256 threads, one voxel per thread, bricks laid out
//                  view-major in a one-dimensional grid (gridDim.y would cap the views); thread 0 finds the CTA's view by a
//                  binary search over the views' first bricks.  Each thread runs the fp64 frustum test, and only then the
//                  walk of include/dsm.h from the camera to the voxel's centre, leaving at the first blocking voxel.  The
//                  counts go through __reduce_add_sync, shared memory and one atomicAdd per counter per CTA.
// The frustum test and the walk are dsm_gain_frustum and dsm_gain_walk (dsm_device.cuh), shared with k_vp_score.  The
// walk is not shared with k_field_carve: carving visits every voxel and stores into the grid, the gain walk reads and
// stops at the first blocking voxel, so a shared helper would branch on its caller.  The kernels carry no error gate and
// are launched without PDL, as the other field kernels.
#include "dsm_device.cuh"
#include <algorithm>

#define GAIN_BLOCK (DSM_GAIN_BX * DSM_GAIN_BY * DSM_GAIN_BZ) // 256

static_assert(sizeof(dsm_view_gain_t) == 32 && sizeof(dsm_gain_info_t) == 32 && sizeof(dsm_gain_camera_t) == 48, "dsm_gain layouts");
static_assert(sizeof(DsmGainView) == 128 && DSM_GAIN_WORDS * 4 == sizeof(dsm_gain_info_t), "the header is the info's size");
static_assert(DSM_FRONTIER_N_LISTED == 3 && DSM_FRONTIER_N_CLUSTERS == 2, "frontier header words");

enum
{
    GAIN_FRUSTUM,
    GAIN_FREE,
    GAIN_UNKNOWN,
    GAIN_OCCUPIED,
    GAIN_FRONTIER,
    GAIN_CLUSTER,
    GAIN_COUNTS
};

__global__ void __launch_bounds__(GAIN_BLOCK) k_gain_slots(const dsm_frontier_cluster_t *__restrict__ table, const int32_t *__restrict__ list,
                                                           const int32_t *__restrict__ frontier_hdr, int frontier_max_clusters,
                                                           int32_t *__restrict__ slot)
{
    const int n_listed = frontier_hdr[DSM_FRONTIER_N_LISTED];
    const int n_table = min(frontier_hdr[DSM_FRONTIER_N_CLUSTERS], frontier_max_clusters);
    for (int j = blockIdx.x * GAIN_BLOCK + threadIdx.x; j < n_listed; j += gridDim.x * GAIN_BLOCK)
        slot[list[j]] = dsm_frontier_cluster_of(table, n_table, j);
}

__global__ void __launch_bounds__(GAIN_BLOCK) k_gain_init(const DsmFieldGrid g, const DsmGainView *__restrict__ views, int n_views,
                                                          const int32_t *__restrict__ fhdr, const int32_t *__restrict__ frontier_hdr,
                                                          const dsm_frontier_cluster_t *__restrict__ table, int frontier_max_clusters,
                                                          int unknown_blocks, int32_t *__restrict__ hdr, dsm_view_gain_t *__restrict__ out)
{
    const int j = blockIdx.x * GAIN_BLOCK + threadIdx.x;
    const int n_table = frontier_hdr ? min(frontier_hdr[DSM_FRONTIER_N_CLUSTERS], frontier_max_clusters) : 0;
    if (j == 0)
    {
        for (int k = 0; k < 3; k++) hdr[DSM_GAIN_ORIGIN + k] = g.o[k];
        hdr[DSM_GAIN_N_VIEWS] = n_views;
        hdr[DSM_GAIN_N_CLUSTERS_TABLE] = n_table;
        hdr[DSM_GAIN_UNKNOWN_BLOCKS] = unknown_blocks;
        hdr[DSM_GAIN_ERR_TAG] = fhdr[DSM_FIELD_ERR_TAG];
        hdr[DSM_GAIN_ERR_FRAME] = fhdr[DSM_FIELD_ERR_FRAME];
    }
    if (j >= n_views) return;
    const DsmGainView &V = views[j];
    const double v = (double)g.voxel;
    bool inside = true;
    for (int k = 0; k < 3; k++)
    {
        const double q = floor(__ddiv_rn(V.P[4 * k + 3], v)) - (double)g.o[k];
        inside = inside && q >= 0.0 && q < (double)g.n[k];
    }
    const int c = V.cluster;
    const bool past = c >= n_table, unlisted = c >= 0 && !past && table[c].offset < 0;
    dsm_view_gain_t r;
    r.n_frustum = r.n_free = r.n_unknown = r.n_occupied = r.n_frontier = 0;
    r.n_cluster = c < 0 || past || unlisted ? -1 : 0;
    r.status = !inside ? 1 : c < 0 ? 0 : past ? 3 : unlisted ? 2 : 0;
    r.reserved = 0;
    out[j] = r;
}

__global__ void __launch_bounds__(GAIN_BLOCK) k_gain_views(const DsmFieldGrid g, const uint8_t *__restrict__ state,
                                                           const DsmGainView *__restrict__ views, int n_views, double fx, double fy,
                                                           double cx, double cy, double width, double height, double range2,
                                                           int unknown_blocks, const int32_t *__restrict__ slot,
                                                           dsm_view_gain_t *__restrict__ out)
{
    __shared__ DsmGainView sv;
    __shared__ int s_view;
    __shared__ unsigned s_cnt[GAIN_COUNTS];
    const int tid = threadIdx.x;
    if (tid == 0)
    {
        int lo = 0, hi = n_views; // the last view whose first brick is <= this one
        while (hi - lo > 1)
        {
            const int m = (lo + hi) / 2;
            if (views[m].brick0 <= (int)blockIdx.x)
                lo = m;
            else
                hi = m;
        }
        s_view = lo;
    }
    if (tid < GAIN_COUNTS) s_cnt[tid] = 0;
    __syncthreads();
    const int j = s_view;
    if (tid < (int)(sizeof(DsmGainView) / 4))
        reinterpret_cast<int32_t *>(&sv)[tid] = reinterpret_cast<const int32_t *>(views + j)[tid];
    __syncthreads();
    const int nbx = (sv.size[0] + DSM_GAIN_BX - 1) / DSM_GAIN_BX, nby = (sv.size[1] + DSM_GAIN_BY - 1) / DSM_GAIN_BY;
    const int b = (int)blockIdx.x - sv.brick0;
    const int dx = b % nbx * DSM_GAIN_BX + tid % DSM_GAIN_BX, dy = b / nbx % nby * DSM_GAIN_BY + tid / DSM_GAIN_BX % DSM_GAIN_BY,
              dz = b / (nbx * nby) * DSM_GAIN_BZ + tid / (DSM_GAIN_BX * DSM_GAIN_BY);
    const int x = sv.lo[0] + dx, y = sv.lo[1] + dy, z = sv.lo[2] + dz;
    const int nx = g.n[0], ny = g.n[1], nz = g.n[2];
    const double v = (double)g.voxel;
    const double tx = sv.P[3], ty = sv.P[7], tz = sv.P[11];
    bool frustum = false, seen = false;
    if (dx < sv.size[0] && dy < sv.size[1] && dz < sv.size[2])
    {
        const double c0 = __dmul_rn(__dadd_rn((double)(g.o[0] + x), 0.5), v), c1 = __dmul_rn(__dadd_rn((double)(g.o[1] + y), 0.5), v),
                     c2 = __dmul_rn(__dadd_rn((double)(g.o[2] + z), 0.5), v);
        const double d0 = __dsub_rn(c0, tx), d1 = __dsub_rn(c1, ty), d2 = __dsub_rn(c2, tz);
        frustum = dsm_gain_frustum<4>(sv.P, d0, d1, d2, fx, fy, cx, cy, width, height, range2);
        if (frustum) seen = dsm_gain_walk(g, state, unknown_blocks, tx, ty, tz, c0, c1, c2);
    }
    unsigned st = 0, front = 0, member = 0;
    if (seen)
    {
        const size_t i = ((size_t)z * ny + y) * nx + x;
        st = __ldg(state + i);
        if (st == DSM_STATE_FREE)
            front = (x > 0 && __ldg(state + i - 1) == DSM_STATE_UNKNOWN) || (x + 1 < nx && __ldg(state + i + 1) == DSM_STATE_UNKNOWN) ||
                    (y > 0 && __ldg(state + i - nx) == DSM_STATE_UNKNOWN) || (y + 1 < ny && __ldg(state + i + nx) == DSM_STATE_UNKNOWN) ||
                    (z > 0 && __ldg(state + i - (size_t)nx * ny) == DSM_STATE_UNKNOWN) ||
                    (z + 1 < nz && __ldg(state + i + (size_t)nx * ny) == DSM_STATE_UNKNOWN);
        member = sv.cluster >= 0 && slot && __ldg(slot + i) == sv.cluster;
    }
    const unsigned n_frustum = __reduce_add_sync(0xffffffffu, frustum), n_free = __reduce_add_sync(0xffffffffu, seen && st == DSM_STATE_FREE),
                   n_unknown = __reduce_add_sync(0xffffffffu, seen && st == DSM_STATE_UNKNOWN),
                   n_occupied = __reduce_add_sync(0xffffffffu, seen && st == DSM_STATE_OCCUPIED),
                   n_front = __reduce_add_sync(0xffffffffu, front), n_member = __reduce_add_sync(0xffffffffu, member);
    if ((tid & 31) == 0)
    {
        if (n_frustum) atomicAdd(&s_cnt[GAIN_FRUSTUM], n_frustum);
        if (n_free) atomicAdd(&s_cnt[GAIN_FREE], n_free);
        if (n_unknown) atomicAdd(&s_cnt[GAIN_UNKNOWN], n_unknown);
        if (n_occupied) atomicAdd(&s_cnt[GAIN_OCCUPIED], n_occupied);
        if (n_front) atomicAdd(&s_cnt[GAIN_FRONTIER], n_front);
        if (n_member) atomicAdd(&s_cnt[GAIN_CLUSTER], n_member);
    }
    __syncthreads();
    // the record's first six words are the counters in GAIN_* order
    if (tid < GAIN_COUNTS && s_cnt[tid]) atomicAdd(reinterpret_cast<int32_t *>(out + j) + tid, (int)s_cnt[tid]);
}

cudaError_t dsm_launch_gain(const DsmFieldGrid &g, const uint8_t *state, const int32_t *dist, const dsm_gain_camera_t &cam,
                            const DsmGainView *views, int n_views, long long bricks, const uint8_t *frontier_res,
                            int frontier_max_clusters, int32_t *slot, uint8_t *res, cudaStream_t st)
{
    const size_t voxels = (size_t)g.n[0] * g.n[1] * g.n[2];
    int32_t *hdr = reinterpret_cast<int32_t *>(res);
    auto *out = reinterpret_cast<dsm_view_gain_t *>(res + 4 * DSM_GAIN_WORDS);
    const int32_t *fieldhdr = dist + dsm_field_header(voxels);
    const int32_t *fhdr = reinterpret_cast<const int32_t *>(frontier_res);
    const auto *table = frontier_res ? reinterpret_cast<const dsm_frontier_cluster_t *>(frontier_res + 4 * DSM_FRONTIER_WORDS) : nullptr;
    if (frontier_res)
    {
        const int32_t *list = reinterpret_cast<const int32_t *>(frontier_res + 4 * DSM_FRONTIER_WORDS +
                                                                sizeof(dsm_frontier_cluster_t) * (size_t)frontier_max_clusters);
        const cudaError_t e = cudaMemsetAsync(slot, 0xff, 4 * voxels, st);
        if (e != cudaSuccess) return e;
        k_gain_slots<<<(unsigned)std::min<size_t>((voxels + GAIN_BLOCK - 1) / GAIN_BLOCK, 1024), GAIN_BLOCK, 0, st>>>(table, list, fhdr,
                                                                                                                   frontier_max_clusters, slot);
    }
    k_gain_init<<<(unsigned)std::max((n_views + GAIN_BLOCK - 1) / GAIN_BLOCK, 1), GAIN_BLOCK, 0, st>>>(
        g, views, n_views, fieldhdr, fhdr, table, frontier_max_clusters, cam.unknown_blocks, hdr, out);
    const double R = (double)cam.max_range;
    if (bricks > 0)
        k_gain_views<<<(unsigned)bricks, GAIN_BLOCK, 0, st>>>(g, state, views, n_views, cam.fx, cam.fy, cam.cx, cam.cy, (double)cam.width,
                                                              (double)cam.height, R * R, cam.unknown_blocks, frontier_res ? slot : nullptr, out);
    return cudaGetLastError();
}
