// View gain (dsm_gain_*, DESIGN.md §8.12): per candidate camera pose, the frustum voxels of the latest known field and
// the free, unknown, occupied, frontier and cluster voxels it would see through the known grid.
//
//   k_gain_slots   one thread per entry of the frontier list (with clusters only): slot[list[j]] = the table entry that
//                  lists j, over a slot grid the enqueue set to -1.
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
// are launched without PDL, as the other field kernels.  The job's C ABI calls (dsm_gain_enable, _enqueue and _wait)
// follow them.
//
// One staged request (H2D), DsmGainView views[n_views] (dsm_device.cuh), and one packed result (D2H):
//   int32 header[DSM_GAIN_WORDS] | dsm_view_gain_t gains[max_views]
// The header's first six words are those of dsm_gain_info_t; its padding carries the field's error words, cleared by
// dsm_gain_wait.
#include "dsm_ctx.hpp"

enum
{
    DSM_GAIN_ORIGIN = 0, // 3 words
    DSM_GAIN_N_VIEWS = 3,
    DSM_GAIN_N_CLUSTERS_TABLE,
    DSM_GAIN_UNKNOWN_BLOCKS,
    DSM_GAIN_ERR_TAG, // the field header's DSM_FIELD_ERR_TAG / _ERR_FRAME, copied by k_gain_init
    DSM_GAIN_ERR_FRAME,
    DSM_GAIN_WORDS = 8 // 32 B
};
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

static size_t gain_res_bytes(int n_views) { return 4 * (size_t)DSM_GAIN_WORDS + sizeof(dsm_view_gain_t) * (size_t)n_views; }

extern "C" int dsm_gain_enable(dsm_ctx *ctx, int max_views)
{
    if (!ctx) return DSM_E_INVALID;
    const DsmField *f = ctx->field.get();
    if (!f || !ctx->views || ctx->gain) return DSM_E_STATE;
    if (max_views < 1 || max_views > DSM_GAIN_MAX_VIEWS) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    auto ga = std::make_unique<DsmGain>();
    ga->max_views = max_views;
    const size_t res = gain_res_bytes(max_views);
    CudaOwner &o = ga->own;
    o.device(&ga->views_dev, (size_t)max_views);
    o.host(&ga->views_host, (size_t)max_views);
    o.device(&ga->slot, f->voxels);
    o.device(&ga->res, res);
    o.host(&ga->res_host, res);
    o.event(&ga->ev);
    return keep(ctx->gain, ga);
}

// Enqueue only: the views staged (pose, box, cluster and first brick) and copied, the kernels on the state grid of the
// latest (known) field request and, with clusters, on the latest frontier job's device result, one D2H copy of the used
// result and the event.  Later field and frontier requests overwrite those buffers only behind the job.
extern "C" int dsm_gain_enqueue(dsm_ctx *ctx, const dsm_gain_camera_t *camera, const double *poses, const int32_t *clusters, int n_views)
{
    if (!ctx) return DSM_E_INVALID;
    DsmGain *ga = ctx->gain.get();
    const DsmField *f = known_field(ctx);
    if (!ga || !f || ga->in_flight) return DSM_E_STATE;
    const DsmFrontier *fr = ctx->frontier.get();
    if (clusters && !read_latest(fr, f)) return DSM_E_STATE;
    if (!camera || n_views < 0 || n_views > ga->max_views || (n_views > 0 && !poses)) return DSM_E_INVALID;
    const dsm_gain_camera_t &c = *camera;
    const double v = (double)f->g.voxel, R = (double)c.max_range;
    if (!gain_camera_ok(c, v)) return DSM_E_INVALID;
    const long long m = 2 * (long long)std::ceil(R / v) + 3;
    if ((long long)n_views * m * m * m > DSM_GAIN_MAX_WORK) return DSM_E_INVALID;
    for (size_t i = 0; i < 12 * (size_t)n_views; i++)
        if (!std::isfinite(poses[i])) return DSM_E_INVALID;
    if (clusters)
        for (int j = 0; j < n_views; j++)
            if (clusters[j] < -1) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    // the previous job's copy out of this staging ended before its wait, which no job in flight implies
    long long bricks = 0;
    for (int j = 0; j < n_views; j++)
    {
        DsmGainView &V = ga->views_host[j];
        std::memcpy(V.P, poses + 12 * (size_t)j, sizeof(V.P));
        gain_box(V.P, c, f->g, V);
        V.cluster = clusters ? clusters[j] : -1;
        V.brick0 = (int)bricks; // below 2^31: the work bound caps the bricks far lower
        bricks += dsm_gain_bricks(V.size);
    }
    const cudaStream_t st = ctx->stream;
    if (n_views > 0) CK(cudaMemcpyAsync(ga->views_dev, ga->views_host, sizeof(DsmGainView) * (size_t)n_views, cudaMemcpyHostToDevice, st));
    const DsmFieldGrid &g = f->g;
    int32_t *hdr = reinterpret_cast<int32_t *>(ga->res);
    auto *out = reinterpret_cast<dsm_view_gain_t *>(ga->res + 4 * DSM_GAIN_WORDS);
    // the frontier job's result, with clusters
    const int32_t *fhdr = clusters ? reinterpret_cast<const int32_t *>(fr->res) : nullptr;
    const auto *table = clusters ? reinterpret_cast<const dsm_frontier_cluster_t *>(fr->res + DsmFrontier::table_at()) : nullptr;
    const int frontier_max_clusters = clusters ? fr->max_clusters : 0;
    if (clusters)
    {
        CK(cudaMemsetAsync(ga->slot, 0xff, 4 * f->voxels, st));
        k_gain_slots<<<(unsigned)std::min<size_t>((f->voxels + GAIN_BLOCK - 1) / GAIN_BLOCK, 1024), GAIN_BLOCK, 0, st>>>(
            table, reinterpret_cast<const int32_t *>(fr->res + fr->list_at()), fhdr, frontier_max_clusters, ga->slot);
    }
    k_gain_init<<<(unsigned)std::max((n_views + GAIN_BLOCK - 1) / GAIN_BLOCK, 1), GAIN_BLOCK, 0, st>>>(
        g, ga->views_dev, n_views, f->dist + dsm_field_header(f->voxels), fhdr, table, frontier_max_clusters, c.unknown_blocks, hdr, out);
    if (bricks > 0)
        k_gain_views<<<(unsigned)bricks, GAIN_BLOCK, 0, st>>>(g, f->occ, ga->views_dev, n_views, c.fx, c.fy, c.cx, c.cy, (double)c.width,
                                                              (double)c.height, R * R, c.unknown_blocks, clusters ? ga->slot : nullptr, out);
    CK(cudaGetLastError());
    return submit(ctx, *ga, ga->res, gain_res_bytes(n_views), f->requests);
}

extern "C" int dsm_gain_wait(dsm_ctx *ctx, dsm_gain_info_t *info, const dsm_view_gain_t **gains)
{
    if (!ctx) return DSM_E_INVALID;
    DsmGain *ga = ctx->gain.get();
    const int rc = wait_head(ctx, ga);
    if (rc != DSM_OK) return rc;
    copy_info(info, ga->words());
    if (gains) *gains = reinterpret_cast<const dsm_view_gain_t *>(ga->res_host + 4 * DSM_GAIN_WORDS);
    return capacity(ctx, ga->words(), DSM_GAIN_ERR_TAG, "dsm_gain_wait", "the field the job read");
}
