// Viewpoints of frontier clusters (dsm_viewpoint_*, DESIGN.md §8.15): clear candidate positions around each cluster of
// the latest frontier job, each scored at its best heading by the sampled cluster voxels it would see.
//
//   k_vp_clusters    one thread per requested cluster: its status, centre voxel and samples (DsmVpCluster) and its
//                    record with zero counts; thread 0 writes the header and copies the field's error words.
//   k_vp_candidates  one thread per (cluster, offset), one cluster per gridDim.y row: the key set to ~0, the inside,
//                    traversable and reached tests, the counts by __syncthreads_count and one atomicAdd per CTA, and the
//                    reached candidates appended to a list by warp-aggregated atomics (the list's order does not matter:
//                    each candidate writes its own key).
//   k_vp_score       persistent CTAs walking the list, one candidate per CTA at a time and one sample per thread: the
//                    mask of rotations whose frustum holds the sample (dsm_gain_frustum), then, for a non-empty mask,
//                    the line of sight (dsm_gain_walk); ballots and popcounts add the seen samples to per-rotation
//                    counts in shared memory, and thread 0 takes the arg-max and writes the candidate's key.
//   k_vp_select      one CTA per cluster: top_k rounds of a block minimum over the cluster's keys above the last one.
// A key packs the ranking (-n_seen, cost, offset index) and the rotation into 63 bits, so the least keys are the
// viewpoints in order and ~0 is no viewpoint.  The kernels carry no error gate and are launched without PDL, as the
// other field kernels.  The job's C ABI calls (dsm_viewpoint_enable, _enqueue and _wait) follow them.
// The terrain job (dsm_viewpoint_enqueue_terrain, DESIGN.md §8.23) runs the same kernels on a VpTerrainGrid: centres,
// candidates, keys and slots on the plane (P, Q, 1) of the latest terrain job, traversable on its status and clearance
// planes, and the camera over a candidate cell at the field voxel eye voxels above its support, from which the walk
// runs through the field's state grid as on the field.
//
// One staged request (H2D, vp_stage_bytes):
//   double rotations[64][9] | int32 offsets[4096][3] | int32 clusters[n_clusters]
// and one packed result (D2H, 64 + 32 n (1 + top_k) B):
//   int32 header[DSM_VP_WORDS] | dsm_viewpoint_cluster_t records[n] | dsm_viewpoint_t slots[n][top_k]
// The header's first ten words are those of dsm_viewpoint_info_t; its last two carry the field's error words, cleared
// by dsm_viewpoint_wait.
#include "dsm_ctx.hpp"

enum
{
    DSM_VP_ORIGIN = 0, // 3 words
    DSM_VP_N_CLUSTERS = 3,
    DSM_VP_N_OFFSETS,
    DSM_VP_N_ROTATIONS,
    DSM_VP_TOP_K,
    DSM_VP_UNKNOWN_BLOCKS,
    DSM_VP_WITH_REACH,
    DSM_VP_N_CLUSTERS_TABLE,
    DSM_VP_ERR_TAG = 14, // the field header's DSM_FIELD_ERR_TAG / _ERR_FRAME, copied by k_vp_clusters
    DSM_VP_ERR_FRAME,
    DSM_VP_WORDS = 16 // 64 B
};
// what k_vp_clusters leaves per requested cluster for the later kernels
struct DsmVpCluster
{
    int32_t g[3];   // the centre voxel
    int32_t status; // of the record
    int32_t base, n, n_s, pad; // the members' list offset and count, the samples
};

#define VP_BLOCK 256
#define VP_NONE 0xffffffffffffffffull

static_assert(sizeof(dsm_viewpoint_params_t) == 40 && sizeof(dsm_viewpoint_cluster_t) == 32 && sizeof(dsm_viewpoint_t) == 32 &&
                  sizeof(dsm_viewpoint_info_t) == 64, "dsm_viewpoint layouts");
static_assert(DSM_VP_WORDS * 4 == sizeof(dsm_viewpoint_info_t) && DSM_VP_N_CLUSTERS_TABLE == 9, "the header starts with the info");
static_assert(DSM_FRONTIER_N_CLUSTERS == 2, "frontier header words");
static_assert(DSM_VIEWPOINT_MAX_SAMPLES < 8192 && DSM_VIEWPOINT_MAX_OFFSETS <= 4096 && DSM_VIEWPOINT_MAX_ROTATIONS <= 64,
              "the key's fields: 13 bits of 8191 - n_seen, 32 of cost, 12 of offset, 6 of rotation");

__device__ __forceinline__ unsigned long long vp_key(int n_seen, uint32_t cost, int offset, int rotation)
{
    return (unsigned long long)(8191 - n_seen) << 50 | (unsigned long long)cost << 18 | (unsigned long long)offset << 6 |
           (unsigned long long)rotation;
}

// The terrain job's grid (DESIGN.md §8.23): the plane of the terrain job (ReachTerrainGrid), its level plane, and du the
// camera's height above the support in voxels along the field's up axis (eye, negated for a negative up)
struct VpTerrainGrid : ReachTerrainGrid
{
    const int16_t *level;
    int du;
};

// What the kernels ask of their grid: the centre voxel of a cluster (reach's start snap of its fp64 centroid, on the
// plane's two axes), the field grid the walk and the member voxels live on, and the field voxel of the camera over a
// candidate (x, y, z).  On the field grid the candidate is that voxel.
__device__ __forceinline__ void vp_centre(const DsmFieldGrid &g, const dsm_frontier_cluster_t &T, int32_t *out)
{
    const double v = (double)g.voxel;
    for (int k = 0; k < 3; k++) out[k] = (int)(floor(__ddiv_rn(T.centroid[k], v)) - (double)g.o[k]);
}
__device__ __forceinline__ void vp_centre(const VpTerrainGrid &g, const dsm_frontier_cluster_t &T, int32_t *out)
{
    const double v = (double)g.voxel;
    const int o0 = g.h0 == 0 ? g.o[0] : g.o[1], o1 = g.h1 == 1 ? g.o[1] : g.o[2]; // selects: no local copy of g
    out[0] = (int)(floor(__ddiv_rn(T.centroid[g.h0], v)) - (double)o0);
    out[1] = (int)(floor(__ddiv_rn(T.centroid[g.h1], v)) - (double)o1);
    out[2] = 0;
}
__device__ __forceinline__ const DsmFieldGrid &vp_field(const DsmFieldGrid &g) { return g; }
__device__ __forceinline__ DsmFieldGrid vp_field(const VpTerrainGrid &g)
{
    DsmFieldGrid f = g;
    for (int k = 0; k < 3; k++) f.n[k] = g.nf[k];
    return f;
}
__device__ __forceinline__ int3 vp_camera(const DsmFieldGrid &, int x, int y, int z) { return make_int3(x, y, z); }
__device__ __forceinline__ int3 vp_camera(const VpTerrainGrid &g, int x, int y, int)
{ // x along h0 and y along h1; the up axis is the third (h0 is 0 or 1, h1 is 1 or 2)
    const int u = (int)g.level[y * g.n[0] + x] + g.du;
    return make_int3(g.h0 == 0 ? x : u, g.h0 == 1 ? x : g.h1 == 1 ? y : u, g.h1 == 2 ? y : u);
}

template <typename Grid>
__global__ void __launch_bounds__(VP_BLOCK) k_vp_clusters(const Grid g, const int32_t *__restrict__ fhdr,
                                                          const int32_t *__restrict__ frontier_hdr,
                                                          const dsm_frontier_cluster_t *__restrict__ table, int frontier_max_clusters,
                                                          const int32_t *__restrict__ clusters, int n_clusters, int n_offsets,
                                                          int n_rotations, int top_k, int unknown_blocks, int with_reach, int max_samples,
                                                          int32_t *__restrict__ hdr, dsm_viewpoint_cluster_t *__restrict__ rec,
                                                          DsmVpCluster *__restrict__ cl, int32_t *__restrict__ count)
{
    const int i = blockIdx.x * VP_BLOCK + threadIdx.x;
    const int n_table = min(frontier_hdr[DSM_FRONTIER_N_CLUSTERS], frontier_max_clusters);
    if (i == 0)
    {
        for (int k = 0; k < 3; k++) hdr[DSM_VP_ORIGIN + k] = g.o[k];
        hdr[DSM_VP_N_CLUSTERS] = n_clusters;
        hdr[DSM_VP_N_OFFSETS] = n_offsets;
        hdr[DSM_VP_N_ROTATIONS] = n_rotations;
        hdr[DSM_VP_TOP_K] = top_k;
        hdr[DSM_VP_UNKNOWN_BLOCKS] = unknown_blocks;
        hdr[DSM_VP_WITH_REACH] = with_reach;
        hdr[DSM_VP_N_CLUSTERS_TABLE] = n_table;
        for (int k = DSM_VP_N_CLUSTERS_TABLE + 1; k < DSM_VP_ERR_TAG; k++) hdr[k] = 0;
        hdr[DSM_VP_ERR_TAG] = fhdr[DSM_FIELD_ERR_TAG];
        hdr[DSM_VP_ERR_FRAME] = fhdr[DSM_FIELD_ERR_FRAME];
        *count = 0;
    }
    if (i >= n_clusters) return;
    const int c = clusters[i];
    const bool past = c >= n_table, unlisted = !past && table[c].offset < 0;
    DsmVpCluster q;
    q.status = past ? 3 : unlisted ? 2 : 0;
    q.base = q.n = q.n_s = q.pad = 0;
    for (int k = 0; k < 3; k++) q.g[k] = 0;
    if (q.status == 0)
    {
        const dsm_frontier_cluster_t &T = table[c];
        vp_centre(g, T, q.g);
        q.base = T.offset;
        q.n = T.n_voxels;
        q.n_s = min(T.n_voxels, max_samples);
    }
    cl[i] = q;
    dsm_viewpoint_cluster_t r;
    r.cluster = c;
    r.status = q.status;
    r.n_samples = q.n_s;
    r.n_inside = r.n_traversable = r.n_reached = r.n_viewpoints = r.reserved = 0;
    rec[i] = r;
}

template <typename Grid>
__global__ void __launch_bounds__(VP_BLOCK) k_vp_candidates(const Grid g, const uint8_t *__restrict__ state,
                                                            const int32_t *__restrict__ dist, const int32_t *__restrict__ offsets,
                                                            int n_offsets, float radius, const uint32_t *__restrict__ reach_cost,
                                                            const DsmVpCluster *__restrict__ cl, dsm_viewpoint_cluster_t *__restrict__ rec,
                                                            unsigned long long *__restrict__ key, int32_t *__restrict__ list,
                                                            int32_t *__restrict__ count)
{
    const int i = blockIdx.y, j = blockIdx.x * VP_BLOCK + threadIdx.x;
    const DsmVpCluster q = cl[i];
    const int item = i * n_offsets + j;
    bool inside = false, trav = false, reached = false;
    if (j < n_offsets)
    {
        key[item] = VP_NONE;
        if (q.status == 0)
        {
            const int x = q.g[0] + offsets[3 * j], y = q.g[1] + offsets[3 * j + 1], z = q.g[2] + offsets[3 * j + 2];
            inside = (unsigned)x < (unsigned)g.n[0] && (unsigned)y < (unsigned)g.n[1] && (unsigned)z < (unsigned)g.n[2];
            if (inside)
            {
                const int c = (z * g.n[1] + y) * g.n[0] + x;
                trav = dsm_traversable(state, dist, c, radius);
                reached = trav && (!reach_cost || reach_cost[c] != 0xffffffffu);
            }
        }
    }
    const unsigned lane = threadIdx.x & 31, ballot = __ballot_sync(0xffffffffu, reached);
    int at = 0;
    if (lane == 0 && ballot) at = atomicAdd(count, __popc(ballot));
    at = __shfl_sync(0xffffffffu, at, 0);
    if (reached) list[at + __popc(ballot & ((1u << lane) - 1))] = item;
    const int n_inside = __syncthreads_count(inside), n_trav = __syncthreads_count(trav), n_reached = __syncthreads_count(reached);
    if (threadIdx.x == 0 && n_inside)
    {
        atomicAdd(&rec[i].n_inside, n_inside);
        if (n_trav) atomicAdd(&rec[i].n_traversable, n_trav);
        if (n_reached) atomicAdd(&rec[i].n_reached, n_reached);
    }
}

template <typename Grid>
__global__ void __launch_bounds__(VP_BLOCK) k_vp_score(const Grid g, const uint8_t *__restrict__ state,
                                                       const double *__restrict__ rotations, int n_rotations,
                                                       const int32_t *__restrict__ offsets, int n_offsets, const DsmVpCluster *__restrict__ cl,
                                                       const int32_t *__restrict__ members, const int32_t *__restrict__ list,
                                                       const int32_t *__restrict__ count, const uint32_t *__restrict__ reach_cost,
                                                       double fx, double fy, double cx, double cy, double width, double height,
                                                       double range2, int unknown_blocks, int min_seen, unsigned long long *__restrict__ key)
{
    __shared__ double s_rot[9 * DSM_VIEWPOINT_MAX_ROTATIONS];
    __shared__ unsigned s_cnt[DSM_VIEWPOINT_MAX_ROTATIONS];
    const int tid = threadIdx.x, lane = tid & 31;
    for (int k = tid; k < 9 * n_rotations; k += VP_BLOCK) s_rot[k] = rotations[k];
    const int n_items = *count;
    const auto &fg = vp_field(g);
    const int nx = fg.n[0], ny = fg.n[1];
    const double v = (double)g.voxel;
    for (int it = blockIdx.x; it < n_items; it += gridDim.x)
    {
        if (tid < DSM_VIEWPOINT_MAX_ROTATIONS) s_cnt[tid] = 0;
        __syncthreads();
        const int item = list[it], i = item / n_offsets, j = item % n_offsets;
        const DsmVpCluster q = cl[i];
        const int x = q.g[0] + offsets[3 * j], y = q.g[1] + offsets[3 * j + 1], z = q.g[2] + offsets[3 * j + 2];
        const int3 t = vp_camera(g, x, y, z);
        const double tx = __dmul_rn(__dadd_rn((double)(g.o[0] + t.x), 0.5), v), ty = __dmul_rn(__dadd_rn((double)(g.o[1] + t.y), 0.5), v),
                     tz = __dmul_rn(__dadd_rn((double)(g.o[2] + t.z), 0.5), v);
        for (int k0 = 0; k0 < q.n_s; k0 += VP_BLOCK)
        {
            const int k = k0 + tid;
            unsigned long long mask = 0;
            bool seen = false;
            if (k < q.n_s)
            {
                const int m = __ldg(members + q.base + (int)((long long)k * q.n / q.n_s));
                const int mx = m % nx, my = m / nx % ny, mz = m / (nx * ny);
                const double c0 = __dmul_rn(__dadd_rn((double)(g.o[0] + mx), 0.5), v), c1 = __dmul_rn(__dadd_rn((double)(g.o[1] + my), 0.5), v),
                             c2 = __dmul_rn(__dadd_rn((double)(g.o[2] + mz), 0.5), v);
                const double d0 = __dsub_rn(c0, tx), d1 = __dsub_rn(c1, ty), d2 = __dsub_rn(c2, tz);
                for (int r = 0; r < n_rotations; r++)
                    if (dsm_gain_frustum<3>(s_rot + 9 * r, d0, d1, d2, fx, fy, cx, cy, width, height, range2)) mask |= 1ull << r;
                seen = mask && dsm_gain_walk(fg, state, unknown_blocks, tx, ty, tz, c0, c1, c2);
            }
            if (__any_sync(0xffffffffu, seen))
                for (int r = 0; r < n_rotations; r++)
                {
                    const unsigned b = __ballot_sync(0xffffffffu, seen && (mask >> r & 1));
                    if (lane == 0 && b) atomicAdd(&s_cnt[r], __popc(b));
                }
        }
        __syncthreads();
        if (tid == 0)
        {
            int best = 0;
            for (int r = 1; r < n_rotations; r++)
                if (s_cnt[r] > s_cnt[best]) best = r;
            const int n_seen = (int)s_cnt[best];
            if (n_seen >= max(1, min_seen))
            {
                const uint32_t cost = reach_cost ? reach_cost[(z * g.n[1] + y) * g.n[0] + x] : 0xffffffffu;
                key[item] = vp_key(n_seen, cost, j, best);
            }
        }
        __syncthreads();
    }
}

template <typename Grid>
__global__ void __launch_bounds__(VP_BLOCK) k_vp_select(const Grid g, const int32_t *__restrict__ offsets, int n_offsets, int top_k,
                                                        const DsmVpCluster *__restrict__ cl, const unsigned long long *__restrict__ key,
                                                        dsm_viewpoint_cluster_t *__restrict__ rec, dsm_viewpoint_t *__restrict__ out)
{
    __shared__ unsigned long long s_min[VP_BLOCK / 32];
    const int i = blockIdx.x, tid = threadIdx.x;
    const unsigned long long *k_i = key + (size_t)i * n_offsets;
    unsigned long long last = 0; // every key is above 0: its top field 8191 - n_seen is at least 4095
    int n_vp = 0;
    for (int s = 0; s < top_k; s++)
    {
        unsigned long long m = VP_NONE;
        for (int j = tid; j < n_offsets; j += VP_BLOCK)
        {
            const unsigned long long k = k_i[j];
            if (k > last && k < m) m = k;
        }
        for (int o = 16; o > 0; o >>= 1)
        {
            const unsigned long long w = __shfl_xor_sync(0xffffffffu, m, o);
            m = w < m ? w : m;
        }
        if ((tid & 31) == 0) s_min[tid >> 5] = m;
        __syncthreads();
        m = s_min[0];
        for (int w = 1; w < VP_BLOCK / 32; w++) m = s_min[w] < m ? s_min[w] : m;
        __syncthreads();
        if (tid == 0)
        {
            dsm_viewpoint_t r;
            r.reserved[0] = r.reserved[1] = r.reserved[2] = 0;
            if (m == VP_NONE)
            {
                r.voxel = r.offset = r.rotation = -1;
                r.n_seen = 0;
                r.cost = 0xffffffffu;
            }
            else
            {
                const DsmVpCluster q = cl[i];
                const int j = (int)(m >> 6 & 4095);
                const int x = q.g[0] + offsets[3 * j], y = q.g[1] + offsets[3 * j + 1], z = q.g[2] + offsets[3 * j + 2];
                r.voxel = (z * g.n[1] + y) * g.n[0] + x;
                r.offset = j;
                r.rotation = (int)(m & 63);
                r.n_seen = 8191 - (int)(m >> 50);
                r.cost = (uint32_t)(m >> 18);
                n_vp++;
            }
            out[(size_t)i * top_k + s] = r;
        }
        if (m != VP_NONE) last = m;
    }
    if (tid == 0) rec[i].n_viewpoints = n_vp;
}

// the persistent CTAs of a k_vp_score instantiation on this device
static int vp_ctas(const void *score)
{
    int dev = 0, sms = 0, per = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, score, VP_BLOCK, 0) != cudaSuccess)
        return 0;
    return sms * per;
}

// byte offsets of the staged request's offsets and clusters and its end, and of the result's slots and its end
static size_t vp_stage_offsets() { return 8 * 9 * (size_t)DSM_VIEWPOINT_MAX_ROTATIONS; }
static size_t vp_stage_clusters() { return vp_stage_offsets() + 12 * (size_t)DSM_VIEWPOINT_MAX_OFFSETS; }
static size_t vp_stage_bytes(int n_clusters) { return vp_stage_clusters() + 4 * (size_t)n_clusters; }
static size_t vp_slots_at(int n) { return 4 * (size_t)DSM_VP_WORDS + sizeof(dsm_viewpoint_cluster_t) * (size_t)n; }
static size_t vp_res_bytes(int n, int top_k) { return vp_slots_at(n) + sizeof(dsm_viewpoint_t) * (size_t)n * top_k; }

extern "C" int dsm_viewpoint_enable(dsm_ctx *ctx, int max_clusters, int max_candidates)
{
    if (!ctx) return DSM_E_INVALID;
    const DsmField *f = ctx->field.get();
    if (!f || !ctx->views || ctx->viewpoint) return DSM_E_STATE;
    if (max_clusters < 1 || max_clusters > DSM_VIEWPOINT_MAX_CLUSTERS || max_candidates < 1 || max_candidates > DSM_VIEWPOINT_MAX_CANDIDATES)
        return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    auto vp = std::make_unique<DsmViewpoint>();
    vp->max_clusters = max_clusters, vp->max_candidates = max_candidates;
    vp->ctas = vp_ctas((const void *)k_vp_score<DsmFieldGrid>);
    vp->ctas_terrain = vp_ctas((const void *)k_vp_score<VpTerrainGrid>);
    const size_t stage = vp_stage_bytes(max_clusters), res = vp_res_bytes(max_clusters, DSM_VIEWPOINT_MAX_TOP_K);
    CudaOwner &o = vp->own;
    o.device(&vp->stage_dev, stage);
    o.host(&vp->stage_host, stage);
    o.device(&vp->cl, (size_t)max_clusters);
    o.device(&vp->key, (size_t)max_candidates);
    o.device(&vp->list, (size_t)max_candidates);
    o.device(&vp->count, 1);
    o.device(&vp->res, res);
    o.host(&vp->res_host, res);
    o.event(&vp->ev);
    return keep(ctx->viewpoint, vp, vp->ctas > 0 && vp->ctas_terrain > 0);
}

// The offsets of include/dsm.h in their order, written as (dx, dy, dz) triples to out (room for
// DSM_VIEWPOINT_MAX_OFFSETS); returns their number, or -1 past that room.
static int viewpoint_offsets(const dsm_viewpoint_params_t &p, int32_t *out)
{
    int n = 0;
    const int r = p.r_max / p.stride * p.stride, h = p.dz_max / p.stride * p.stride;
    for (int dz = -h; dz <= h; dz += p.stride)
        for (int dy = -r; dy <= r; dy += p.stride)
            for (int dx = -r; dx <= r; dx += p.stride)
            {
                const int q = dx * dx + dy * dy;
                if (q < p.r_min * p.r_min || q > p.r_max * p.r_max) continue;
                if (n == DSM_VIEWPOINT_MAX_OFFSETS) return -1;
                out[3 * n] = dx, out[3 * n + 1] = dy, out[3 * n + 2] = dz;
                n++;
            }
    return n;
}

// The argument checks both enqueues share (include/dsm.h), on a grid of voxel edge v: the offsets written to the
// staging and their number returned, or -1 for DSM_E_INVALID
static int vp_args(const DsmViewpoint &vp, const dsm_gain_camera_t *camera, const double *rotations, int n_rotations,
                   const int32_t *clusters, int n_clusters, const dsm_viewpoint_params_t *params, float v)
{
    if (!camera || !params || !rotations || n_rotations < 1 || n_rotations > DSM_VIEWPOINT_MAX_ROTATIONS || n_clusters < 0 ||
        n_clusters > vp.max_clusters || (n_clusters > 0 && !clusters))
        return -1;
    const dsm_gain_camera_t &c = *camera;
    const dsm_viewpoint_params_t &p = *params;
    if (!gain_camera_ok(c, (double)v)) return -1;
    if (p.r_min < 0 || p.r_min > p.r_max || p.r_max > DSM_VIEWPOINT_MAX_RADIUS || p.dz_max < 0 || p.dz_max > DSM_VIEWPOINT_MAX_DZ ||
        p.stride < 1 || p.stride > DSM_VIEWPOINT_MAX_STRIDE || p.max_samples < 1 || p.max_samples > DSM_VIEWPOINT_MAX_SAMPLES ||
        p.min_seen < 0 || p.top_k < 1 || p.top_k > DSM_VIEWPOINT_MAX_TOP_K || (p.with_reach != 0 && p.with_reach != 1) ||
        !std::isfinite(p.radius) || !(p.radius >= 0.f))
        return -1;
    for (size_t i = 0; i < 9 * (size_t)n_rotations; i++)
        if (!std::isfinite(rotations[i])) return -1;
    for (int i = 0; i < n_clusters; i++)
        if (clusters[i] < 0) return -1;
    // the previous job's copy out of this staging ended before its wait, which no job in flight implies
    const int n_offsets = viewpoint_offsets(p, reinterpret_cast<int32_t *>(vp.stage_host + vp_stage_offsets()));
    if (n_offsets < 1 || (long long)n_clusters * n_offsets > vp.max_candidates ||
        (long long)n_clusters * n_offsets * p.max_samples > DSM_VIEWPOINT_MAX_WORK)
        return -1;
    return n_offsets;
}

// The job on grid g after vp_args: the rotations and clusters staged, one H2D copy, the kernels with the candidates'
// traversable test on (state, dist), the walk on the field's state grid walk_state, the error words of fhdr and the
// latest frontier job's device result, then the enqueue's submit of the field request `request`
template <typename Grid>
static int vp_launch(dsm_ctx *ctx, DsmViewpoint &vp, const Grid &g, int ctas, const uint8_t *state, const int32_t *dist,
                     const uint8_t *walk_state, const int32_t *fhdr, const DsmFrontier &fr, const uint32_t *cost, const dsm_gain_camera_t &c,
                     const double *rotations, int n_rotations, const int32_t *clusters, int n_clusters, const dsm_viewpoint_params_t &p,
                     int n_offsets, uint64_t request)
{
    CK(cudaSetDevice(ctx->device));
    const cudaStream_t st = ctx->stream;
    std::memcpy(vp.stage_host, rotations, 72 * (size_t)n_rotations);
    if (n_clusters > 0) std::memcpy(vp.stage_host + vp_stage_clusters(), clusters, 4 * (size_t)n_clusters);
    CK(cudaMemcpyAsync(vp.stage_dev, vp.stage_host, vp_stage_bytes(n_clusters), cudaMemcpyHostToDevice, st));
    int32_t *hdr = reinterpret_cast<int32_t *>(vp.res);
    auto *rec = reinterpret_cast<dsm_viewpoint_cluster_t *>(vp.res + 4 * DSM_VP_WORDS);
    auto *out = reinterpret_cast<dsm_viewpoint_t *>(vp.res + vp_slots_at(n_clusters));
    const auto *table = reinterpret_cast<const dsm_frontier_cluster_t *>(fr.res + DsmFrontier::table_at());
    const int32_t *members = reinterpret_cast<const int32_t *>(fr.res + fr.list_at());
    const double *rot = reinterpret_cast<const double *>(vp.stage_dev);
    const int32_t *offsets = reinterpret_cast<const int32_t *>(vp.stage_dev + vp_stage_offsets());
    k_vp_clusters<<<(unsigned)std::max((n_clusters + VP_BLOCK - 1) / VP_BLOCK, 1), VP_BLOCK, 0, st>>>(
        g, fhdr, reinterpret_cast<const int32_t *>(fr.res), table, fr.max_clusters,
        reinterpret_cast<const int32_t *>(vp.stage_dev + vp_stage_clusters()), n_clusters, n_offsets, n_rotations, p.top_k, c.unknown_blocks,
        p.with_reach, p.max_samples, hdr, rec, vp.cl, vp.count);
    if (n_clusters > 0)
    {
        k_vp_candidates<<<dim3((unsigned)((n_offsets + VP_BLOCK - 1) / VP_BLOCK), (unsigned)n_clusters), VP_BLOCK, 0, st>>>(
            g, state, dist, offsets, n_offsets, p.radius, cost, vp.cl, rec, vp.key, vp.list, vp.count);
        const double R = (double)c.max_range;
        k_vp_score<<<(unsigned)ctas, VP_BLOCK, 0, st>>>(g, walk_state, rot, n_rotations, offsets, n_offsets, vp.cl, members, vp.list, vp.count,
                                                        cost, c.fx, c.fy, c.cx, c.cy, (double)c.width, (double)c.height, R * R,
                                                        c.unknown_blocks, p.min_seen, vp.key);
        k_vp_select<<<(unsigned)n_clusters, VP_BLOCK, 0, st>>>(g, offsets, n_offsets, p.top_k, vp.cl, vp.key, rec, out);
    }
    CK(cudaGetLastError());
    vp.n_clusters = n_clusters, vp.top_k = p.top_k;
    return submit(ctx, vp, vp.res, vp_res_bytes(n_clusters, p.top_k), request);
}

// Enqueue only: the rotations, offsets and clusters staged and copied, the kernels on the grids of the latest (known)
// field request, the latest frontier job's device result and (with_reach) the latest reach job's cost grid, one D2H copy
// of the used result and the event.  Later field, frontier and reach requests overwrite those buffers only behind the
// job.
extern "C" int dsm_viewpoint_enqueue(dsm_ctx *ctx, const dsm_gain_camera_t *camera, const double *rotations, int n_rotations,
                                     const int32_t *clusters, int n_clusters, const dsm_viewpoint_params_t *params)
{
    if (!ctx) return DSM_E_INVALID;
    DsmViewpoint *vp = ctx->viewpoint.get();
    const DsmField *f = known_field(ctx);
    if (!vp || !f || vp->in_flight) return DSM_E_STATE;
    const DsmFrontier *fr = ctx->frontier.get();
    if (!read_latest(fr, f)) return DSM_E_STATE;
    const int n_offsets = vp_args(*vp, camera, rotations, n_rotations, clusters, n_clusters, params, f->g.voxel);
    if (n_offsets < 0) return DSM_E_INVALID;
    const DsmReach *re = ctx->reach.get();
    if (params->with_reach && !read_latest(re, f)) return DSM_E_STATE;
    return vp_launch(ctx, *vp, f->g, vp->ctas, f->occ, f->dist, f->occ, f->dist + dsm_field_header(f->voxels), *fr,
                     params->with_reach ? re->cost[0] : nullptr, *camera, rotations, n_rotations, clusters, n_clusters, *params, n_offsets,
                     f->requests);
}

// Enqueue only: the job of dsm_viewpoint_enqueue on the plane of the latest terrain job (DESIGN.md §8.23), with the
// camera eye voxels above each candidate cell's support, in stream order behind that job.  The walk reads the field's
// state grid, so the latest field request must be the one the terrain job read; later field, terrain, frontier and
// reach requests overwrite what the job reads only behind it.
extern "C" int dsm_viewpoint_enqueue_terrain(dsm_ctx *ctx, const dsm_gain_camera_t *camera, const double *rotations, int n_rotations,
                                             const int32_t *clusters, int n_clusters, const dsm_viewpoint_params_t *params, int eye)
{
    if (!ctx) return DSM_E_INVALID;
    DsmViewpoint *vp = ctx->viewpoint.get();
    const DsmTerrain *tr = ctx->terrain.get();
    if (!vp || !tr || tr->request == 0 || tr->request != ctx->field->requests || vp->in_flight) return DSM_E_STATE;
    const DsmField *f = ctx->field.get();
    const DsmFrontier *fr = ctx->frontier.get();
    if (!(fr && fr->request == tr->request)) return DSM_E_STATE;
    const int n_offsets = vp_args(*vp, camera, rotations, n_rotations, clusters, n_clusters, params, f->g.voxel);
    if (n_offsets < 0 || params->dz_max != 0 || eye < 1 || eye > tr->headroom) return DSM_E_INVALID;
    const DsmReach *re = ctx->reach.get();
    if (params->with_reach && !(re && re->terrain == tr->enqueues)) return DSM_E_STATE;
    const int cells = tr->cells;
    VpTerrainGrid g;
    static_cast<ReachTerrainGrid &>(g) = reach_terrain_grid(f->g, *tr);
    g.level = reinterpret_cast<const int16_t *>(tr->res + DsmTerrain::level_at(cells));
    g.du = tr->up > 0 ? eye : -eye;
    return vp_launch(ctx, *vp, g, vp->ctas_terrain, tr->res + DsmTerrain::status_at(cells), reinterpret_cast<const int32_t *>(tr->res),
                     f->occ, reinterpret_cast<const int32_t *>(tr->res + DsmTerrain::header_at(cells)), *fr,
                     params->with_reach ? re->cost[0] : nullptr, *camera, rotations, n_rotations, clusters, n_clusters, *params, n_offsets,
                     tr->request);
}

extern "C" int dsm_viewpoint_wait(dsm_ctx *ctx, dsm_viewpoint_info_t *info, const dsm_viewpoint_cluster_t **clusters,
                                  const dsm_viewpoint_t **viewpoints)
{
    if (!ctx) return DSM_E_INVALID;
    DsmViewpoint *vp = ctx->viewpoint.get();
    const int rc = wait_head(ctx, vp);
    if (rc != DSM_OK) return rc;
    copy_info(info, vp->words());
    if (clusters) *clusters = reinterpret_cast<const dsm_viewpoint_cluster_t *>(vp->res_host + 4 * DSM_VP_WORDS);
    if (viewpoints) *viewpoints = reinterpret_cast<const dsm_viewpoint_t *>(vp->res_host + vp_slots_at(vp->n_clusters));
    return capacity(ctx, vp->words(), DSM_VP_ERR_TAG, "dsm_viewpoint_wait", "the field the job read");
}
