// The distance field of dsm_field_enqueue (DESIGN.md §8.7): a local voxel grid of the GPU-resident map and its exact
// Euclidean distance transform, in stream order.
//
//   k_field_mark      one pass over the live pool slots (update_times >= min_update_times) and the stored surfels: every
//                     point inside the grid stores a 1 into the occupancy grid (cleared by the caller).  Idempotent, so
//                     no atomics; the live sizes come from the device, surplus CTAs exit at once.
//   k_field_rows      per x-row, the squared 1-D distance to the nearest occupied voxel (a max scan from the left and a
//                     min scan from the right, one warp per row) into the distance grid; counts the occupied voxels.
//   k_field_lines     along y, then along z: the lower envelope of the parabolas f(u) + (x - u)^2 of one line
//                     (Meijster's separable pass) and its minimum at every voxel, in place.  One thread per line, the
//                     lanes of a warp on consecutive x, so every global access is coalesced; the envelope lives in
//                     shared memory, one packed word (f << 10 | u) per entry.  The z pass writes the fp32 distances.
// With a signed grid (DESIGN.md §8.16) the same three passes run again, after the first three, over the complement F of
// the sites: k_field_rows<KNOWN, true>, k_field_lines<false>, and k_field_lines_signed, which writes the signed distance
// of every site and copies the finished distance of every voxel of F from the first z pass.
//
// Squared distances are int32; an empty line holds FIELD_INF.  Every finite value is below 3 * 1023^2 < 2^22, so a site
// and its value pack into one word and the conversion to float is exact.  The kernels carry no error gate and are
// launched without PDL: each begins after everything enqueued before it has completed.
//
// dsm_capi.cu enqueues the field through the launchers at the end of this file; the planner queries' C ABI calls
// (dsm_field_query_enable, _enqueue, _enqueue_signed and _wait) follow their kernels.
#include "dsm_ctx.hpp"
#include <climits>

#define FIELD_INF INT_MAX
#define FIELD_MARK_BLOCK 256
#define FIELD_ROW_WARPS 8
#define FIELD_BATCH 8 // line loads in flight per thread in the envelope pass

__global__ void __launch_bounds__(FIELD_MARK_BLOCK) k_field_mark(const dsm_surfel_t *pool, const int32_t *res, int pool_grid,
                                                                 int min_update_times, const dsm_surfel_t *store,
                                                                 const int32_t *store_size, const DsmFieldGrid g, uint8_t *occ,
                                                                 int32_t *header)
{
    if (blockIdx.x == 0 && threadIdx.x == 0)
    { // the error word at the request, recorded, not waited on (as k_cloud_mirror does)
        header[DSM_FIELD_ERR_TAG] = res[2];
        header[DSM_FIELD_ERR_FRAME] = res[3];
    }
    const bool in_pool = (int)blockIdx.x < pool_grid;
    const int first = (in_pool ? blockIdx.x : blockIdx.x - pool_grid) * FIELD_MARK_BLOCK;
    const int n = in_pool ? res[1] : *store_size;
    if (first >= n) return; // the grid is sized from the host's upper bounds
    const int i = first + threadIdx.x;
    if (i >= n) return;
    const dsm_surfel_t *e = (in_pool ? pool : store) + i;
    if (in_pool && e->update_times < min_update_times) return;
    const float qx = floorf(e->px / g.voxel), qy = floorf(e->py / g.voxel), qz = floorf(e->pz / g.voxel);
    // fp32 compares against exact bounds: a NaN or infinite coordinate fails them
    if (!(qx >= g.lo[0] && qx < g.hi[0] && qy >= g.lo[1] && qy < g.hi[1] && qz >= g.lo[2] && qz < g.hi[2])) return;
    const int x = (int)qx - g.o[0], y = (int)qy - g.o[1], z = (int)qz - g.o[2];
    occ[((size_t)z * g.n[1] + y) * g.n[0] + x] = 1;
}

// KNOWN (dsm_field_enqueue_known, DESIGN.md §8.9): the grid holds states 0 unknown, 1 occupied, 2 free, the sites are
// the voxels that are not free, and the warp counts occupied, free and site voxels; CTA 0 copies the error words into
// the query view (DSM_FIELD_VIEW).  Otherwise every nonzero byte is a site and an occupied voxel.
// COMPLEMENT (the signed grid, DESIGN.md §8.16): the distance to the nearest voxel of F, the voxels that are not sites,
// into the signed grid, and the count of F into header[DSM_SIGNED_N_F] of the signed grid's header.
template <bool KNOWN, bool COMPLEMENT = false>
__global__ void __launch_bounds__(32 * FIELD_ROW_WARPS) k_field_rows(const DsmFieldGrid g, const uint8_t *occ, int32_t *dist, int32_t *header)
{
    __shared__ int32_t s_left[FIELD_ROW_WARPS][1024]; // nearest site x at or left of each x, -1 if none
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (KNOWN && !COMPLEMENT && blockIdx.x == 0 && threadIdx.x == 0)
    { // k_field_mark wrote them before this pass
        header[DSM_FIELD_VIEW + DSM_FIELD_ERR_TAG] = header[DSM_FIELD_ERR_TAG];
        header[DSM_FIELD_VIEW + DSM_FIELD_ERR_FRAME] = header[DSM_FIELD_ERR_FRAME];
    }
    const int row = blockIdx.x * FIELD_ROW_WARPS + warp, nx = g.n[0];
    if (row >= g.n[1] * g.n[2]) return;
    const uint8_t *o = occ + (size_t)row * nx;
    int32_t *out = dist + (size_t)row * nx;
    int32_t *left = s_left[warp];
    int carry = -1, count = 0, n_free = 0;
    for (int base = 0; base < nx; base += 32)
    {
        const int x = base + lane;
        const bool hit = x < nx && ((KNOWN ? o[x] != DSM_STATE_FREE : o[x] != 0) != COMPLEMENT);
        if (KNOWN && !COMPLEMENT)
        {
            const int st = x < nx ? o[x] : 0;
            count += __popc(__ballot_sync(0xffffffffu, st == DSM_STATE_OCCUPIED));
            n_free += __popc(__ballot_sync(0xffffffffu, st == DSM_STATE_FREE));
        }
        int v = hit ? x : -1;
        for (int k = 1; k < 32; k <<= 1)
        {
            const int t = __shfl_up_sync(0xffffffffu, v, k);
            if (lane >= k) v = max(v, t);
        }
        v = max(v, carry);
        if (x < nx) left[x] = v;
        carry = __shfl_sync(0xffffffffu, v, 31);
        if (!KNOWN || COMPLEMENT) count += __popc(__ballot_sync(0xffffffffu, hit));
    }
    carry = INT_MAX;
    for (int base = (nx - 1) & ~31; base >= 0; base -= 32)
    {
        const int x = base + lane;
        const bool hit = x < nx && ((KNOWN ? o[x] != DSM_STATE_FREE : o[x] != 0) != COMPLEMENT);
        int v = hit ? x : INT_MAX;
        for (int k = 1; k < 32; k <<= 1)
        {
            const int t = __shfl_down_sync(0xffffffffu, v, k);
            if (lane + k < 32) v = min(v, t);
        }
        v = min(v, carry);
        carry = __shfl_sync(0xffffffffu, v, 0);
        if (x < nx)
        {
            const int l = left[x];
            const int d = min(l >= 0 ? x - l : INT_MAX, v != INT_MAX ? v - x : INT_MAX);
            out[x] = d == INT_MAX ? FIELD_INF : d * d;
        }
    }
    if (lane == 0 && count > 0) atomicAdd(&header[COMPLEMENT ? DSM_SIGNED_N_F : DSM_FIELD_N_OCCUPIED], count);
    if (KNOWN && !COMPLEMENT && lane == 0)
    {
        if (n_free > 0) atomicAdd(&header[DSM_FIELD_N_FREE], n_free);
        if (n_free < nx) atomicAdd(&header[DSM_FIELD_VIEW + DSM_FIELD_N_OCCUPIED], nx - n_free);
    }
}

__device__ __forceinline__ uint32_t env_pack(int u, int f) { return ((uint32_t)f << 10) | (uint32_t)u; }
__device__ __forceinline__ int env_at(uint32_t e, int x)
{
    const int d = x - (int)(e & 1023u);
    return (int)(e >> 10) + d * d;
}
// the last x at which site e is at least as close as site (u, fu), u > e's site: floor of the parabolas' intersection
__device__ __forceinline__ int env_sep(uint32_t e, int u, int fu)
{
    const int s = (int)(e & 1023u), fs = (int)(e >> 10);
    const int num = u * u - s * s + fu - fs, den = 2 * (u - s);
    const int q = num / den;
    return (num % den != 0 && num < 0) ? q - 1 : q;
}

// What an envelope pass writes at each voxel of its line: the squared distance d2, the distance sqrtf((float)d2) * voxel
// (+inf for an empty line), or the signed distance (include/dsm.h): for a site (d2 > 0, the squared distance to F) the
// negative depth (1 - sqrtf((float)d2)) * voxel, for a voxel of F (d2 == 0) the finished distance at the same index of
// `pos`, and -inf for an empty line (F is empty)
enum
{
    LINES_SQUARED,
    LINES_DIST,
    LINES_SIGNED,
};

// One line of `len` voxels at stride `step` per thread; line (x, blockIdx.y) starts at dist + blockIdx.y * outer + x.
template <int OUT>
__device__ __forceinline__ void field_lines(int32_t *dist, const int32_t *pos, int nx, int len, int step, int outer, float voxel)
{
    extern __shared__ uint32_t s_env[]; // [len][32]: entry k of lane l at k * 32 + l (conflict-free)
    const int x = blockIdx.x * 32 + threadIdx.x;
    if (x >= nx) return;
    int32_t *line = dist + (size_t)blockIdx.y * outer + x;
    uint32_t *env = s_env + threadIdx.x;
    int top = -1, t_top = 0; // the envelope's last entry and the first x it is lowest at
    for (int u0 = 0; u0 < len; u0 += FIELD_BATCH)
    {
        int f[FIELD_BATCH];
#pragma unroll
        for (int j = 0; j < FIELD_BATCH; j++) f[j] = u0 + j < len ? line[(size_t)(u0 + j) * step] : FIELD_INF;
#pragma unroll
        for (int j = 0; j < FIELD_BATCH; j++)
        {
            const int u = u0 + j, fu = f[j];
            if (fu == FIELD_INF) continue;
            // drop the entries that site u is strictly closer than at the start of their interval
            while (top >= 0 && env_at(env[top * 32], t_top) > fu + (t_top - u) * (t_top - u))
            {
                top--;
                t_top = top >= 1 ? 1 + env_sep(env[(top - 1) * 32], (int)(env[top * 32] & 1023u), (int)(env[top * 32] >> 10)) : 0;
            }
            if (top < 0)
            {
                top = 0;
                t_top = 0;
                env[0] = env_pack(u, fu);
            }
            else
            {
                const int w = 1 + env_sep(env[top * 32], u, fu);
                if (w < len)
                {
                    top++;
                    t_top = w;
                    env[top * 32] = env_pack(u, fu);
                }
            }
        }
    }
    if (top < 0)
    {
        const int32_t none = OUT == LINES_SIGNED ? __float_as_int(-INFINITY) : (OUT == LINES_DIST ? __float_as_int(INFINITY) : FIELD_INF);
        for (int u = 0; u < len; u++) line[(size_t)u * step] = none;
        return;
    }
    // the lowest entry at x only moves right as x grows: advance while the next one is at least as low
    int k = 0;
    uint32_t cur = env[0];
    for (int u = 0; u < len; u++)
    {
        int d = env_at(cur, u);
        while (k < top)
        {
            const uint32_t nxt = env[(k + 1) * 32];
            const int dn = env_at(nxt, u);
            if (dn > d) break;
            k++;
            cur = nxt;
            d = dn;
        }
        if (OUT == LINES_SQUARED)
            line[(size_t)u * step] = d;
        else if (OUT == LINES_DIST)
            line[(size_t)u * step] = __float_as_int(sqrtf((float)d) * voxel);
        else
        {
            const size_t i = (size_t)blockIdx.y * outer + x + (size_t)u * step;
            line[(size_t)u * step] = d == 0 ? pos[i] : __float_as_int(__fmul_rn(__fsub_rn(1.f, sqrtf((float)d)), voxel));
        }
    }
}

// LAST: the minimum becomes sqrtf((float)d2) * voxel (+inf for an empty line) in place of the squared distance.
template <bool LAST>
__global__ void __launch_bounds__(32) k_field_lines(int32_t *dist, int nx, int len, int step, int outer, float voxel)
{
    field_lines<LAST ? LINES_DIST : LINES_SQUARED>(dist, nullptr, nx, len, step, outer, voxel);
}

// The signed grid's last pass, along z: sdist holds the squared distances to F of the y pass, dist the finished distance
// grid of the same request (its z pass has completed: both run in order on one stream), and one thread copies the site
// count and the error words of the request's query view `hdr` into the signed grid's header `shdr`.
__global__ void __launch_bounds__(32) k_field_lines_signed(int32_t *sdist, const int32_t *__restrict__ dist, const int32_t *__restrict__ hdr,
                                                           int32_t *shdr, int nx, int len, int step, int outer, float voxel)
{
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0)
    {
        shdr[DSM_SIGNED_N_SITES] = hdr[DSM_FIELD_N_OCCUPIED];
        shdr[DSM_SIGNED_ERR_TAG] = hdr[DSM_FIELD_ERR_TAG];
        shdr[DSM_SIGNED_ERR_FRAME] = hdr[DSM_FIELD_ERR_FRAME];
    }
    field_lines<LINES_SIGNED>(sdist, dist, nx, len, step, outer, voxel);
}

// ---- planner queries against the latest field (dsm_field_query_*, DESIGN.md §8.8) ----
//   k_field_query      one thread per point: fp64 addressing, eight gathers from the grid (L2-resident at planner
//                      sizes), trilinear distance and gradient in fp32, one float4 store.
//   k_field_clearance  one warp per trajectory, the lanes on consecutive samples; each lane walks the host-staged
//                      segment starts, so the device never rounds a sample count.  A shuffle reduction gives the
//                      minimum (ties to the lower index), the lowest hit and the outside count: the result is the same
//                      whatever the schedule.
// Every fp32 step is an explicit _rn intrinsic, so the numpy restatement (oracle/pyoracle_field_query.py) is bit-exact.
// The point query itself (q_sample, q_empty) lives in dsm_device.cuh, shared with the trajectory job.
// SIGNED (DESIGN.md §8.16): the same on the signed grid, whose header gives two rules in place of the "no site" one: no
// site, +inf; no voxel of F, -inf (an interpolation of infinities of one sign would be NaN).
//
// One packed request (H2D) and one packed result (D2H):
//   request  double points[n_points][3] | double waypoints[n_wp][3] | int32 offsets[n_traj + 1] | int32 first[n_wp]
//            (first[w]: the trajectory's index of waypoint w's first sample, staged by the host; the last waypoint's
//            entry is the index of the final sample)
//   result   int32 header[DSM_QUERY_WORDS] | float4 samples[n_points] | dsm_clearance_t clearance[n_traj]
enum
{
    DSM_QUERY_ERR_TAG,   // the field header's DSM_FIELD_ERR_TAG / _ERR_FRAME, copied by k_field_query
    DSM_QUERY_ERR_FRAME,
    DSM_QUERY_WORDS = 4  // 16 B: the samples stay float4-aligned
};
#define FIELD_QUERY_BLOCK 256
#define FIELD_CLEAR_WARPS 8

template <bool SIGNED>
__global__ void __launch_bounds__(FIELD_QUERY_BLOCK) k_field_query(const float *__restrict__ dist, const int32_t *__restrict__ fhdr, const DsmFieldGrid g,
                                                                   const double *__restrict__ pts, int n, float4 *__restrict__ out, int32_t *rhdr)
{
    if (blockIdx.x == 0 && threadIdx.x == 0)
    { // the field's error words at its request travel with the query's results
        rhdr[DSM_QUERY_ERR_TAG] = fhdr[DSM_FIELD_ERR_TAG];
        rhdr[DSM_QUERY_ERR_FRAME] = fhdr[DSM_FIELD_ERR_FRAME];
    }
    const int i = blockIdx.x * FIELD_QUERY_BLOCK + threadIdx.x;
    if (i >= n) return;
    const double *p = pts + 3 * (size_t)i;
    bool inside;
    float fill;
    const bool empty = q_empty<SIGNED>(fhdr, fill);
    out[i] = q_sample<true>(dist, g, empty, fill, p[0], p[1], p[2], inside);
}

template <bool SIGNED>
__global__ void __launch_bounds__(32 * FIELD_CLEAR_WARPS) k_field_clearance(const float *__restrict__ dist, const int32_t *__restrict__ fhdr,
                                                                            const DsmFieldGrid g, const double *__restrict__ wp,
                                                                            const int32_t *__restrict__ offsets, const int32_t *__restrict__ first,
                                                                            int n_traj, float radius, dsm_clearance_t *__restrict__ out)
{
    const int lane = threadIdx.x & 31, traj = blockIdx.x * FIELD_CLEAR_WARPS + (threadIdx.x >> 5);
    if (traj >= n_traj) return; // whole warps only
    float fill;
    const bool empty = q_empty<SIGNED>(fhdr, fill);
    const int last = offsets[traj + 1] - 1, total = first[last] + 1;
    float best = INFINITY;
    int arg = INT_MAX, hit = INT_MAX, outside = 0; // INT_MAX: none yet
    int w = offsets[traj]; // the segment of this lane's sample: first[w] <= s < first[w + 1], or w == last
    for (int s = lane; s < total; s += 32)
    {
        while (w < last && first[w + 1] <= s) w++;
        const double *a = wp + 3 * (size_t)w;
        double px = a[0], py = a[1], pz = a[2];
        if (w < last)
        {
            const double *b = a + 3;
            const double f = (double)(s - first[w]) / (double)(first[w + 1] - first[w]);
            px = __dadd_rn(px, __dmul_rn(f, __dsub_rn(b[0], a[0])));
            py = __dadd_rn(py, __dmul_rn(f, __dsub_rn(b[1], a[1])));
            pz = __dadd_rn(pz, __dmul_rn(f, __dsub_rn(b[2], a[2])));
        }
        bool inside;
        const float d = q_sample<false>(dist, g, empty, fill, px, py, pz, inside).x;
        if (!inside)
        {
            outside++;
            continue;
        }
        if (arg == INT_MAX || d < best) best = d, arg = s; // this lane's samples rise: the first minimum stays
        if (hit == INT_MAX && d < radius) hit = s;
    }
    for (int k = 16; k > 0; k >>= 1)
    {
        const float ob = __shfl_xor_sync(0xffffffffu, best, k);
        const int oa = __shfl_xor_sync(0xffffffffu, arg, k);
        hit = min(hit, __shfl_xor_sync(0xffffffffu, hit, k));
        outside += __shfl_xor_sync(0xffffffffu, outside, k);
        if (oa != INT_MAX && (arg == INT_MAX || ob < best || (ob == best && oa < arg))) best = ob, arg = oa;
    }
    if (lane == 0)
    {
        dsm_clearance_t c;
        c.min_dist = best;
        c.argmin = arg == INT_MAX ? -1 : arg;
        c.first_hit = hit == INT_MAX ? -1 : hit;
        c.n_outside = outside;
        out[traj] = c;
    }
}

// the packed request's sections at `base` (the pinned staging or its device twin), and the byte offsets of both layouts
struct QueryRequest
{
    double *points, *waypoints;
    int32_t *offsets, *first;
};
static QueryRequest query_request(uint8_t *base, int n_points, int n_wp, int n_traj)
{
    QueryRequest r;
    r.points = reinterpret_cast<double *>(base);
    r.waypoints = r.points + 3 * (size_t)n_points;
    r.offsets = reinterpret_cast<int32_t *>(r.waypoints + 3 * (size_t)n_wp);
    r.first = r.offsets + n_traj + 1;
    return r;
}
static size_t query_req_bytes(int n_points, int n_wp, int n_traj) { return 24 * ((size_t)n_points + n_wp) + 4 * ((size_t)n_traj + 1 + n_wp); }
static size_t query_clearance_at(int n_points) { return 16 * (1 + (size_t)n_points); }
static size_t query_res_bytes(int n_points, int n_traj) { return query_clearance_at(n_points) + 16 * (size_t)n_traj; }

extern "C" int dsm_field_query_enable(dsm_ctx *ctx, int max_points, int max_trajectories, int max_waypoints)
{
    if (!ctx) return DSM_E_INVALID;
    if (!ctx->field || ctx->field_query) return DSM_E_STATE;
    for (int n : {max_points, max_trajectories, max_waypoints})
        if (n < 0 || n > DSM_FIELD_QUERY_MAX_SAMPLES) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    auto q = std::make_unique<DsmFieldQuery>();
    q->max_points = max_points, q->max_traj = max_trajectories, q->max_wp = max_waypoints;
    const size_t req = query_req_bytes(max_points, max_waypoints, max_trajectories);
    const size_t res = query_res_bytes(max_points, max_trajectories);
    q->own.host(&q->req_host, req);
    q->own.device(&q->req_dev, req);
    q->own.device(&q->res_dev, res);
    q->own.host(&q->res_host, res);
    q->own.event(&q->ev);
    return keep(ctx->field_query, q);
}

// Stages the request on the calling thread (checking it and counting the samples on the way), then enqueues one H2D
// copy, the two kernels on the grid of the latest field request (sgn: on its signed grid), one D2H copy of the results
// and the event.
static int field_query_enqueue(dsm_ctx *ctx, bool sgn, const double *points, int n_points, const double *waypoints, const int32_t *offsets,
                               int n_trajectories, float step, float radius)
{
    if (!ctx) return DSM_E_INVALID;
    DsmFieldQuery *q = ctx->field_query.get();
    const DsmField *f = ctx->field.get();
    if (!q || !f || !f->requested || q->in_flight) return DSM_E_STATE;
    if (sgn && !f->signed_latest) return DSM_E_STATE;
    if (n_points < 0 || n_points > q->max_points || n_trajectories < 0 || n_trajectories > q->max_traj) return DSM_E_INVALID;
    if ((n_points > 0 && !points) || (n_trajectories > 0 && (!waypoints || !offsets))) return DSM_E_INVALID;
    if (!std::isfinite(step) || !(step > 0.f) || !std::isfinite(radius) || !(radius >= 0.f)) return DSM_E_INVALID;
    const int n_wp = n_trajectories > 0 ? offsets[n_trajectories] : 0;
    if (n_trajectories > 0)
    {
        if (offsets[0] != 0 || n_wp > q->max_wp) return DSM_E_INVALID;
        for (int j = 0; j < n_trajectories; j++)
            if (offsets[j + 1] <= offsets[j]) return DSM_E_INVALID;
    }
    const QueryRequest h = query_request(q->req_host, n_points, n_wp, n_trajectories);
    if (n_points > 0) std::memcpy(h.points, points, 24 * (size_t)n_points);
    // one pass over the waypoints: copy, check, and count each segment's samples m = max(1, ceil(L / step)).  The
    // ceil is an integer test, exact once q = L / step is known to be at most 2^26 (a NaN or infinite q fails that).
    const double dstep = (double)step;
    int64_t total = 0; // samples of the call so far
    for (int j = 0; j < n_trajectories; j++)
    {
        const int w0 = offsets[j], w1 = offsets[j + 1];
        int64_t s = 0; // samples of trajectory j so far
        for (int w = w0; w < w1; w++)
        {
            const double *a = waypoints + 3 * (size_t)w;
            double *c = h.waypoints + 3 * (size_t)w;
            c[0] = a[0], c[1] = a[1], c[2] = a[2];
            if (!std::isfinite(a[0]) || !std::isfinite(a[1]) || !std::isfinite(a[2])) return DSM_E_INVALID;
            h.first[w] = (int32_t)s;
            int64_t m = 1; // the last waypoint: one sample
            if (w + 1 < w1)
            {
                const double *b = a + 3;
                const double dx = b[0] - a[0], dy = b[1] - a[1], dz = b[2] - a[2];
                const double q = std::sqrt((dx * dx + dy * dy) + dz * dz) / dstep;
                if (!(q <= (double)DSM_FIELD_QUERY_MAX_SAMPLES)) return DSM_E_INVALID;
                m = (int64_t)q;
                m += (double)m < q;
                m = std::max<int64_t>(m, 1);
            }
            if (m > DSM_FIELD_QUERY_MAX_SAMPLES - total - s) return DSM_E_INVALID;
            s += m;
        }
        total += s;
    }
    if (n_trajectories > 0) std::memcpy(h.offsets, offsets, 4 * ((size_t)n_trajectories + 1));
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(q->req_dev, q->req_host, query_req_bytes(n_points, n_wp, n_trajectories), cudaMemcpyHostToDevice, ctx->stream));
    const QueryRequest d = query_request(q->req_dev, n_points, n_wp, n_trajectories);
    int32_t *r_hdr = reinterpret_cast<int32_t *>(q->res_dev);
    float4 *r_samples = reinterpret_cast<float4 *>(q->res_dev + 16);
    dsm_clearance_t *r_clear = reinterpret_cast<dsm_clearance_t *>(q->res_dev + query_clearance_at(n_points));
    // a known field's query view holds its site count where a plain field's header holds its occupied count; the signed
    // grid's header holds it in the same word
    const int32_t *grid = sgn ? f->sgn->grid : f->dist;
    const int32_t *f_hdr = grid + dsm_field_header(f->voxels) + (!sgn && f->known ? DSM_FIELD_VIEW : 0);
    const float *dist = reinterpret_cast<const float *>(grid);
    const int qb = (n_points + FIELD_QUERY_BLOCK - 1) / FIELD_QUERY_BLOCK;
    (sgn ? k_field_query<true> : k_field_query<false>)<<<qb > 1 ? qb : 1, FIELD_QUERY_BLOCK, 0, ctx->stream>>>(dist, f_hdr, f->g, d.points,
                                                                                                            n_points, r_samples, r_hdr);
    if (n_trajectories > 0)
        (sgn ? k_field_clearance<true> : k_field_clearance<false>)<<<(n_trajectories + FIELD_CLEAR_WARPS - 1) / FIELD_CLEAR_WARPS,
                                                                     32 * FIELD_CLEAR_WARPS, 0, ctx->stream>>>(
            dist, f_hdr, f->g, d.waypoints, d.offsets, d.first, n_trajectories, radius, r_clear);
    CK(cudaGetLastError());
    q->n_points = n_points, q->n_traj = n_trajectories;
    return submit(ctx, *q, q->res_dev, query_res_bytes(n_points, n_trajectories), f->requests);
}

extern "C" int dsm_field_query_enqueue(dsm_ctx *ctx, const double *points, int n_points, const double *waypoints, const int32_t *offsets,
                                       int n_trajectories, float step, float radius)
{
    return field_query_enqueue(ctx, false, points, n_points, waypoints, offsets, n_trajectories, step, radius);
}

extern "C" int dsm_field_query_enqueue_signed(dsm_ctx *ctx, const double *points, int n_points, const double *waypoints,
                                              const int32_t *offsets, int n_trajectories, float step, float radius)
{
    return field_query_enqueue(ctx, true, points, n_points, waypoints, offsets, n_trajectories, step, radius);
}

extern "C" int dsm_field_query_wait(dsm_ctx *ctx, const dsm_field_sample_t **samples, const dsm_clearance_t **clearance)
{
    if (!ctx) return DSM_E_INVALID;
    DsmFieldQuery *q = ctx->field_query.get();
    const int rc = wait_head(ctx, q);
    if (rc != DSM_OK) return rc;
    if (samples) *samples = reinterpret_cast<const dsm_field_sample_t *>(q->res_host + 16);
    if (clearance) *clearance = reinterpret_cast<const dsm_clearance_t *>(q->res_host + query_clearance_at(q->n_points));
    return capacity(ctx, q->words(), DSM_QUERY_ERR_TAG, "dsm_field_query_wait", "the field the query read");
}

int dsm_field_setup()
{
    const int smem = 1024 * 32 * 4; // the longest line
    cudaError_t e = cudaFuncSetAttribute(k_field_lines<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_field_lines<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_field_lines_signed, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    return e == cudaSuccess ? 0 : -1;
}

void dsm_launch_field_mark(const dsm_surfel_t *pool, const int32_t *res, int pool_upper, int min_update_times, const dsm_surfel_t *store,
                           const int32_t *store_size, int store_upper, const DsmFieldGrid &g, uint8_t *occ, int32_t *header, cudaStream_t s)
{
    const int pool_chunks = (pool_upper + FIELD_MARK_BLOCK - 1) / FIELD_MARK_BLOCK;
    const int pool_grid = pool_chunks > 1 ? pool_chunks : 1; // CTA 0 exists and records the error word
    const int store_grid = store ? (store_upper + FIELD_MARK_BLOCK - 1) / FIELD_MARK_BLOCK : 0;
    k_field_mark<<<pool_grid + store_grid, FIELD_MARK_BLOCK, 0, s>>>(pool, res, pool_grid, min_update_times, store, store_size, g, occ, header);
}

void dsm_launch_field_edt(const DsmFieldGrid &g, const uint8_t *occ, bool known, int32_t *dist, int32_t *header, int32_t *sdist, cudaStream_t s)
{
    const int nx = g.n[0], ny = g.n[1], nz = g.n[2];
    const int rows = ny * nz;
    const unsigned rb = (unsigned)(rows + FIELD_ROW_WARPS - 1) / FIELD_ROW_WARPS;
    if (known)
        k_field_rows<true><<<rb, 32 * FIELD_ROW_WARPS, 0, s>>>(g, occ, dist, header);
    else
        k_field_rows<false><<<rb, 32 * FIELD_ROW_WARPS, 0, s>>>(g, occ, dist, header);
    const unsigned xb = (unsigned)(nx + 31) / 32;
    // along y: lines (x, z) at stride nx; along z: lines (x, y) at stride nx * ny
    k_field_lines<false><<<dim3(xb, nz), 32, (size_t)ny * 32 * 4, s>>>(dist, nx, ny, nx, nx * ny, g.voxel);
    k_field_lines<true><<<dim3(xb, ny), 32, (size_t)nz * 32 * 4, s>>>(dist, nx, nz, nx * ny, nx, g.voxel);
    if (!sdist) return;
    // the signed grid: the same passes over the complement; its last pass reads the finished grid above
    int32_t *sheader = sdist + dsm_field_header((size_t)nx * ny * nz);
    if (known)
        k_field_rows<true, true><<<rb, 32 * FIELD_ROW_WARPS, 0, s>>>(g, occ, sdist, sheader);
    else
        k_field_rows<false, true><<<rb, 32 * FIELD_ROW_WARPS, 0, s>>>(g, occ, sdist, sheader);
    k_field_lines<false><<<dim3(xb, nz), 32, (size_t)ny * 32 * 4, s>>>(sdist, nx, ny, nx, nx * ny, g.voxel);
    k_field_lines_signed<<<dim3(xb, ny), 32, (size_t)nz * 32 * 4, s>>>(sdist, dist, header + (known ? DSM_FIELD_VIEW : 0), sheader, nx, nz,
                                                                       nx * ny, nx, g.voxel);
}

// ---- known space (dsm_views_*, dsm_field_enqueue_known, DESIGN.md §8.9) ----
//   k_views_capture  one thread per seed of a frame slot: plane row 1 (posi.xyz, mean_depth) becomes the seed's ray in
//                    camera coordinates, w = 1, or a ray with w = 0 (none) unless mean_depth > 0 and posi is finite.
//   k_field_carve    one thread per (view, ray): the fp64 Amanatides-Woo walk of include/dsm.h from the camera to the
//                    ray's end, which stores DSM_STATE_FREE into every visited grid voxel whose byte is 0.  Runs after
//                    k_field_mark and before the rows pass; only 2s are stored and only over 0s, so concurrent stores of
//                    one voxel store the same value and need no atomics.  A one-dimensional grid, view-major (`per_view`
//                    CTAs per view): gridDim.y would cap the views at 65535.
#define VIEWS_BLOCK 256

__global__ void __launch_bounds__(VIEWS_BLOCK) k_views_capture(const float4 *__restrict__ plane, int S, float4 *__restrict__ rays)
{
    const int s = blockIdx.x * VIEWS_BLOCK + threadIdx.x;
    if (s >= S) return;
    const float4 r = plane[(size_t)s * 3 + 1];
    const bool ok = r.w > 0.f && isfinite(r.x) && isfinite(r.y) && isfinite(r.z);
    rays[s] = ok ? make_float4(r.x, r.y, r.z, 1.f) : make_float4(0.f, 0.f, 0.f, 0.f);
}

__global__ void __launch_bounds__(CARVE_BLOCK) k_field_carve(const float4 *__restrict__ rays, int S, int per_view, const double *__restrict__ poses,
                                                             const int32_t *__restrict__ slots, double max_range, const DsmFieldGrid g,
                                                             uint8_t *occ)
{
    const int j = (int)blockIdx.x / per_view;
    const int s = ((int)blockIdx.x - j * per_view) * CARVE_BLOCK + threadIdx.x;
    if (s >= S) return;
    const float4 r = rays[(size_t)slots[j] * S + s];
    if (r.w == 0.f) return;
    const double *P = poses + 12 * (size_t)j; // row-major [R | t], camera to world
    const double px = (double)r.x, py = (double)r.y, pz = (double)r.z, v = (double)g.voxel;
    double a[3], b[3], d[3];
#pragma unroll
    for (int k = 0; k < 3; k++)
    {
        a[k] = P[4 * k + 3];
        b[k] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(P[4 * k], px), __dmul_rn(P[4 * k + 1], py)), __dmul_rn(P[4 * k + 2], pz)), a[k]);
        d[k] = __dsub_rn(b[k], a[k]);
    }
    const double L = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2])));
    const bool truncated = L > max_range;
    if (truncated)
    {
        const double f = __ddiv_rn(max_range, L);
#pragma unroll
        for (int k = 0; k < 3; k++) b[k] = __dadd_rn(a[k], __dmul_rn(f, d[k]));
    }
    int i[3], e[3], st[3];
    double tM[3], tD[3];
#pragma unroll
    for (int k = 0; k < 3; k++)
    {
        const double wa = __ddiv_rn(a[k], v), wb = __ddiv_rn(b[k], v);
        // a ray with a non-finite endpoint carves nothing (fmax / fmin below would pass over a NaN); the walk stays
        // within one voxel of the box of its two end voxels: a segment whose box misses the grid by more than that
        // visits nothing in it (and this keeps the voxel indices below in int range)
        if (!(isfinite(wa) && isfinite(wb))) return;
        if (!(fmax(wa, wb) >= (double)(g.o[k] - 1) && fmin(wa, wb) < (double)(g.o[k] + g.n[k] + 1))) return;
        i[k] = (int)floor(wa);
        e[k] = (int)floor(wb);
        const double delta = __dsub_rn(wb, wa);
        st[k] = delta > 0.0 ? 1 : (delta < 0.0 ? -1 : 0);
        tD[k] = st[k] != 0 ? __drcp_rn(fabs(delta)) : INFINITY;
        tM[k] = st[k] != 0 ? __ddiv_rn(__dsub_rn((double)(st[k] > 0 ? i[k] + 1 : i[k]), wa), delta) : INFINITY;
    }
    // scalars from here on: the walk picks an axis per step, and indexing the arrays by it would put them on the stack
    int ix = i[0], iy = i[1], iz = i[2];
    double mx = tM[0], my = tM[1], mz = tM[2];
    const int nx = g.n[0], ny = g.n[1], nz = g.n[2];
    while (true)
    {
        const bool end = ix == e[0] && iy == e[1] && iz == e[2];
        const int x = ix - g.o[0], y = iy - g.o[1], z = iz - g.o[2];
        if ((!end || truncated) && (unsigned)x < (unsigned)nx && (unsigned)y < (unsigned)ny && (unsigned)z < (unsigned)nz)
        {
            uint8_t *c = occ + ((size_t)z * ny + y) * nx + x;
            if (*c == DSM_STATE_UNKNOWN) *c = DSM_STATE_FREE;
        }
        if (end) break;
        // argmin, the lowest axis on ties
        if (mx <= my && mx <= mz)
        {
            if (mx > 1.0) break;
            ix += st[0];
            mx = __dadd_rn(mx, tD[0]);
        }
        else if (my <= mz)
        {
            if (my > 1.0) break;
            iy += st[1];
            my = __dadd_rn(my, tD[1]);
        }
        else
        {
            if (mz > 1.0) break;
            iz += st[2];
            mz = __dadd_rn(mz, tD[2]);
        }
    }
}

void dsm_launch_views_capture(const float4 *plane, int S, float4 *rays, cudaStream_t s)
{
    k_views_capture<<<(S + VIEWS_BLOCK - 1) / VIEWS_BLOCK, VIEWS_BLOCK, 0, s>>>(plane, S, rays);
}

void dsm_launch_field_carve(const DsmFieldGrid &g, const float4 *rays, int S, const double *poses, const int32_t *slots, int n_views,
                            float max_range, uint8_t *occ, cudaStream_t s)
{
    const int per_view = dsm_carve_ctas_per_view(S);
    if (n_views > 0)
        k_field_carve<<<(unsigned)(n_views * per_view), CARVE_BLOCK, 0, s>>>(rays, S, per_view, poses, slots, (double)max_range, g, occ);
}
