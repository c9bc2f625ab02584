// Travel cost through known free space (dsm_reach_*, DESIGN.md §8.11): the cost to go from a start voxel to every
// traversable voxel of the latest known field, the viewpoints of goals and frontier clusters, and their paths.
//
//   k_reach_start    one warp: snaps the start into its approach window, fills the header's start and target counts,
//                    copies the field's error words and schedules the start's tile for round 0.
//   k_reach_init     one thread per voxel: the traversable grid (free and dist >= radius), both cost buffers at
//                    UINT32_MAX but the start at 0, and the traversable count.
//   k_reach_round    launched max_rounds times; a fixed set of persistent CTAs walks round r's schedule, one 8x8x8 tile
//                    per CTA of 512 threads, one voxel per thread.  The tile and its one-voxel halo are staged in shared
//                    memory from buffer r % 2; Bellman-Ford sweeps in place run until __syncthreads_or reports no change
//                    (the tile-local fixed point with the halo frozen, unique whatever the interleaving); the tile is
//                    written to buffer (r + 1) % 2, and a tile that changed schedules itself and its 26 neighbours for
//                    round r + 1, a stamp per tile keeping each listed once; round 0's tile, the start's, counts as changed.  A round with an empty schedule exits at once.
//   k_reach_settle   copies the tiles of the pending schedule (non-empty only when max_rounds cut the job) into the other
//                    buffer, so both hold the latest cost of every voxel and the kernels below read buffer 0.
//   k_reach_reached  the reached count and the converged flag.
//   k_reach_targets  one warp per goal and per member of the frontier list: the window's best (cost + chamfer, voxel)
//                    by a 64-bit atomicMin; a second pass picks the lowest member attaining a cluster's minimum.
//   k_reach_records  one thread per target record.
//   k_reach_paths    one warp per reached target, lanes on the 26 neighbours and a shuffle argmin per step: a counting
//                    walk, a cub exclusive scan of the lengths, then the writing walk.
// The terrain job (dsm_reach_enqueue_terrain, DESIGN.md §8.21) runs the same kernels on the plane (P, Q, 1) of the latest
// terrain job's status and clearance planes: the rounds on flat 32 x 16 x 1 tiles (k_reach_round<32, 16, 1>: a 34 x 18
// halo, 8 neighbours per sweep, 9 neighbour tiles), and the target kernels on a ReachTerrainGrid, which maps a frontier
// member voxel to its column's cell.
// The matrix job (dsm_reach_matrix_*, DESIGN.md §8.13) runs the same rounds from many sites at once; its kernels follow
// the reach job's C ABI calls (dsm_reach_enable, _enqueue and _wait) below, share reach_snap and reach_relax with
// k_reach_start and k_reach_round, and are followed by its own (dsm_reach_matrix_enable, _enqueue and _wait).
// The kernels carry no error gate and are launched without PDL, as the other field kernels.
#include "dsm_ctx.hpp"
#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>
#include <type_traits>

// One packed result (D2H):
//   int32 header[DSM_REACH_WORDS] | dsm_reach_target_t targets[max_targets] | int32 path[max_path_voxels]
// The header's first 14 words are those of dsm_reach_info_t; the last two carry the field's error words.
enum
{
    DSM_REACH_ORIGIN = 0, // 3 words
    DSM_REACH_START_VOXEL = 3,
    DSM_REACH_START_STATUS,
    DSM_REACH_START_APPROACH,
    DSM_REACH_ROUNDS,
    DSM_REACH_CONVERGED,
    DSM_REACH_N_TRAVERSABLE,
    DSM_REACH_N_REACHED,
    DSM_REACH_N_GOALS,
    DSM_REACH_N_CLUSTERS_TOTAL,
    DSM_REACH_N_TARGETS,
    DSM_REACH_N_PATH_VOXELS,
    DSM_REACH_ERR_TAG, // the field header's DSM_FIELD_ERR_TAG / _ERR_FRAME, copied by k_reach_start
    DSM_REACH_ERR_FRAME,
    DSM_REACH_WORDS = 16 // 64 B
};
#define DSM_REACH_TILE 8 // tiles of 8 x 8 x 8 voxels, one CTA of 512 threads each
#define RC_BLOCK 256
#define RC_T DSM_REACH_TILE
#define RC_TILE (RC_T * RC_T * RC_T) // 512 threads
#define RC_H (RC_T + 2)              // the staged tile with its halo
#define RC_INF 0xffffffffu
#define RC_FLAT_X 32 // the terrain job's tiles: 32 x 16 x 1 cells of its plane
#define RC_FLAT_Y 16

// A round's tile of TX x TY x TZ voxels, one per CTA of RC_TILE threads, and the shared-memory halo it is staged with.
// A flat tile (TZ == 1) runs on a grid one voxel thick: no halo and no moves along z, and 9 neighbour tiles.
template <int TX, int TY, int TZ>
struct ReachTile
{
    static_assert(TX * TY * TZ == RC_TILE, "one voxel per thread");
    static constexpr int DZ = TZ == 1 ? 0 : 1; // the moves' z offsets span -DZ .. DZ
    static constexpr int HX = TX + 2, HY = TY + 2, HZ = TZ + 2 * DZ;
    static constexpr int HALO = HX * HY * HZ;
    static constexpr int NB = DZ ? 27 : 9; // the tile and its neighbour tiles
};

static_assert(sizeof(dsm_reach_target_t) == 32 && sizeof(dsm_reach_info_t) == 64, "dsm_reach layouts");
static_assert(DSM_REACH_N_PATH_VOXELS == 13 && DSM_REACH_WORDS * 4 == sizeof(dsm_reach_info_t), "the header starts with the info");
static_assert(DSM_FRONTIER_N_LISTED == 3 && DSM_FRONTIER_N_CLUSTERS == 2, "frontier header words");

// the cost of a move or an offset: 10 a + 4 b + 3 c for the sorted absolute components a >= b >= c
__host__ __device__ __forceinline__ int reach_chamfer(int dx, int dy, int dz)
{
    dx = abs(dx), dy = abs(dy), dz = abs(dz);
    const int a = max(dx, max(dy, dz)), c = min(dx, min(dy, dz)), b = dx + dy + dz - a - c;
    return 10 * a + 4 * b + 3 * c;
}

__device__ __forceinline__ bool reach_inside(const DsmFieldGrid &g, int x, int y, int z)
{
    return (unsigned)x < (unsigned)g.n[0] && (unsigned)y < (unsigned)g.n[1] && (unsigned)z < (unsigned)g.n[2];
}
__device__ __forceinline__ int reach_index(const DsmFieldGrid &g, int x, int y, int z) { return (z * g.n[1] + y) * g.n[0] + x; }

__device__ __forceinline__ unsigned long long warp_min64(unsigned long long v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
    {
        const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
        v = w < v ? w : v;
    }
    return v;
}

// the snap of voxel s into its window (include/dsm.h): the least chamfer(u - s) << 32 | u over the window's traversable
// voxels u, on the whole warp; ~0 when s lies outside the grid or no voxel of the window is traversable
__device__ __forceinline__ unsigned long long reach_snap(const DsmFieldGrid &g, const uint8_t *state, const int32_t *dist, const int3 s,
                                                         float radius, int k, int lane)
{
    const int w = 2 * k + 1;
    unsigned long long key = ~0ull;
    if (reach_inside(g, s.x, s.y, s.z))
        for (int q = lane; q < w * w * w; q += 32)
        {
            const int dx = q % w - k, dy = q / w % w - k, dz = q / (w * w) - k;
            const int x = s.x + dx, y = s.y + dy, z = s.z + dz;
            if (!reach_inside(g, x, y, z)) continue;
            const int i = reach_index(g, x, y, z);
            if (!dsm_traversable(state, dist, i, radius)) continue;
            const unsigned long long c = ((unsigned long long)reach_chamfer(dx, dy, dz) << 32) | (unsigned)i;
            key = c < key ? c : key;
        }
    return warp_min64(key);
}

// The tile-local fixed point of the staged tile (vs: the tile and its halo, ReachTile's HALO words, voxel si of this
// thread, tv its traversable flag, c its cost): Bellman-Ford sweeps in place until __syncthreads_or reports no change,
// with the halo frozen; unique whatever the interleaving.  Every thread of the CTA calls it.  Returns the voxel's cost.
template <int TX, int TY, int TZ>
__device__ __forceinline__ uint32_t reach_relax(volatile uint32_t *vs, int si, bool tv, uint32_t c)
{
    typedef ReachTile<TX, TY, TZ> T;
    while (true)
    { // only traversable voxels ever hold a finite cost, so a finite neighbour is a traversable one
        bool changed = false;
        if (tv)
        {
            uint32_t best = c;
#pragma unroll
            for (int dz = -T::DZ; dz <= T::DZ; dz++)
#pragma unroll
                for (int dy = -1; dy <= 1; dy++)
#pragma unroll
                    for (int dx = -1; dx <= 1; dx++)
                    {
                        if (dx == 0 && dy == 0 && dz == 0) continue;
                        const uint32_t v = vs[si + (dz * T::HY + dy) * T::HX + dx];
                        const uint32_t w = (uint32_t)reach_chamfer(dx, dy, dz);
                        if (v != RC_INF && v + w < best) best = v + w;
                    }
            if (best < c)
            {
                c = best;
                vs[si] = c;
                changed = true;
            }
        }
        if (!__syncthreads_or(changed)) break;
    }
    return c;
}

template <int TX, int TY, int TZ>
__global__ void __launch_bounds__(32) k_reach_start(const DsmFieldGrid g, const uint8_t *__restrict__ state, const int32_t *__restrict__ dist,
                                                    const int32_t *__restrict__ fhdr, const int3 s, float radius, int k, int n_goals,
                                                    int max_targets, const int32_t *__restrict__ frontier_hdr, int frontier_max_clusters,
                                                    const int3 tn, int32_t *__restrict__ sched0, int32_t *__restrict__ stamp,
                                                    int32_t *__restrict__ count, int32_t *__restrict__ hdr)
{
    const int lane = threadIdx.x;
    const bool in = reach_inside(g, s.x, s.y, s.z);
    const unsigned long long key = reach_snap(g, state, dist, s, radius, k, lane);
    if (lane != 0) return;
    const int u = key == ~0ull ? -1 : (int)(unsigned)key;
    for (int d = 0; d < 3; d++) hdr[DSM_REACH_ORIGIN + d] = g.o[d];
    hdr[DSM_REACH_START_VOXEL] = u;
    hdr[DSM_REACH_START_STATUS] = !in ? 1 : u < 0 ? 2 : 0;
    hdr[DSM_REACH_START_APPROACH] = u < 0 ? 0 : (int)(key >> 32);
    const int n_clusters = frontier_hdr ? min(frontier_hdr[DSM_FRONTIER_N_CLUSTERS], frontier_max_clusters) : 0;
    hdr[DSM_REACH_N_GOALS] = n_goals;
    hdr[DSM_REACH_N_CLUSTERS_TOTAL] = n_clusters;
    hdr[DSM_REACH_N_TARGETS] = n_goals + min(n_clusters, max_targets - n_goals);
    hdr[DSM_REACH_ERR_TAG] = fhdr[DSM_FIELD_ERR_TAG];
    hdr[DSM_REACH_ERR_FRAME] = fhdr[DSM_FIELD_ERR_FRAME];
    count[1] = count[2] = 0;
    count[0] = u >= 0;
    if (u >= 0)
    {
        const int x = u % g.n[0], y = u / g.n[0] % g.n[1], z = u / (g.n[0] * g.n[1]);
        const int t = ((z / TZ) * tn.y + y / TY) * tn.x + x / TX;
        sched0[0] = t;
        stamp[t] = 0;
    }
}

__global__ void __launch_bounds__(RC_BLOCK) k_reach_init(const uint8_t *__restrict__ state, const int32_t *__restrict__ dist, int voxels,
                                                         float radius, uint8_t *__restrict__ trav, uint32_t *__restrict__ c0,
                                                         uint32_t *__restrict__ c1, int32_t *hdr)
{
    const int i = blockIdx.x * RC_BLOCK + threadIdx.x;
    const bool t = i < voxels && dsm_traversable(state, dist, i, radius);
    if (i < voxels)
    {
        const uint32_t c = i == hdr[DSM_REACH_START_VOXEL] ? 0u : RC_INF;
        trav[i] = t;
        c0[i] = c;
        c1[i] = c;
    }
    const int n = __syncthreads_count(t);
    if (threadIdx.x == 0 && n > 0) atomicAdd(&hdr[DSM_REACH_N_TRAVERSABLE], n);
}

template <int TX, int TY, int TZ>
__global__ void __launch_bounds__(RC_TILE) k_reach_round(const DsmFieldGrid g, const int3 tn, const uint8_t *__restrict__ trav,
                                                         const uint32_t *__restrict__ cin, uint32_t *__restrict__ cout,
                                                         const int32_t *__restrict__ sched_in, int32_t *__restrict__ sched_out,
                                                         int32_t *__restrict__ stamp, int32_t *count, int32_t *hdr, int r)
{
    typedef ReachTile<TX, TY, TZ> T;
    __shared__ uint32_t s[T::HALO];
    const int n = count[r % 3];
    if (blockIdx.x == 0 && threadIdx.x == 0)
    {
        count[(r + 2) % 3] = 0; // round r - 1's count; round r + 1 adds to it
        if (n > 0) hdr[DSM_REACH_ROUNDS] = r + 1;
    }
    if (n == 0) return;
    const int t = threadIdx.x, lx = t % TX, ly = t / TX % TY, lz = t / (TX * TY);
    const int si = ((lz + T::DZ) * T::HY + ly + 1) * T::HX + lx + 1;
    volatile uint32_t *vs = s;
    for (int q = blockIdx.x; q < n; q += gridDim.x)
    {
        const int tile = sched_in[q];
        const int tx = tile % tn.x, ty = tile / tn.x % tn.y, tz = tile / (tn.x * tn.y);
        const int x0 = tx * TX - 1, y0 = ty * TY - 1, z0 = tz * TZ - T::DZ;
        for (int h = t; h < T::HALO; h += RC_TILE)
        {
            const int x = x0 + h % T::HX, y = y0 + h / T::HX % T::HY, z = z0 + h / (T::HX * T::HY);
            s[h] = reach_inside(g, x, y, z) ? cin[reach_index(g, x, y, z)] : RC_INF;
        }
        const int x = x0 + 1 + lx, y = y0 + 1 + ly, z = z0 + T::DZ + lz;
        const bool inside = reach_inside(g, x, y, z);
        const int i = inside ? reach_index(g, x, y, z) : 0;
        const bool tv = inside && trav[i];
        __syncthreads();
        const uint32_t c0 = s[si];
        const uint32_t c = reach_relax<TX, TY, TZ>(vs, si, tv, c0);
        if (inside) cout[i] = c;
        // round 0's only tile holds the seeded start: it counts as changed even when none of its other voxels is reached,
        // or a start cut off from the rest of its tile would end the job after one round
        if ((__syncthreads_or(c != c0) || r == 0) && t < T::NB)
        {
            const int ax = tx + t % 3 - 1, ay = ty + t / 3 % 3 - 1, az = tz + t / 9 - T::DZ;
            if ((unsigned)ax < (unsigned)tn.x && (unsigned)ay < (unsigned)tn.y && (unsigned)az < (unsigned)tn.z)
            {
                const int a = (az * tn.y + ay) * tn.x + ax;
                if (atomicMax(&stamp[a], r + 1) < r + 1) sched_out[atomicAdd(&count[(r + 1) % 3], 1)] = a;
            }
        }
        __syncthreads(); // the next tile overwrites s
    }
}

template <int TX, int TY, int TZ>
__global__ void __launch_bounds__(RC_TILE) k_reach_settle(const DsmFieldGrid g, const int3 tn, const uint32_t *__restrict__ src,
                                                          uint32_t *__restrict__ dst, const int32_t *__restrict__ sched, const int32_t *count, int r)
{
    const int n = count[r % 3];
    const int t = threadIdx.x, lx = t % TX, ly = t / TX % TY, lz = t / (TX * TY);
    for (int q = blockIdx.x; q < n; q += gridDim.x)
    {
        const int tile = sched[q];
        const int x = tile % tn.x * TX + lx, y = tile / tn.x % tn.y * TY + ly, z = tile / (tn.x * tn.y) * TZ + lz;
        if (reach_inside(g, x, y, z))
        {
            const int i = reach_index(g, x, y, z);
            dst[i] = src[i];
        }
    }
}

__global__ void __launch_bounds__(RC_BLOCK) k_reach_reached(const uint32_t *__restrict__ cost, int voxels, const int32_t *count, int max_rounds, int32_t *hdr)
{
    const int i = blockIdx.x * RC_BLOCK + threadIdx.x;
    if (blockIdx.x == 0 && threadIdx.x == 0) hdr[DSM_REACH_CONVERGED] = count[max_rounds % 3] == 0;
    const int n = __syncthreads_count(i < voxels && cost[i] != RC_INF);
    if (threadIdx.x == 0 && n > 0) atomicAdd(&hdr[DSM_REACH_N_REACHED], n);
}

// the window's least (cost[u] + chamfer(g - u)) << 32 | u over reached voxels u, on the whole warp
__device__ __forceinline__ unsigned long long reach_window(const DsmFieldGrid &g, const uint8_t *trav, const uint32_t *cost, int gx, int gy,
                                                           int gz, int k, int lane)
{
    const int w = 2 * k + 1;
    unsigned long long key = ~0ull;
    for (int q = lane; q < w * w * w; q += 32)
    {
        const int dx = q % w - k, dy = q / w % w - k, dz = q / (w * w) - k;
        const int x = gx + dx, y = gy + dy, z = gz + dz;
        if (!reach_inside(g, x, y, z)) continue;
        const int i = reach_index(g, x, y, z);
        const uint32_t c = cost[i];
        if (!trav[i] || c == RC_INF) continue;
        const unsigned long long v = ((unsigned long long)(c + (uint32_t)reach_chamfer(dx, dy, dz)) << 32) | (unsigned)i;
        key = v < key ? v : key;
    }
    return warp_min64(key);
}

// A field voxel's target coordinates: the voxel itself on the field grid, the cell of its column on the terrain plane;
// reach_cell that cell's index
__device__ __forceinline__ int3 reach_member(const DsmFieldGrid &g, int v) { return make_int3(v % g.n[0], v / g.n[0] % g.n[1], v / (g.n[0] * g.n[1])); }
__device__ __forceinline__ int3 reach_member(const ReachTerrainGrid &g, int v)
{
    const int x = v % g.nf[0], y = v / g.nf[0] % g.nf[1], z = v / (g.nf[0] * g.nf[1]);
    return make_int3(g.h0 == 0 ? x : y, g.h1 == 1 ? y : z, 0); // h0 is 0 or 1, h1 is 1 or 2
}
__device__ __forceinline__ int reach_cell(const ReachTerrainGrid &g, int v)
{
    const int3 c = reach_member(g, v);
    return c.y * g.n[0] + c.x;
}

template <int PASS, typename Grid>
__global__ void __launch_bounds__(RC_BLOCK) k_reach_targets(const Grid g, const uint8_t *__restrict__ trav, const uint32_t *__restrict__ cost,
                                                            const int32_t *__restrict__ goals, const int32_t *__restrict__ fhdr,
                                                            const dsm_frontier_cluster_t *__restrict__ table, const int32_t *__restrict__ list,
                                                            int k, const int32_t *__restrict__ hdr, unsigned long long *best, int32_t *member)
{
    const int lane = threadIdx.x & 31;
    const int n_goals = hdr[DSM_REACH_N_GOALS], n_cl = hdr[DSM_REACH_N_TARGETS] - n_goals;
    const int n_members = n_cl > 0 ? fhdr[DSM_FRONTIER_N_LISTED] : 0;
    const int warps = gridDim.x * (RC_BLOCK / 32);
    for (int item = blockIdx.x * (RC_BLOCK / 32) + (threadIdx.x >> 5); item < n_goals + n_members; item += warps)
    {
        int tg, gx, gy, gz, gi = 0;
        if (item < n_goals)
        {
            if (PASS == 1) continue; // a goal is its own target voxel
            tg = item;
            gx = goals[3 * item], gy = goals[3 * item + 1], gz = goals[3 * item + 2];
            if (!reach_inside(g, gx, gy, gz)) continue;
        }
        else
        {
            const int j = item - n_goals;
            const int c = dsm_frontier_cluster_of(table, n_cl, j);
            if (c < 0) continue; // a member of a cluster past max_targets
            tg = n_goals + c;
            gi = list[j];
            const int3 m = reach_member(g, gi);
            gx = m.x, gy = m.y, gz = m.z;
        }
        const unsigned long long key = reach_window(g, trav, cost, gx, gy, gz, k, lane);
        if (lane != 0 || key == ~0ull) continue;
        if (PASS == 0)
            atomicMin(&best[tg], key);
        else if (key == best[tg])
            atomicMin(&member[tg], gi);
    }
}

template <typename Grid>
__global__ void __launch_bounds__(RC_BLOCK) k_reach_records(const Grid g, const uint32_t *__restrict__ cost, const int32_t *__restrict__ goals,
                                                            const dsm_frontier_cluster_t *__restrict__ table, const unsigned long long *__restrict__ best,
                                                            const int32_t *__restrict__ member, const int32_t *__restrict__ hdr,
                                                            dsm_reach_target_t *__restrict__ out)
{
    const int t = blockIdx.x * RC_BLOCK + threadIdx.x;
    const int n_goals = hdr[DSM_REACH_N_GOALS];
    if (t >= hdr[DSM_REACH_N_TARGETS]) return;
    dsm_reach_target_t r;
    int status;
    const unsigned long long b = best[t];
    if (t < n_goals)
    {
        const int x = goals[3 * t], y = goals[3 * t + 1], z = goals[3 * t + 2];
        const bool in = reach_inside(g, x, y, z);
        r.target = in ? reach_index(g, x, y, z) : -1;
        status = !in ? 1 : b == ~0ull ? 2 : 0;
    }
    else
    {
        const dsm_frontier_cluster_t &c = table[t - n_goals];
        status = c.offset < 0 ? 3 : b == ~0ull ? 2 : 0;
        r.target = status == 0 ? member[t] : c.first;
        if constexpr (std::is_same<Grid, ReachTerrainGrid>::value) r.target = reach_cell(g, r.target);
    }
    const int u = (int)(unsigned)b;
    r.cost = status == 0 ? (uint32_t)(b >> 32) : RC_INF;
    r.approach = status == 0 ? (int)(r.cost - cost[u]) : -1;
    r.viewpoint = status == 0 ? u : -1;
    r.path_offset = -1;
    r.path_len = 0;
    r.status = status;
    r.reserved = 0;
    out[t] = r;
}

// the walk's next voxel from x (cost cx > 0): the traversable neighbour p minimising (cost[p] + w(p, x), p), on the
// whole warp (lane l < 26 takes the l-th neighbour); -1 when none has a lower cost (a walk never meets that)
__device__ __forceinline__ int reach_step(const DsmFieldGrid &g, const uint8_t *trav, const uint32_t *cost, int x, uint32_t cx, int lane)
{
    const int d = lane < 13 ? lane : lane + 1; // 0 .. 26 without the centre, 13
    const int dx = d % 3 - 1, dy = d / 3 % 3 - 1, dz = d / 9 - 1;
    const int px = x % g.n[0] + dx, py = x / g.n[0] % g.n[1] + dy, pz = x / (g.n[0] * g.n[1]) + dz;
    unsigned long long key = ~0ull;
    if (lane < 26 && reach_inside(g, px, py, pz))
    {
        const int p = reach_index(g, px, py, pz);
        const uint32_t c = cost[p];
        if (trav[p] && c != RC_INF) key = ((unsigned long long)c + (unsigned)reach_chamfer(dx, dy, dz)) << 32 | (unsigned)p;
    }
    key = warp_min64(key);
    if (key == ~0ull) return -1;
    const int p = (int)(unsigned)key;
    return cost[p] < cx ? p : -1;
}

// WRITE == false: len[t] = the walk's voxel count (0 unless status 0) for every t < max_targets.  WRITE: the record's
// path fields, and the path start -> viewpoint at ofs[t] when it fits.
template <bool WRITE>
__global__ void __launch_bounds__(RC_BLOCK) k_reach_paths(const DsmFieldGrid g, const uint8_t *__restrict__ trav, const uint32_t *__restrict__ cost,
                                                          int max_targets, int max_path, long long *len, const long long *__restrict__ ofs,
                                                          dsm_reach_target_t *rec, int32_t *__restrict__ path, int32_t *hdr)
{
    const int lane = threadIdx.x & 31;
    const int warps = gridDim.x * (RC_BLOCK / 32), n_targets = hdr[DSM_REACH_N_TARGETS];
    for (int t = blockIdx.x * (RC_BLOCK / 32) + (threadIdx.x >> 5); t < max_targets; t += warps)
    {
        const bool reached = t < n_targets && rec[t].status == 0;
        if (!WRITE && !reached)
        {
            if (lane == 0) len[t] = 0;
            continue;
        }
        if (!reached) continue;
        long long n = 0, at = 0;
        bool listed = false;
        if (WRITE)
        {
            n = len[t], at = ofs[t];
            listed = at + n <= (long long)max_path;
            if (lane == 0)
            {
                rec[t].path_len = (int)n;
                rec[t].path_offset = listed ? (int)at : -1;
                if (listed) atomicMax(&hdr[DSM_REACH_N_PATH_VOXELS], (int)(at + n));
            }
            if (!listed) continue;
        }
        int x = rec[t].viewpoint;
        long long step = 0;
        while (true)
        {
            if (WRITE && lane == 0) path[at + n - 1 - step] = x;
            step++;
            const uint32_t cx = cost[x];
            if (cx == 0) break;
            x = reach_step(g, trav, cost, x, cx, lane);
            if (x < 0) break;
            if (WRITE && step == n) break; // the counting walk stopped here
        }
        if (!WRITE && lane == 0) len[t] = step;
    }
}

static unsigned rc_blocks(long long n) { return n > 0 ? (unsigned)((n + RC_BLOCK - 1) / RC_BLOCK) : 1u; }

// the persistent CTAs of a round kernel on this device
static int reach_ctas(const void *round)
{
    int dev = 0, sms = 0, per = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, round, RC_TILE, 0) != cudaSuccess)
        return 0;
    return sms * per;
}

// the CUB scratch of the path-length scan; 0 on a CUB error
static size_t reach_temp_bytes(const DsmReach &b)
{
    size_t n = 0;
    if (cub::DeviceScan::ExclusiveSum(nullptr, n, b.len, b.ofs, std::max(b.max_targets, 1), (cudaStream_t)0) != cudaSuccess) return 0;
    return std::max(n, (size_t)1);
}

// byte offsets of the result's path list and its end
static size_t reach_path_at(const DsmReach &b) { return 4 * (size_t)DSM_REACH_WORDS + sizeof(dsm_reach_target_t) * (size_t)b.max_targets; }
static size_t reach_res_bytes(const DsmReach &b) { return reach_path_at(b) + 4 * (size_t)b.max_path; }

extern "C" int dsm_reach_enable(dsm_ctx *ctx, int max_targets, int max_path_voxels, int max_rounds)
{
    if (!ctx) return DSM_E_INVALID;
    const DsmField *f = ctx->field.get();
    if (!f || !ctx->views || ctx->reach) return DSM_E_STATE;
    for (int n : {max_targets, max_path_voxels})
        if (n < 0 || n > DSM_REACH_MAX_CAPACITY) return DSM_E_INVALID;
    if (max_rounds < 1 || max_rounds > DSM_REACH_MAX_ROUNDS || f->voxels > (size_t)DSM_REACH_MAX_VOXELS) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    auto re = std::make_unique<DsmReach>();
    DsmReach &b = *re;
    b.voxels = (int)f->voxels;
    for (int k = 0; k < 3; k++) b.tn[k] = (f->g.n[k] + DSM_REACH_TILE - 1) / DSM_REACH_TILE;
    b.tiles = b.tn[0] * b.tn[1] * b.tn[2];
    b.max_targets = max_targets, b.max_path = max_path_voxels, b.max_rounds = max_rounds;
    b.ctas = reach_ctas((const void *)k_reach_round<RC_T, RC_T, RC_T>);
    b.ctas_flat = reach_ctas((const void *)k_reach_round<RC_FLAT_X, RC_FLAT_Y, 1>);
    const size_t tg = (size_t)std::max(max_targets, 1);
    const size_t res = reach_res_bytes(b);
    CudaOwner &o = re->own;
    o.device(&b.trav, f->voxels);
    for (uint32_t **p : {&b.cost[0], &b.cost[1]}) o.device(p, f->voxels);
    for (int32_t **p : {&b.stamp, &b.sched[0], &b.sched[1]}) o.device(p, (size_t)b.tiles);
    o.device(&b.count, 3);
    o.device(&b.goals, 3 * tg);
    o.device(&b.best, tg);
    o.device(&b.member, tg);
    o.device(&b.len, tg);
    o.device(&b.ofs, tg);
    o.device(&b.res, res);
    o.host(&re->goals_host, 3 * tg);
    o.host(&re->res_host, res);
    o.host(&re->cost_host, f->voxels);
    o.event(&re->ev);
    b.temp_bytes = reach_temp_bytes(b);
    if (b.temp_bytes) o.device(reinterpret_cast<uint8_t **>(&b.temp), b.temp_bytes);
    return keep(ctx->reach, re, b.ctas > 0 && b.ctas_flat > 0 && b.temp_bytes != 0);
}

// floor(p / (double)v) - o, clamped to [-1, n]: outside the grid stays outside
static int reach_voxel(double p, float v, int o, int n)
{
    const double q = std::floor(p / (double)v) - (double)o;
    return q < 0.0 ? -1 : q >= (double)n ? n : (int)q;
}

// a point's column on that plane: its two in-plane voxel coordinates, whatever its height
static void reach_terrain_cell(const ReachTerrainGrid &g, const double *p, int32_t out[3])
{
    out[0] = reach_voxel(p[g.h0], g.voxel, g.o[g.h0], g.n[0]);
    out[1] = reach_voxel(p[g.h1], g.voxel, g.o[g.h1], g.n[1]);
    out[2] = 0;
}

// the flat 32 x 16 tiles per axis of a plane of n0 x n1 cells
static int3 reach_flat_tn(int n0, int n1) { return make_int3((n0 + RC_FLAT_X - 1) / RC_FLAT_X, (n1 + RC_FLAT_Y - 1) / RC_FLAT_Y, 1); }

// the argument checks both enqueues share (include/dsm.h)
static bool reach_args_ok(const DsmReach &b, const double start[3], float radius, int approach, const double *goals, int n_goals)
{
    if (!start || !std::isfinite(radius) || !(radius >= 0.f) || approach < 0 || approach > DSM_REACH_MAX_APPROACH || n_goals < 0 ||
        n_goals > b.max_targets || (n_goals > 0 && !goals))
        return false;
    for (int k = 0; k < 3; k++)
        if (!std::isfinite(start[k])) return false;
    for (size_t i = 0; i < 3 * (size_t)n_goals; i++)
        if (!std::isfinite(goals[i])) return false;
    return true;
}

// The job on grid g of `cells` voxels cut into tiles of TX x TY x TZ (tn per axis, `tiles` in all, rounds on `ctas`
// persistent CTAs), over the traversable test of (state, dist) and with the field error words of fhdr, from start voxel
// s to the goal voxels already staged in b.goals and, with fr, the clusters of that frontier job; then the D2H copy of
// the cost grid with host_copy.  The enqueue submits the result.
template <int TX, int TY, int TZ, typename Grid>
static int reach_launch(dsm_ctx *ctx, DsmReach &b, const Grid &g, const int3 tn, int tiles, int ctas, int cells, const uint8_t *state,
                        const int32_t *dist, const int32_t *fhdr, const int3 s, float radius, int approach, int n_goals,
                        const DsmFrontier *fr, int host_copy)
{
    const cudaStream_t st = ctx->stream;
    const bool with_frontiers = fr != nullptr;
    CK(cudaMemsetAsync(b.res, 0, 4 * DSM_REACH_WORDS, st));
    int32_t *hdr = reinterpret_cast<int32_t *>(b.res);
    auto *rec = reinterpret_cast<dsm_reach_target_t *>(b.res + 4 * DSM_REACH_WORDS);
    int32_t *path = reinterpret_cast<int32_t *>(b.res + reach_path_at(b));
    // the frontier job's result, with frontiers
    const int32_t *frontier_hdr = with_frontiers ? reinterpret_cast<const int32_t *>(fr->res) : nullptr;
    const auto *table = with_frontiers ? reinterpret_cast<const dsm_frontier_cluster_t *>(fr->res + DsmFrontier::table_at()) : nullptr;
    const int32_t *list = with_frontiers ? reinterpret_cast<const int32_t *>(fr->res + fr->list_at()) : nullptr;
    const int frontier_max_clusters = with_frontiers ? fr->max_clusters : 0;
    CK(cudaMemsetAsync(b.stamp, 0xff, 4 * (size_t)tiles, st));
    if (b.max_targets > 0) CK(cudaMemsetAsync(b.best, 0xff, 8 * (size_t)b.max_targets, st));
    if (b.max_targets > 0) CK(cudaMemsetAsync(b.member, 0x7f, 4 * (size_t)b.max_targets, st));
    k_reach_start<TX, TY, TZ><<<1, 32, 0, st>>>(g, state, dist, fhdr, s, radius, approach, n_goals, b.max_targets, frontier_hdr,
                                                frontier_max_clusters, tn, b.sched[0], b.stamp, b.count, hdr);
    k_reach_init<<<rc_blocks(cells), RC_BLOCK, 0, st>>>(state, dist, cells, radius, b.trav, b.cost[0], b.cost[1], hdr);
    for (int r = 0; r < b.max_rounds; r++)
        k_reach_round<TX, TY, TZ><<<ctas, RC_TILE, 0, st>>>(g, tn, b.trav, b.cost[r % 2], b.cost[(r + 1) % 2], b.sched[r % 2],
                                                            b.sched[(r + 1) % 2], b.stamp, b.count, hdr, r);
    const int r = b.max_rounds;
    k_reach_settle<TX, TY, TZ><<<ctas, RC_TILE, 0, st>>>(g, tn, b.cost[r % 2], b.cost[(r + 1) % 2], b.sched[r % 2], b.count, r);
    k_reach_reached<<<rc_blocks(cells), RC_BLOCK, 0, st>>>(b.cost[0], cells, b.count, r, hdr);
    CK(cudaGetLastError());
    if (b.max_targets > 0)
    {
        const unsigned warp_blocks = 2 * (unsigned)ctas; // the target and path kernels' warps walk their work
        k_reach_targets<0><<<warp_blocks, RC_BLOCK, 0, st>>>(g, b.trav, b.cost[0], b.goals, frontier_hdr, table, list, approach, hdr, b.best,
                                                             b.member);
        if (with_frontiers)
            k_reach_targets<1><<<warp_blocks, RC_BLOCK, 0, st>>>(g, b.trav, b.cost[0], b.goals, frontier_hdr, table, list, approach, hdr,
                                                                 b.best, b.member);
        k_reach_records<<<rc_blocks(b.max_targets), RC_BLOCK, 0, st>>>(g, b.cost[0], b.goals, table, b.best, b.member, hdr, rec);
        k_reach_paths<false><<<warp_blocks, RC_BLOCK, 0, st>>>(g, b.trav, b.cost[0], b.max_targets, b.max_path, b.len, b.ofs, rec, path, hdr);
        CK(cudaGetLastError());
        size_t n = b.temp_bytes;
        CK(cub::DeviceScan::ExclusiveSum(b.temp, n, b.len, b.ofs, b.max_targets, st));
        k_reach_paths<true><<<warp_blocks, RC_BLOCK, 0, st>>>(g, b.trav, b.cost[0], b.max_targets, b.max_path, b.len, b.ofs, rec, path, hdr);
        CK(cudaGetLastError());
    }
    if (host_copy) CK(cudaMemcpyAsync(b.cost_host, b.cost[0], 4 * (size_t)cells, cudaMemcpyDeviceToHost, st));
    b.host_copy = host_copy != 0;
    return DSM_OK;
}

// Enqueue only: the goal voxels staged and copied, the job on the grids of the latest (known) field request and, with
// frontiers, on the latest frontier job's device result, one D2H copy of the result capacity (and of the cost grid with
// host_copy) and the event.  Later field and frontier requests overwrite those buffers only behind the job.
extern "C" int dsm_reach_enqueue(dsm_ctx *ctx, const double start[3], float radius, int approach, const double *goals, int n_goals,
                                 int with_frontiers, int host_copy)
{
    if (!ctx) return DSM_E_INVALID;
    DsmReach *re = ctx->reach.get();
    const DsmField *f = known_field(ctx);
    if (!re || !f || re->in_flight) return DSM_E_STATE;
    const DsmFrontier *fr = ctx->frontier.get();
    if (with_frontiers && !read_latest(fr, f)) return DSM_E_STATE;
    DsmReach &b = *re;
    if (!reach_args_ok(b, start, radius, approach, goals, n_goals)) return DSM_E_INVALID;
    const DsmFieldGrid &g = f->g;
    CK(cudaSetDevice(ctx->device));
    // the previous job's copy out of this staging ended before its wait, which no job in flight implies
    for (size_t i = 0; i < 3 * (size_t)n_goals; i++) re->goals_host[i] = reach_voxel(goals[i], g.voxel, g.o[i % 3], g.n[i % 3]);
    if (n_goals > 0) CK(cudaMemcpyAsync(b.goals, re->goals_host, 12 * (size_t)n_goals, cudaMemcpyHostToDevice, ctx->stream));
    const int3 s = make_int3(reach_voxel(start[0], g.voxel, g.o[0], g.n[0]), reach_voxel(start[1], g.voxel, g.o[1], g.n[1]),
                             reach_voxel(start[2], g.voxel, g.o[2], g.n[2]));
    const int3 tn = make_int3(b.tn[0], b.tn[1], b.tn[2]);
    const int rc = reach_launch<RC_T, RC_T, RC_T>(ctx, b, g, tn, b.tiles, b.ctas, b.voxels, f->occ, f->dist, f->dist + dsm_field_header(f->voxels),
                                                  s, radius, approach, n_goals, with_frontiers ? fr : nullptr, host_copy);
    if (rc != DSM_OK) return rc;
    re->terrain = 0;
    return submit(ctx, *re, b.res, reach_res_bytes(b), f->requests);
}

// Enqueue only: the job of dsm_reach_enqueue on the plane of the latest terrain job (DESIGN.md §8.21), the points'
// columns staged as cells of that plane, in stream order behind that job.  A later terrain, field or frontier request
// overwrites what the job reads only behind it.  The job pairs with no field request (request 0), so a field viewpoint
// job never reads its cost grid as a field's; it records the terrain job it ran on for a terrain viewpoint job.
extern "C" int dsm_reach_enqueue_terrain(dsm_ctx *ctx, const double start[3], float radius, int approach, const double *goals, int n_goals,
                                         int with_frontiers, int host_copy)
{
    if (!ctx) return DSM_E_INVALID;
    DsmReach *re = ctx->reach.get();
    const DsmTerrain *tr = ctx->terrain.get();
    if (!re || !tr || tr->request == 0 || re->in_flight) return DSM_E_STATE;
    const DsmFrontier *fr = ctx->frontier.get();
    if (with_frontiers && !(fr && fr->request == tr->request)) return DSM_E_STATE;
    DsmReach &b = *re;
    if (!reach_args_ok(b, start, radius, approach, goals, n_goals)) return DSM_E_INVALID;
    const ReachTerrainGrid g = reach_terrain_grid(ctx->field->g, *tr);
    const int cells = tr->cells;
    CK(cudaSetDevice(ctx->device));
    // the previous job's copy out of this staging ended before its wait, which no job in flight implies
    for (int i = 0; i < n_goals; i++) reach_terrain_cell(g, goals + 3 * i, re->goals_host + 3 * i);
    if (n_goals > 0) CK(cudaMemcpyAsync(b.goals, re->goals_host, 12 * (size_t)n_goals, cudaMemcpyHostToDevice, ctx->stream));
    int32_t sc[3];
    reach_terrain_cell(g, start, sc);
    const int3 s = make_int3(sc[0], sc[1], sc[2]);
    const int3 tn = reach_flat_tn(g.n[0], g.n[1]);
    const uint8_t *status = tr->res + DsmTerrain::status_at(cells);
    const int32_t *clearance = reinterpret_cast<const int32_t *>(tr->res);
    const int32_t *thdr = reinterpret_cast<const int32_t *>(tr->res + DsmTerrain::header_at(cells));
    const int rc = reach_launch<RC_FLAT_X, RC_FLAT_Y, 1>(ctx, b, g, tn, tn.x * tn.y, b.ctas_flat, cells, status, clearance, thdr, s, radius,
                                                         approach, n_goals, with_frontiers ? fr : nullptr, host_copy);
    if (rc != DSM_OK) return rc;
    re->terrain = tr->enqueues;
    return submit(ctx, *re, b.res, reach_res_bytes(b), 0);
}

extern "C" int dsm_reach_wait(dsm_ctx *ctx, dsm_reach_info_t *info, const dsm_reach_target_t **targets, const int32_t **path,
                              const uint32_t **cost)
{
    if (!ctx) return DSM_E_INVALID;
    DsmReach *re = ctx->reach.get();
    const int rc = wait_head(ctx, re);
    if (rc != DSM_OK) return rc;
    copy_info(info, re->words());
    if (targets) *targets = reinterpret_cast<const dsm_reach_target_t *>(re->res_host + 4 * DSM_REACH_WORDS);
    if (path) *path = reinterpret_cast<const int32_t *>(re->res_host + reach_path_at(*re));
    if (cost) *cost = re->host_copy ? re->cost_host : nullptr;
    return capacity(ctx, re->words(), DSM_REACH_ERR_TAG, "dsm_reach_wait", "the field the job read");
}

// ---- the matrix job (dsm_reach_matrix_*, DESIGN.md §8.13): the reach job's rounds from many sites at once, on the
// active tiles only ----
//   k_rm_tiles    one CTA per tile, one voxel per thread: the tile's traversable mask (a ballot per warp), its active
//                 flag (__syncthreads_count) and the traversable count.
//   (a cub exclusive scan of the flags)
//   k_rm_slots    one thread per tile: slot[tile] (-1 inactive), tile_of[slot] for slots below max_tiles, and the header.
//   k_rm_sites    one warp per site: the snap, the site record's first words, and round 0's schedule, u's slot.
//   k_rm_init     one CTA per (site, slot): both cost buffers at UINT32_MAX but the site's own voxel at 0.
//   k_rm_round    launched max_rounds times on persistent CTAs; each forms the exclusive prefix of the sites' round-r
//                 schedule lengths and walks the (site, slot) items, one per CTA, exactly as k_reach_round walks tiles:
//                 stage, reach_relax, write, and a changed tile schedules itself and its active neighbours per site.
//   k_rm_reached  one CTA per (site, slot): the site's reached count.
//   k_rm_gather   one thread per matrix entry; thread (i, 0) finishes site i's record.
// No settle step: every tile a round leaves out holds equal buffers (a tile that changed schedules itself), so buffer
// max_rounds % 2 holds the latest cost of every voxel, and the last two kernels read it.
// The terrain matrix job (dsm_reach_matrix_enqueue_terrain, DESIGN.md §8.22) runs the same kernels on the plane of the
// latest terrain job, as the terrain reach job does: k_rm_tiles, _sites, _init, _round and _gather on flat 32 x 16 x 1
// tiles (k_rm_round<32, 16, 1>: a 34 x 18 halo, 9 neighbour slots), k_rm_slots and k_rm_reached unchanged.
//
// One packed result of a job on n sites (D2H, 64 + 32 n + 4 n^2 B):
//   int32 header[DSM_RM_WORDS] | dsm_reach_site_t sites[n] | uint32 matrix[n][n]
// The header's first nine words are those of dsm_reach_matrix_info_t; its last two carry the field's error words,
// cleared by dsm_reach_matrix_wait.
enum
{
    DSM_RM_ORIGIN = 0, // 3 words
    DSM_RM_N_SITES = 3,
    DSM_RM_STATUS,
    DSM_RM_N_TRAVERSABLE,
    DSM_RM_N_ACTIVE_TILES,
    DSM_RM_MAX_TILES,
    DSM_RM_ROUNDS,
    DSM_RM_ERR_TAG = 14, // the field header's DSM_FIELD_ERR_TAG / _ERR_FRAME, copied by k_rm_slots
    DSM_RM_ERR_FRAME,
    DSM_RM_WORDS = 16 // 64 B
};
#define RM_SITES DSM_REACH_MATRIX_MAX_SITES
#define RM_WORDS (RC_TILE / 32) // mask words per tile
static_assert(sizeof(dsm_reach_site_t) == 32 && sizeof(dsm_reach_matrix_info_t) == 64, "dsm_reach_matrix layouts");
static_assert(DSM_RM_WORDS * 4 == sizeof(dsm_reach_matrix_info_t) && DSM_RM_ROUNDS == 8, "the header starts with the info");
static_assert(RM_SITES == 2 * RC_TILE, "k_rm_round scans two sites per thread");

__device__ __forceinline__ int3 rm_tile_xyz(const int3 tn, int tile) { return make_int3(tile % tn.x, tile / tn.x % tn.y, tile / (tn.x * tn.y)); }
// the tile of voxel u and u's tile-local index, on tiles of TX x TY x TZ
template <int TX, int TY, int TZ>
__device__ __forceinline__ int rm_tile_of_voxel(const DsmFieldGrid &g, const int3 tn, int u, int &local)
{
    const int x = u % g.n[0], y = u / g.n[0] % g.n[1], z = u / (g.n[0] * g.n[1]);
    local = ((z % TZ) * TY + y % TY) * TX + x % TX;
    return ((z / TZ) * tn.y + y / TY) * tn.x + x / TX;
}

template <int TX, int TY, int TZ>
__global__ void __launch_bounds__(RC_TILE) k_rm_tiles(const DsmFieldGrid g, const int3 tn, const uint8_t *__restrict__ state,
                                                      const int32_t *__restrict__ dist, float radius, int32_t *__restrict__ flag,
                                                      uint32_t *__restrict__ mask, int32_t *hdr)
{
    const int tile = blockIdx.x, t = threadIdx.x;
    const int3 tc = rm_tile_xyz(tn, tile);
    const int x = tc.x * TX + t % TX, y = tc.y * TY + t / TX % TY, z = tc.z * TZ + t / (TX * TY);
    const bool tv = reach_inside(g, x, y, z) && dsm_traversable(state, dist, reach_index(g, x, y, z), radius);
    const unsigned b = __ballot_sync(0xffffffffu, tv);
    if ((t & 31) == 0) mask[(size_t)tile * RM_WORDS + t / 32] = b;
    const int n = __syncthreads_count(tv);
    if (t == 0)
    {
        flag[tile] = n > 0;
        if (n > 0) atomicAdd(&hdr[DSM_RM_N_TRAVERSABLE], n);
    }
}

__global__ void __launch_bounds__(RC_BLOCK) k_rm_slots(const DsmFieldGrid g, int tiles, int max_tiles, int n_sites, const int32_t *__restrict__ flag,
                                                       const int32_t *__restrict__ scan, const int32_t *__restrict__ fhdr,
                                                       int32_t *__restrict__ slot, int32_t *__restrict__ tile_of, int32_t *hdr)
{
    const int tile = blockIdx.x * RC_BLOCK + threadIdx.x;
    if (tile >= tiles) return;
    const int s = scan[tile];
    slot[tile] = flag[tile] ? s : -1;
    if (flag[tile] && s < max_tiles) tile_of[s] = tile;
    if (tile == tiles - 1)
    {
        const int n_active = s + flag[tile];
        for (int d = 0; d < 3; d++) hdr[DSM_RM_ORIGIN + d] = g.o[d];
        hdr[DSM_RM_N_SITES] = n_sites;
        hdr[DSM_RM_STATUS] = n_active > max_tiles;
        hdr[DSM_RM_N_ACTIVE_TILES] = n_active;
        hdr[DSM_RM_MAX_TILES] = max_tiles;
        hdr[DSM_RM_ERR_TAG] = fhdr[DSM_FIELD_ERR_TAG];
        hdr[DSM_RM_ERR_FRAME] = fhdr[DSM_FIELD_ERR_FRAME];
    }
}

template <int TX, int TY, int TZ>
__global__ void __launch_bounds__(RC_BLOCK) k_rm_sites(const DsmFieldGrid g, const int3 tn, const uint8_t *__restrict__ state,
                                                       const int32_t *__restrict__ dist, const int32_t *__restrict__ sites, int n_sites,
                                                       float radius, int k, int max_tiles, const int32_t *__restrict__ slot,
                                                       int32_t *__restrict__ sched0, int32_t *__restrict__ stamp, int32_t *__restrict__ count,
                                                       const int32_t *hdr, dsm_reach_site_t *__restrict__ rec)
{
    const int i = blockIdx.x * (RC_BLOCK / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= n_sites) return;
    const int3 s = make_int3(sites[3 * i], sites[3 * i + 1], sites[3 * i + 2]);
    const unsigned long long key = reach_snap(g, state, dist, s, radius, k, lane);
    if (lane != 0) return;
    const int u = key == ~0ull ? -1 : (int)(unsigned)key;
    dsm_reach_site_t r;
    r.voxel = u;
    r.status = !reach_inside(g, s.x, s.y, s.z) ? 1 : u < 0 ? 2 : 0;
    r.approach = u < 0 ? 0 : (int)(key >> 32);
    r.rounds = r.converged = r.n_reached = 0; // k_rm_gather fills them
    r.reserved[0] = r.reserved[1] = 0;
    rec[i] = r;
    const bool seeded = u >= 0 && hdr[DSM_RM_STATUS] == 0;
    count[3 * i + 1] = count[3 * i + 2] = 0;
    count[3 * i] = seeded;
    if (seeded)
    {
        int local;
        const int a = slot[rm_tile_of_voxel<TX, TY, TZ>(g, tn, u, local)];
        sched0[(size_t)i * max_tiles] = a;
        stamp[(size_t)i * max_tiles + a] = 0;
    }
}

template <int TX, int TY, int TZ>
__global__ void __launch_bounds__(RC_TILE) k_rm_init(const DsmFieldGrid g, const int3 tn, int n_sites, int max_tiles, const int32_t *__restrict__ slot,
                                                     const dsm_reach_site_t *__restrict__ rec, const int32_t *__restrict__ hdr,
                                                     uint32_t *__restrict__ c0, uint32_t *__restrict__ c1)
{
    if (hdr[DSM_RM_STATUS] != 0) return;
    const int n_active = hdr[DSM_RM_N_ACTIVE_TILES], t = threadIdx.x;
    for (long long q = blockIdx.x; q < (long long)n_sites * n_active; q += gridDim.x)
    {
        const int i = (int)(q / n_active), a = (int)(q % n_active);
        const int u = rec[i].voxel;
        int local = -1;
        const bool own = u >= 0 && slot[rm_tile_of_voxel<TX, TY, TZ>(g, tn, u, local)] == a;
        const uint32_t c = own && local == t ? 0u : RC_INF;
        const size_t at = ((size_t)i * max_tiles + a) * RC_TILE + t;
        c0[at] = c;
        c1[at] = c;
    }
}

template <int TX, int TY, int TZ>
__global__ void __launch_bounds__(RC_TILE) k_rm_round(const int3 tn, int n_sites, int max_tiles, const int32_t *__restrict__ slot,
                                                      const int32_t *__restrict__ tile_of, const uint32_t *__restrict__ mask,
                                                      const uint32_t *__restrict__ cin, uint32_t *__restrict__ cout,
                                                      const int32_t *__restrict__ sched_in, int32_t *__restrict__ sched_out,
                                                      int32_t *__restrict__ stamp, int32_t *count, int32_t *__restrict__ rounds, int32_t *hdr, int r)
{
    typedef ReachTile<TX, TY, TZ> T;
    static_assert((TX & (TX - 1)) == 0 && (TY & (TY - 1)) == 0 && (TZ & (TZ - 1)) == 0, "the halo's masks");
    typedef cub::BlockScan<int, RC_TILE> Scan;
    __shared__ uint32_t s[T::HALO];
    __shared__ int pre[RM_SITES + 1]; // the exclusive prefix of the sites' schedule lengths; pre[n_sites] the total
    __shared__ int nb[T::NB];         // the item's neighbour slots (-1 inactive or outside), NB / 2 its own
    __shared__ typename Scan::TempStorage scan_tmp;
    const int t = threadIdx.x;
    int len[2];
    for (int e = 0; e < 2; e++) len[e] = 2 * t + e < n_sites ? count[3 * (2 * t + e) + r % 3] : 0;
    int total;
    Scan(scan_tmp).ExclusiveSum(len, len, total);
    for (int e = 0; e < 2; e++)
        if (2 * t + e < n_sites) pre[2 * t + e] = len[e];
    if (t == 0) pre[n_sites] = total;
    if (blockIdx.x == 0)
    {
        for (int i = t; i < n_sites; i += RC_TILE)
        {
            count[3 * i + (r + 2) % 3] = 0; // round r - 1's count; round r + 1 adds to it
            if (count[3 * i + r % 3] > 0) rounds[i] = r + 1;
        }
        if (t == 0 && total > 0) hdr[DSM_RM_ROUNDS] = r + 1;
    }
    if (total == 0) return;
    __syncthreads();
    const int lx = t % TX, ly = t / TX % TY, lz = t / (TX * TY);
    const int si = ((lz + T::DZ) * T::HY + ly + 1) * T::HX + lx + 1;
    volatile uint32_t *vs = s;
    for (int q = blockIdx.x; q < total; q += gridDim.x)
    {
        int lo = 0, hi = n_sites - 1; // the last site i with pre[i] <= q: the one whose schedule holds item q
        while (lo < hi)
        {
            const int mid = (lo + hi + 1) / 2;
            if (pre[mid] <= q) lo = mid;
            else hi = mid - 1;
        }
        const int i = lo;
        const size_t row = (size_t)i * max_tiles;
        const int a = sched_in[row + q - pre[i]], tile = tile_of[a];
        const int3 tc = rm_tile_xyz(tn, tile);
        if (t < T::NB)
        {
            const int ax = tc.x + t % 3 - 1, ay = tc.y + t / 3 % 3 - 1, az = tc.z + t / 9 - T::DZ;
            nb[t] = (unsigned)ax < (unsigned)tn.x && (unsigned)ay < (unsigned)tn.y && (unsigned)az < (unsigned)tn.z
                        ? slot[(az * tn.y + ay) * tn.x + ax]
                        : -1;
        }
        __syncthreads();
        for (int h = t; h < T::HALO; h += RC_TILE)
        { // halo coordinate 0 is the lower neighbour's last voxel, HX - 1 the upper neighbour's voxel 0 (a flat tile's
          // halo has one layer along z, its own)
            const int hx = h % T::HX, hy = h / T::HX % T::HY, hz = h / (T::HX * T::HY);
            const int d = (hx > 0) + (hx == T::HX - 1) + 3 * ((hy > 0) + (hy == T::HY - 1)) + 9 * T::DZ * ((hz > 0) + (hz == T::HZ - 1));
            const int local = (((hz + TZ - T::DZ) & (TZ - 1)) * TY + ((hy + TY - 1) & (TY - 1))) * TX + ((hx + TX - 1) & (TX - 1));
            const int b = nb[d];
            s[h] = b < 0 ? RC_INF : cin[(row + b) * RC_TILE + local];
        }
        const bool tv = (mask[(size_t)tile * RM_WORDS + t / 32] >> (t % 32)) & 1u;
        __syncthreads();
        const uint32_t c0 = s[si];
        const uint32_t c = reach_relax<TX, TY, TZ>(vs, si, tv, c0);
        cout[(row + a) * RC_TILE + t] = c;
        // as k_reach_round, round 0's tile is the seeded start's and counts as changed; only active tiles are listed,
        // since an inactive one holds UINT32_MAX for good
        if ((__syncthreads_or(c != c0) || r == 0) && t < T::NB)
        {
            const int b = nb[t];
            if (b >= 0 && atomicMax(&stamp[row + b], r + 1) < r + 1) sched_out[row + atomicAdd(&count[3 * i + (r + 1) % 3], 1)] = b;
        }
        __syncthreads(); // the next item overwrites s and nb
    }
}

__global__ void __launch_bounds__(RC_TILE) k_rm_reached(int n_sites, int max_tiles, const uint32_t *__restrict__ cost, const int32_t *__restrict__ hdr,
                                                        int32_t *reached)
{
    if (hdr[DSM_RM_STATUS] != 0) return;
    const int n_active = hdr[DSM_RM_N_ACTIVE_TILES];
    for (long long q = blockIdx.x; q < (long long)n_sites * n_active; q += gridDim.x)
    {
        const int i = (int)(q / n_active), a = (int)(q % n_active);
        const int n = __syncthreads_count(cost[((size_t)i * max_tiles + a) * RC_TILE + threadIdx.x] != RC_INF);
        if (threadIdx.x == 0 && n > 0) atomicAdd(&reached[i], n);
    }
}

template <int TX, int TY, int TZ>
__global__ void __launch_bounds__(RC_BLOCK) k_rm_gather(const DsmFieldGrid g, const int3 tn, int n_sites, int max_tiles, int max_rounds,
                                                        const int32_t *__restrict__ slot, const uint32_t *__restrict__ cost,
                                                        const int32_t *__restrict__ count, const int32_t *__restrict__ rounds,
                                                        const int32_t *__restrict__ reached, const int32_t *__restrict__ hdr,
                                                        dsm_reach_site_t *rec, uint32_t *__restrict__ matrix)
{
    const long long e = (long long)blockIdx.x * RC_BLOCK + threadIdx.x;
    if (e >= (long long)n_sites * n_sites) return;
    const int i = (int)(e / n_sites), j = (int)(e % n_sites);
    const bool ok = hdr[DSM_RM_STATUS] == 0;
    const int ui = rec[i].voxel, uj = rec[j].voxel; // -1 unless the site's status is 0
    uint32_t m = RC_INF;
    if (ok && ui >= 0 && uj >= 0)
    {
        int local;
        const int a = slot[rm_tile_of_voxel<TX, TY, TZ>(g, tn, uj, local)];
        m = cost[((size_t)i * max_tiles + a) * RC_TILE + local];
    }
    matrix[e] = m;
    if (j == 0)
    { // a site without a start is a reach job that reaches nothing: converged after 0 rounds; a cut job ran no round
        rec[i].rounds = ok ? rounds[i] : 0;
        rec[i].converged = ok && count[3 * i + max_rounds % 3] == 0;
        rec[i].n_reached = ok ? reached[i] : 0;
    }
}

// the CUB scratch of a tile scan over `tiles` flags; 0 on a CUB error
static size_t rm_temp_bytes(const DsmReachMatrix &b, int tiles)
{
    size_t n = 0;
    if (cub::DeviceScan::ExclusiveSum(nullptr, n, b.flag, b.scan, tiles, (cudaStream_t)0) != cudaSuccess) return 0;
    return std::max(n, (size_t)1);
}

// byte offsets of an n-site result's matrix and its end
static size_t rm_matrix_at(int n) { return 4 * (size_t)DSM_RM_WORDS + sizeof(dsm_reach_site_t) * (size_t)n; }
static size_t rm_res_bytes(int n) { return rm_matrix_at(n) + 4 * (size_t)n * n; }

extern "C" int dsm_reach_matrix_enable(dsm_ctx *ctx, int max_sites, int max_tiles, int max_rounds)
{
    if (!ctx) return DSM_E_INVALID;
    const DsmField *f = ctx->field.get();
    if (!f || !ctx->views || ctx->reach_matrix) return DSM_E_STATE;
    int tn[3];
    for (int k = 0; k < 3; k++) tn[k] = (f->g.n[k] + DSM_REACH_TILE - 1) / DSM_REACH_TILE;
    const long long tiles = (long long)tn[0] * tn[1] * tn[2];
    if (max_sites < 1 || max_sites > DSM_REACH_MATRIX_MAX_SITES || max_tiles < 1 || max_tiles > tiles || max_rounds < 1 ||
        max_rounds > DSM_REACH_MAX_ROUNDS || f->voxels > (size_t)DSM_REACH_MAX_VOXELS ||
        4096ull * (unsigned long long)max_sites * (unsigned long long)max_tiles > DSM_REACH_MATRIX_MAX_COST_BYTES)
        return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    auto rm = std::make_unique<DsmReachMatrix>();
    DsmReachMatrix &b = *rm;
    b.voxels = (int)f->voxels;
    for (int k = 0; k < 3; k++) b.tn[k] = tn[k];
    b.tiles = (int)tiles;
    b.max_sites = max_sites, b.max_tiles = max_tiles, b.max_rounds = max_rounds;
    b.ctas = reach_ctas((const void *)k_rm_round<RC_T, RC_T, RC_T>);
    b.ctas_flat = reach_ctas((const void *)k_rm_round<RC_FLAT_X, RC_FLAT_Y, 1>);
    const size_t items = (size_t)max_sites * max_tiles, res = rm_res_bytes(max_sites);
    CudaOwner &o = rm->own;
    for (int32_t **p : {&b.flag, &b.scan, &b.slot}) o.device(p, (size_t)b.tiles);
    o.device(&b.mask, 16 * (size_t)b.tiles);
    o.device(&b.tile_of, (size_t)max_tiles);
    for (uint32_t **p : {&b.cost[0], &b.cost[1]}) o.device(p, items * 512);
    for (int32_t **p : {&b.stamp, &b.sched[0], &b.sched[1]}) o.device(p, items);
    o.device(&b.count, 3 * (size_t)max_sites);
    for (int32_t **p : {&b.rounds, &b.reached}) o.device(p, (size_t)max_sites);
    o.device(&b.sites, 3 * (size_t)max_sites);
    o.device(&b.res, res);
    o.host(&rm->sites_host, 3 * (size_t)max_sites);
    o.host(&rm->res_host, res);
    o.event(&rm->ev);
    // the scan runs over the field's tiles or over the flat tiles of a terrain plane, whichever the up axis: scratch
    // for the field's count need not cover a smaller one
    b.temp_bytes = rm_temp_bytes(b, b.tiles);
    for (int a = 0; a < 3 && b.temp_bytes; a++)
    {
        const int3 ft = reach_flat_tn(f->g.n[a == 0 ? 1 : 0], f->g.n[a == 2 ? 1 : 2]);
        const size_t n = rm_temp_bytes(b, ft.x * ft.y);
        b.temp_bytes = n ? std::max(b.temp_bytes, n) : 0;
    }
    if (b.temp_bytes) o.device(reinterpret_cast<uint8_t **>(&b.temp), b.temp_bytes);
    return keep(ctx->reach_matrix, rm, b.ctas > 0 && b.ctas_flat > 0 && b.temp_bytes != 0);
}

// the argument checks both matrix enqueues share (include/dsm.h)
static bool rm_args_ok(const DsmReachMatrix &b, const double *points, int n_points, float radius, int approach)
{
    if (!points || !std::isfinite(radius) || !(radius >= 0.f) || approach < 0 || approach > DSM_REACH_MAX_APPROACH || n_points < 1 ||
        n_points > b.max_sites ||
        (unsigned long long)n_points * (unsigned long long)b.max_tiles * (unsigned long long)b.max_rounds > DSM_REACH_MATRIX_MAX_WORK)
        return false;
    for (size_t i = 0; i < 3 * (size_t)n_points; i++)
        if (!std::isfinite(points[i])) return false;
    return true;
}

// The job of n sites already staged in rm.sites_host on grid g cut into tiles of TX x TY x TZ (tn per axis, `tiles` in
// all, rounds on `ctas` persistent CTAs), over the traversable test of (state, dist) and with the field error words of
// fhdr.  The enqueue submits the result.
template <int TX, int TY, int TZ>
static int rm_launch(dsm_ctx *ctx, DsmReachMatrix &b, const DsmFieldGrid &g, const int3 tn, int tiles, int ctas, const uint8_t *state,
                     const int32_t *dist, const int32_t *fhdr, int n, float radius, int approach)
{
    const cudaStream_t st = ctx->stream;
    CK(cudaMemcpyAsync(b.sites, b.sites_host, 12 * (size_t)n, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(b.res, 0, 4 * DSM_RM_WORDS, st));
    int32_t *hdr = reinterpret_cast<int32_t *>(b.res);
    auto *rec = reinterpret_cast<dsm_reach_site_t *>(b.res + 4 * DSM_RM_WORDS);
    auto *matrix = reinterpret_cast<uint32_t *>(b.res + rm_matrix_at(n));
    CK(cudaMemsetAsync(b.stamp, 0xff, 4 * (size_t)n * b.max_tiles, st));
    CK(cudaMemsetAsync(b.rounds, 0, 4 * (size_t)n, st));
    CK(cudaMemsetAsync(b.reached, 0, 4 * (size_t)n, st));
    k_rm_tiles<TX, TY, TZ><<<tiles, RC_TILE, 0, st>>>(g, tn, state, dist, radius, b.flag, b.mask, hdr);
    CK(cudaGetLastError());
    size_t tb = b.temp_bytes;
    CK(cub::DeviceScan::ExclusiveSum(b.temp, tb, b.flag, b.scan, tiles, st));
    k_rm_slots<<<rc_blocks(tiles), RC_BLOCK, 0, st>>>(g, tiles, b.max_tiles, n, b.flag, b.scan, fhdr, b.slot, b.tile_of, hdr);
    k_rm_sites<TX, TY, TZ><<<rc_blocks(32ll * n), RC_BLOCK, 0, st>>>(g, tn, state, dist, b.sites, n, radius, approach, b.max_tiles, b.slot,
                                                                    b.sched[0], b.stamp, b.count, hdr, rec);
    k_rm_init<TX, TY, TZ><<<ctas, RC_TILE, 0, st>>>(g, tn, n, b.max_tiles, b.slot, rec, hdr, b.cost[0], b.cost[1]);
    for (int r = 0; r < b.max_rounds; r++)
        k_rm_round<TX, TY, TZ><<<ctas, RC_TILE, 0, st>>>(tn, n, b.max_tiles, b.slot, b.tile_of, b.mask, b.cost[r % 2], b.cost[(r + 1) % 2],
                                                         b.sched[r % 2], b.sched[(r + 1) % 2], b.stamp, b.count, b.rounds, hdr, r);
    const uint32_t *last = b.cost[b.max_rounds % 2];
    k_rm_reached<<<ctas, RC_TILE, 0, st>>>(n, b.max_tiles, last, hdr, b.reached);
    k_rm_gather<TX, TY, TZ><<<rc_blocks((long long)n * n), RC_BLOCK, 0, st>>>(g, tn, n, b.max_tiles, b.max_rounds, b.slot, last, b.count,
                                                                             b.rounds, b.reached, hdr, rec, matrix);
    CK(cudaGetLastError());
    b.n_sites = n;
    return DSM_OK;
}

// Enqueue only: the points' voxels staged and copied, the job on the grids of the latest (known) field request, one D2H
// copy of the n-site result and the event.  A later field request overwrites those grids only behind the job.
extern "C" int dsm_reach_matrix_enqueue(dsm_ctx *ctx, const double *points, int n_points, float radius, int approach)
{
    if (!ctx) return DSM_E_INVALID;
    DsmReachMatrix *rm = ctx->reach_matrix.get();
    const DsmField *f = known_field(ctx);
    if (!rm || !f || rm->in_flight) return DSM_E_STATE;
    DsmReachMatrix &b = *rm;
    if (!rm_args_ok(b, points, n_points, radius, approach)) return DSM_E_INVALID;
    const DsmFieldGrid &g = f->g;
    const int n = n_points;
    CK(cudaSetDevice(ctx->device));
    // the previous job's copy out of this staging ended before its wait, which no job in flight implies
    for (size_t i = 0; i < 3 * (size_t)n; i++) rm->sites_host[i] = reach_voxel(points[i], g.voxel, g.o[i % 3], g.n[i % 3]);
    const int3 tn = make_int3(b.tn[0], b.tn[1], b.tn[2]);
    const int rc = rm_launch<RC_T, RC_T, RC_T>(ctx, b, g, tn, b.tiles, b.ctas, f->occ, f->dist, f->dist + dsm_field_header(f->voxels), n,
                                               radius, approach);
    if (rc != DSM_OK) return rc;
    return submit(ctx, *rm, b.res, rm_res_bytes(n), f->requests);
}

// Enqueue only: the job of dsm_reach_matrix_enqueue on the plane of the latest terrain job (DESIGN.md §8.22), the
// points' columns staged as cells of that plane, in stream order behind that job.  A later terrain, field or frontier
// request overwrites what the job reads only behind it.  The job pairs with no field request (request 0).
extern "C" int dsm_reach_matrix_enqueue_terrain(dsm_ctx *ctx, const double *points, int n_points, float radius, int approach)
{
    if (!ctx) return DSM_E_INVALID;
    DsmReachMatrix *rm = ctx->reach_matrix.get();
    const DsmTerrain *tr = ctx->terrain.get();
    if (!rm || !tr || tr->request == 0 || rm->in_flight) return DSM_E_STATE;
    DsmReachMatrix &b = *rm;
    if (!rm_args_ok(b, points, n_points, radius, approach)) return DSM_E_INVALID;
    const ReachTerrainGrid g = reach_terrain_grid(ctx->field->g, *tr);
    const int n = n_points, cells = tr->cells;
    CK(cudaSetDevice(ctx->device));
    // the previous job's copy out of this staging ended before its wait, which no job in flight implies
    for (int i = 0; i < n; i++) reach_terrain_cell(g, points + 3 * i, rm->sites_host + 3 * i);
    const int3 tn = reach_flat_tn(g.n[0], g.n[1]);
    const uint8_t *status = tr->res + DsmTerrain::status_at(cells);
    const int32_t *clearance = reinterpret_cast<const int32_t *>(tr->res);
    const int32_t *thdr = reinterpret_cast<const int32_t *>(tr->res + DsmTerrain::header_at(cells));
    const int rc = rm_launch<RC_FLAT_X, RC_FLAT_Y, 1>(ctx, b, g, tn, tn.x * tn.y, b.ctas_flat, status, clearance, thdr, n, radius, approach);
    if (rc != DSM_OK) return rc;
    return submit(ctx, *rm, b.res, rm_res_bytes(n), 0);
}

extern "C" int dsm_reach_matrix_wait(dsm_ctx *ctx, dsm_reach_matrix_info_t *info, const dsm_reach_site_t **sites, const uint32_t **matrix)
{
    if (!ctx) return DSM_E_INVALID;
    DsmReachMatrix *rm = ctx->reach_matrix.get();
    const int rc = wait_head(ctx, rm);
    if (rc != DSM_OK) return rc;
    copy_info(info, rm->words());
    if (sites) *sites = reinterpret_cast<const dsm_reach_site_t *>(rm->res_host + 4 * DSM_RM_WORDS);
    if (matrix) *matrix = reinterpret_cast<const uint32_t *>(rm->res_host + rm_matrix_at(rm->n_sites));
    return capacity(ctx, rm->words(), DSM_RM_ERR_TAG, "dsm_reach_matrix_wait", "the field the job read");
}
