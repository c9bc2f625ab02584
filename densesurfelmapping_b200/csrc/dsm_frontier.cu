// Exploration frontiers of the latest known field (dsm_frontier_*, DESIGN.md §8.10): the 26-connected components of
// the free voxels that have an unknown face neighbour, their statistics and member lists, in stream order.
//
//   k_frontier_mark     one warp per x-row, reading the row and its four neighbouring rows (y +-1, z +-1), coalesced:
//                       label[i] = i for a frontier voxel, -1 otherwise; one atomic per warp counts them.  CTA 0 copies
//                       the field's error words into the result header.
//   k_frontier_tile     one CTA per 32x4x4 tile: the lock-free atomicMin union-find of Playne & Hawick (2018) over the
//                       13 backward neighbours inside the tile, in shared memory; every frontier voxel then points at
//                       the global index of its tile-local root (the tile's lowest index of its piece).
//   k_frontier_seam     the same union over the backward neighbours across tile faces, on the label grid.
//   k_frontier_flatten  every frontier voxel's label becomes its root: the component's lowest index, its `first`.
// The union keeps every label pointing at a lower index of the same component and links roots only by atomicMin, so
// the final roots are the components' minima whatever the interleaving.
//   roots               the voxels that are their own root, compacted in index order (fr_select): the components.
//   k_frontier_number   label[root of component k] = -2 - k, so any member finds k through its root in one step.
//   k_frontier_count    members per component (warp-aggregated integer atomics).
//   k_frontier_keep, a cub exclusive scan and k_frontier_slot: the clusters (count >= min_voxels), numbered in
//                       component order; the first max_clusters get a table slot.
//   k_frontier_reduce   per table slot, bounds, coordinate sums, unknown faces and open directions (warp-aggregated
//                       integer atomics; the sums exact in 64 bits).
//   a cub exclusive scan of the slots' sizes, then k_frontier_table: one thread per cluster writes its record, its
//                       list offset (-1 past max_voxels) and its centroid.
//   the list            the listed clusters' members compacted in linear order (fr_select) into the first n_listed
//                       entries of max_voxels, the rest keyed past every cluster, then cub's stable radix sort by table
//                       slot: members grouped by cluster in table order, ascending within one.
// The kernels carry no error gate and are launched without PDL, as the other field kernels.  The job's C ABI calls
// (dsm_frontier_enable, _enqueue and _wait) follow them.
#include "dsm_ctx.hpp"
#include <climits>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#define FR_ROW_WARPS 8
#define FR_BLOCK 256
#define FR_TX 32 // tile: 32 x 4 x 4 voxels, one thread each
#define FR_TY 4
#define FR_TZ 4
#define FR_TILE (FR_TX * FR_TY * FR_TZ)

static_assert(sizeof(dsm_frontier_cluster_t) == 96 && offsetof(dsm_frontier_cluster_t, n_faces) == 40 &&
                  offsetof(dsm_frontier_cluster_t, centroid) == 72, "dsm_frontier_cluster_t layout");
static_assert(sizeof(dsm_frontier_counts_t) == 16 && offsetof(dsm_frontier_counts_t, n_listed) == 12, "dsm_frontier_counts_t layout");
static_assert(DSM_FRONTIER_N_LISTED == 3 && 4 * DSM_FRONTIER_WORDS % 8 == 0, "the header starts with the counts");

// what k_frontier_reduce accumulates per table entry (integer atomics only)
struct DsmFrontierAcc
{
    int32_t lo[3], hi[3];
    unsigned long long sum[3], faces, open[3]; // two's complement int64
};

// the 13 backward neighbours of the 26-neighbourhood: dz < 0, or dz == 0 and dy < 0, or dz == dy == 0 and dx < 0
__constant__ int8_t c_back[13][3] = {{-1, -1, -1}, {0, -1, -1}, {1, -1, -1}, {-1, 0, -1}, {0, 0, -1}, {1, 0, -1}, {-1, 1, -1},
                                     {0, 1, -1},   {1, 1, -1},  {-1, -1, 0}, {0, -1, 0},  {1, -1, 0},  {-1, 0, 0}};

__global__ void __launch_bounds__(32 * FR_ROW_WARPS) k_frontier_mark(const DsmFieldGrid g, const uint8_t *__restrict__ st,
                                                                    const int32_t *__restrict__ fhdr, int32_t *__restrict__ label, int32_t *hdr)
{
    if (blockIdx.x == 0 && threadIdx.x == 0)
    { // the field's error words at its request travel with the result
        hdr[DSM_FRONTIER_ERR_TAG] = fhdr[DSM_FIELD_ERR_TAG];
        hdr[DSM_FRONTIER_ERR_FRAME] = fhdr[DSM_FIELD_ERR_FRAME];
    }
    const int lane = threadIdx.x & 31, row = blockIdx.x * FR_ROW_WARPS + (threadIdx.x >> 5);
    const int nx = g.n[0], ny = g.n[1], nz = g.n[2];
    if (row >= ny * nz) return; // whole warps only
    const int y = row % ny, z = row / ny;
    const size_t base = (size_t)row * nx;
    const uint8_t *c = st + base;
    const uint8_t *ym = y > 0 ? c - nx : nullptr, *yp = y + 1 < ny ? c + nx : nullptr;
    const uint8_t *zm = z > 0 ? c - (size_t)nx * ny : nullptr, *zp = z + 1 < nz ? c + (size_t)nx * ny : nullptr;
    int count = 0;
    for (int x0 = 0; x0 < nx; x0 += 32)
    {
        const int x = x0 + lane;
        bool fr = false;
        if (x < nx && c[x] == DSM_STATE_FREE)
            fr = (x > 0 && c[x - 1] == DSM_STATE_UNKNOWN) || (x + 1 < nx && c[x + 1] == DSM_STATE_UNKNOWN) ||
                 (ym && ym[x] == DSM_STATE_UNKNOWN) || (yp && yp[x] == DSM_STATE_UNKNOWN) || (zm && zm[x] == DSM_STATE_UNKNOWN) ||
                 (zp && zp[x] == DSM_STATE_UNKNOWN);
        if (x < nx) label[base + x] = fr ? (int32_t)(base + x) : -1;
        count += __popc(__ballot_sync(0xffffffffu, fr));
    }
    if (lane == 0 && count > 0) atomicAdd(&hdr[DSM_FRONTIER_N_FRONTIER], count);
}

// Union-find on labels that only ever point at a lower index of the same set; a root points at itself.  Loads bypass
// L1 (other CTAs lower the labels); every store is an atomicMin, so no link is ever raised or lost.
__device__ __forceinline__ int uf_find(int32_t *L, int x)
{
    while (true)
    {
        const int p = __ldcg(L + x);
        if (p == x) return x;
        const int gp = __ldcg(L + p);
        if (gp == p) return p;
        atomicMin(L + x, gp); // path halving
        x = gp;
    }
}
__device__ __forceinline__ void uf_union(int32_t *L, int a, int b)
{
    while (true)
    {
        a = uf_find(L, a);
        b = uf_find(L, b);
        if (a == b) return;
        if (a > b)
        {
            const int t = a;
            a = b;
            b = t;
        }
        const int old = atomicMin(L + b, a); // link the higher root under the lower
        if (old == b) return;
        b = old; // b was linked meanwhile: join its new parent with a
    }
}
// the same on a tile's shared labels
__device__ __forceinline__ int uf_find_s(volatile int32_t *L, int x)
{
    while (true)
    {
        const int p = L[x];
        if (p == x) return x;
        x = p;
    }
}
__device__ __forceinline__ void uf_union_s(int32_t *L, int a, int b)
{
    while (true)
    {
        a = uf_find_s(L, a);
        b = uf_find_s(L, b);
        if (a == b) return;
        if (a > b)
        {
            const int t = a;
            a = b;
            b = t;
        }
        const int old = atomicMin(L + b, a);
        if (old == b) return;
        b = old;
    }
}

__device__ __forceinline__ bool in_tile(int lx, int ly, int lz)
{
    return (unsigned)lx < FR_TX && (unsigned)ly < FR_TY && (unsigned)lz < FR_TZ;
}

__global__ void __launch_bounds__(FR_TILE) k_frontier_tile(const DsmFieldGrid g, int32_t *__restrict__ label)
{
    __shared__ int32_t s[FR_TILE];
    const int t = threadIdx.x, lx = t % FR_TX, ly = t / FR_TX % FR_TY, lz = t / (FR_TX * FR_TY);
    const int x = blockIdx.x * FR_TX + lx, y = blockIdx.y * FR_TY + ly, z = blockIdx.z * FR_TZ + lz;
    const int nx = g.n[0], ny = g.n[1];
    const bool inside = x < nx && y < ny && z < g.n[2];
    const size_t i = ((size_t)z * ny + y) * nx + x;
    const bool fr = inside && label[i] >= 0;
    s[t] = fr ? t : -1;
    __syncthreads();
    if (fr)
        for (int k = 0; k < 13; k++)
        {
            const int ax = lx + c_back[k][0], ay = ly + c_back[k][1], az = lz + c_back[k][2];
            if (!in_tile(ax, ay, az)) continue;
            const int u = (az * FR_TY + ay) * FR_TX + ax;
            if (s[u] >= 0) uf_union_s(s, t, u); // outside the grid s is -1
        }
    __syncthreads();
    if (!fr) return;
    const int r = uf_find_s(s, t);
    const int rx = blockIdx.x * FR_TX + r % FR_TX, ry = blockIdx.y * FR_TY + r / FR_TX % FR_TY, rz = blockIdx.z * FR_TZ + r / (FR_TX * FR_TY);
    label[i] = (int32_t)(((size_t)rz * ny + ry) * nx + rx); // the tile's order is the grid's: its lowest index
}

__global__ void __launch_bounds__(FR_TILE) k_frontier_seam(const DsmFieldGrid g, int32_t *label)
{
    const int t = threadIdx.x, lx = t % FR_TX, ly = t / FR_TX % FR_TY, lz = t / (FR_TX * FR_TY);
    // every backward neighbour is inside the tile (those with dz = -1 reach y + 1 as well)
    if (lx > 0 && lx < FR_TX - 1 && ly > 0 && ly < FR_TY - 1 && lz > 0) return;
    const int x = blockIdx.x * FR_TX + lx, y = blockIdx.y * FR_TY + ly, z = blockIdx.z * FR_TZ + lz;
    const int nx = g.n[0], ny = g.n[1], nz = g.n[2];
    if (x >= nx || y >= ny || z >= nz) return;
    const int i = (z * ny + y) * nx + x;
    if (__ldcg(label + i) < 0) return;
    for (int k = 0; k < 13; k++)
    {
        const int dx = c_back[k][0], dy = c_back[k][1], dz = c_back[k][2];
        if (in_tile(lx + dx, ly + dy, lz + dz)) continue;
        const int ax = x + dx, ay = y + dy, az = z + dz;
        if ((unsigned)ax >= (unsigned)nx || (unsigned)ay >= (unsigned)ny || az < 0) continue;
        const int j = (az * ny + ay) * nx + ax;
        if (__ldcg(label + j) >= 0) uf_union(label, i, j);
    }
}

__global__ void __launch_bounds__(FR_BLOCK) k_frontier_flatten(int32_t *label, int voxels)
{
    const int i = blockIdx.x * FR_BLOCK + threadIdx.x;
    if (i >= voxels || __ldcg(label + i) < 0) return;
    int r = i;
    while (true)
    { // no unions run any more: every store below is of the final root, the lowest index of the set
        const int p = __ldcg(label + r);
        if (p == r) break;
        r = p;
    }
    label[i] = r;
}

struct FrIsRoot
{
    const int32_t *label;
    __device__ bool operator()(int i) const { return label[i] == i; }
};

// the component of voxel i after k_frontier_number, or -1 when i is no frontier voxel
__device__ __forceinline__ int fr_comp(const int32_t *label, int i)
{
    const int l = label[i];
    if (l == -1) return -1;
    return l < -1 ? -2 - l : -2 - label[l];
}

__global__ void __launch_bounds__(FR_BLOCK) k_frontier_number(int32_t *label, const int32_t *__restrict__ roots, int32_t *count, const int32_t *hdr)
{
    const int k = blockIdx.x * FR_BLOCK + threadIdx.x;
    if (k >= hdr[DSM_FRONTIER_N_COMPONENTS]) return;
    label[roots[k]] = -2 - k;
    count[k] = 0;
}

__global__ void __launch_bounds__(FR_BLOCK) k_frontier_count(const int32_t *__restrict__ label, int voxels, int32_t *count)
{
    const int i = blockIdx.x * FR_BLOCK + threadIdx.x, lane = threadIdx.x & 31;
    const int c = i < voxels ? fr_comp(label, i) : -1;
    unsigned todo = __ballot_sync(0xffffffffu, c >= 0);
    while (todo)
    { // one atomic per component present in the warp
        const int cl = __shfl_sync(0xffffffffu, c, __ffs(todo) - 1);
        const unsigned peers = __ballot_sync(0xffffffffu, c == cl);
        if (lane == __ffs(peers) - 1) atomicAdd(&count[cl], __popc(peers));
        todo &= ~peers;
    }
}

__global__ void __launch_bounds__(FR_BLOCK) k_frontier_keep(const int32_t *__restrict__ count, int max_comp, int min_voxels,
                                                           int32_t *__restrict__ keep, const int32_t *hdr)
{
    const int k = blockIdx.x * FR_BLOCK + threadIdx.x;
    if (k >= max_comp) return;
    keep[k] = k < hdr[DSM_FRONTIER_N_COMPONENTS] && count[k] >= min_voxels;
}

// keep becomes cmap: the component's table slot, or -1 (no cluster, or past max_clusters)
__global__ void __launch_bounds__(FR_BLOCK) k_frontier_slot(const int32_t *__restrict__ count, int32_t *keep_cmap, const int32_t *__restrict__ cid,
                                                           int max_clusters, int32_t *__restrict__ slot_comp, int32_t *__restrict__ sizes,
                                                           DsmFrontierAcc *__restrict__ acc, int32_t *hdr)
{
    const int k = blockIdx.x * FR_BLOCK + threadIdx.x;
    const int n = hdr[DSM_FRONTIER_N_COMPONENTS];
    if (k >= n) return;
    const int kept = keep_cmap[k], c = cid[k];
    if (k == n - 1) hdr[DSM_FRONTIER_N_CLUSTERS] = c + kept;
    const bool slot = kept && c < max_clusters;
    keep_cmap[k] = slot ? c : -1;
    if (!slot) return;
    slot_comp[c] = k;
    sizes[c] = count[k];
    DsmFrontierAcc &a = acc[c];
    for (int d = 0; d < 3; d++)
    {
        a.lo[d] = INT_MAX, a.hi[d] = INT_MIN;
        a.sum[d] = 0ull, a.open[d] = 0ull;
    }
    a.faces = 0ull;
}

__device__ __forceinline__ void acc_add(unsigned long long *p, int v)
{
    if (v != 0) atomicAdd(p, (unsigned long long)(long long)v);
}

__global__ void __launch_bounds__(FR_BLOCK) k_frontier_reduce(const DsmFieldGrid g, const uint8_t *__restrict__ st, const int32_t *__restrict__ label,
                                                             const int32_t *__restrict__ cmap, DsmFrontierAcc *acc)
{
    const int nx = g.n[0], ny = g.n[1], nz = g.n[2], voxels = nx * ny * nz;
    const int i = blockIdx.x * FR_BLOCK + threadIdx.x, lane = threadIdx.x & 31;
    int c = -1;
    if (i < voxels)
    {
        const int k = fr_comp(label, i);
        if (k >= 0) c = cmap[k];
    }
    int x = 0, y = 0, z = 0, faces = 0, ox = 0, oy = 0, oz = 0;
    if (c >= 0)
    {
        x = i % nx, y = i / nx % ny, z = i / (nx * ny);
        const size_t sy = (size_t)nx, sz = (size_t)nx * ny;
        const bool u[6] = {x > 0 && st[i - 1] == DSM_STATE_UNKNOWN,      x + 1 < nx && st[i + 1] == DSM_STATE_UNKNOWN,
                           y > 0 && st[i - sy] == DSM_STATE_UNKNOWN,     y + 1 < ny && st[i + sy] == DSM_STATE_UNKNOWN,
                           z > 0 && st[i - sz] == DSM_STATE_UNKNOWN,     z + 1 < nz && st[i + sz] == DSM_STATE_UNKNOWN};
        faces = u[0] + u[1] + u[2] + u[3] + u[4] + u[5];
        ox = (int)u[1] - (int)u[0], oy = (int)u[3] - (int)u[2], oz = (int)u[5] - (int)u[4];
    }
    unsigned todo = __ballot_sync(0xffffffffu, c >= 0);
    while (todo)
    { // per table slot present in the warp: 32-bit warp reductions (exact: at most 32 voxels), then one set of atomics
        const int cl = __shfl_sync(0xffffffffu, c, __ffs(todo) - 1);
        const bool in = c == cl;
        const unsigned peers = __ballot_sync(0xffffffffu, in);
        const int lo_x = __reduce_min_sync(0xffffffffu, in ? x : INT_MAX), hi_x = __reduce_max_sync(0xffffffffu, in ? x : INT_MIN);
        const int lo_y = __reduce_min_sync(0xffffffffu, in ? y : INT_MAX), hi_y = __reduce_max_sync(0xffffffffu, in ? y : INT_MIN);
        const int lo_z = __reduce_min_sync(0xffffffffu, in ? z : INT_MAX), hi_z = __reduce_max_sync(0xffffffffu, in ? z : INT_MIN);
        const int sx = __reduce_add_sync(0xffffffffu, in ? x : 0), sy = __reduce_add_sync(0xffffffffu, in ? y : 0);
        const int sz = __reduce_add_sync(0xffffffffu, in ? z : 0), sf = __reduce_add_sync(0xffffffffu, in ? faces : 0);
        const int sox = __reduce_add_sync(0xffffffffu, in ? ox : 0), soy = __reduce_add_sync(0xffffffffu, in ? oy : 0);
        const int soz = __reduce_add_sync(0xffffffffu, in ? oz : 0);
        if (lane == __ffs(peers) - 1)
        {
            DsmFrontierAcc &a = acc[cl];
            atomicMin(&a.lo[0], lo_x), atomicMin(&a.lo[1], lo_y), atomicMin(&a.lo[2], lo_z);
            atomicMax(&a.hi[0], hi_x), atomicMax(&a.hi[1], hi_y), atomicMax(&a.hi[2], hi_z);
            acc_add(&a.sum[0], sx), acc_add(&a.sum[1], sy), acc_add(&a.sum[2], sz);
            acc_add(&a.faces, sf);
            acc_add(&a.open[0], sox), acc_add(&a.open[1], soy), acc_add(&a.open[2], soz);
        }
        todo &= ~peers;
    }
}

__global__ void __launch_bounds__(FR_BLOCK) k_frontier_table(const DsmFieldGrid g, const int32_t *__restrict__ roots, const int32_t *__restrict__ slot_comp,
                                                            const int32_t *__restrict__ sizes, const int32_t *__restrict__ offs,
                                                            const DsmFrontierAcc *__restrict__ acc, int max_clusters, int max_voxels,
                                                            dsm_frontier_cluster_t *__restrict__ table, int32_t *hdr)
{
    const int c = blockIdx.x * FR_BLOCK + threadIdx.x;
    if (c >= min(hdr[DSM_FRONTIER_N_CLUSTERS], max_clusters)) return;
    const int n = sizes[c], pre = offs[c];
    const bool listed = (int64_t)pre + n <= (int64_t)max_voxels; // pre <= the frontier count, below 2^30
    if (listed)
    {
        atomicMax(&hdr[DSM_FRONTIER_N_LISTED], pre + n);
        atomicMax(&hdr[DSM_FRONTIER_N_LISTED_CLUSTERS], c + 1);
    }
    const DsmFrontierAcc &a = acc[c];
    dsm_frontier_cluster_t r;
    r.n_voxels = n;
    r.first = roots[slot_comp[c]];
    r.offset = listed ? pre : -1;
    r.reserved = 0;
    r.n_faces = (int64_t)a.faces;
    const double v = (double)g.voxel;
    for (int d = 0; d < 3; d++)
    {
        r.lo[d] = a.lo[d], r.hi[d] = a.hi[d];
        r.open[d] = (int64_t)a.open[d];
        r.centroid[d] = __dmul_rn(__dadd_rn(__ddiv_rn((double)(int64_t)a.sum[d], (double)n), __dadd_rn((double)g.o[d], 0.5)), v);
    }
    table[c] = r;
}

struct FrIsListed
{
    const int32_t *label, *cmap, *hdr;
    __device__ bool operator()(int i) const
    {
        const int k = fr_comp(label, i);
        if (k < 0) return false;
        const int c = cmap[k];
        return c >= 0 && c < hdr[DSM_FRONTIER_N_LISTED_CLUSTERS];
    }
};

// keys of the compacted members (their table slots) and, past them, a key above every slot with index 0
__global__ void __launch_bounds__(FR_BLOCK) k_frontier_keys(const int32_t *__restrict__ label, const int32_t *__restrict__ cmap, int32_t *idx,
                                                           uint32_t *__restrict__ keys, int max_voxels, uint32_t past, const int32_t *hdr)
{
    const int k = blockIdx.x * FR_BLOCK + threadIdx.x;
    if (k >= max_voxels) return;
    if (k < hdr[DSM_FRONTIER_N_SELECTED])
        keys[k] = (uint32_t)cmap[fr_comp(label, idx[k])];
    else
    {
        keys[k] = past;
        idx[k] = 0;
    }
}

// Ordered compaction of the indices i in [0, n) with pred(i): FR_SEL indices per CTA.  k_frontier_sel_count counts each
// CTA's, a cub exclusive scan places the CTAs, and k_frontier_sel_write writes each CTA's in index order (256 at a time:
// ballots and the eight warp totals); the last CTA stores the total into *count.
#define FR_SEL (FR_BLOCK * 8)
template <class P>
__global__ void __launch_bounds__(FR_BLOCK) k_frontier_sel_count(const P pred, int n, int32_t *__restrict__ blk)
{
    int total = 0;
    for (int j = 0; j < FR_SEL / FR_BLOCK; j++)
    {
        const int i = blockIdx.x * FR_SEL + j * FR_BLOCK + threadIdx.x;
        total += __syncthreads_count(i < n && pred(i));
    }
    if (threadIdx.x == 0) blk[blockIdx.x] = total;
}
template <class P>
__global__ void __launch_bounds__(FR_BLOCK) k_frontier_sel_write(const P pred, int n, const int32_t *__restrict__ blk_ofs, int32_t *__restrict__ out,
                                                                int32_t *count)
{
    __shared__ int s_w[FR_BLOCK / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int at = blk_ofs[blockIdx.x];
    for (int j = 0; j < FR_SEL / FR_BLOCK; j++)
    {
        const int i = blockIdx.x * FR_SEL + j * FR_BLOCK + threadIdx.x;
        const bool f = i < n && pred(i);
        const unsigned b = __ballot_sync(0xffffffffu, f);
        if (lane == 0) s_w[warp] = __popc(b);
        __syncthreads();
        int before = 0, total = 0;
        for (int w = 0; w < FR_BLOCK / 32; w++)
        {
            before += w < warp ? s_w[w] : 0;
            total += s_w[w];
        }
        if (f) out[at + before + __popc(b & ((1u << lane) - 1u))] = i;
        at += total;
        __syncthreads();
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) *count = at;
}

static unsigned fr_blocks(int n) { return n > 0 ? (unsigned)((n + FR_BLOCK - 1) / FR_BLOCK) : 1u; }
static int fr_key_bits(int max_clusters) { return 32 - __builtin_clz((unsigned)max_clusters | 1u); } // the key past every slot fits
static int fr_sel_blocks(int voxels) { return (voxels + FR_SEL - 1) / FR_SEL; }
static size_t fr_res_bytes(const DsmFrontier &b) { return b.list_at() + 4 * (size_t)b.max_voxels; }

template <class P>
static cudaError_t fr_select(const DsmFrontier &b, const P &pred, int32_t *out, int32_t *count, cudaStream_t s)
{
    const int nb = fr_sel_blocks(b.voxels);
    k_frontier_sel_count<<<nb, FR_BLOCK, 0, s>>>(pred, b.voxels, b.blk);
    size_t n = b.temp_bytes;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(b.temp, n, b.blk, b.blk_ofs, nb, s);
    if (e != cudaSuccess) return e;
    k_frontier_sel_write<<<nb, FR_BLOCK, 0, s>>>(pred, b.voxels, b.blk_ofs, out, count);
    return cudaGetLastError();
}

// The CUB calls of the job at the sizes fixed at enable (0: the CTA scan of fr_select, 1: the cluster numbering, 2: the
// list offsets, 3: the list's sort); temp == nullptr only sizes the scratch into *bytes.
static cudaError_t fr_cub(const DsmFrontier &b, void *temp, size_t *bytes, cudaStream_t s, int which)
{
    size_t n = temp ? b.temp_bytes : 0;
    cudaError_t e = cudaSuccess;
    switch (which)
    {
    case 0: e = cub::DeviceScan::ExclusiveSum(temp, n, b.blk, b.blk_ofs, fr_sel_blocks(b.voxels), s); break;
    case 1: e = cub::DeviceScan::ExclusiveSum(temp, n, b.cmap, b.cid, b.max_comp, s); break;
    case 2: e = cub::DeviceScan::ExclusiveSum(temp, n, b.sizes, b.offs, b.max_clusters, s); break;
    default:
        e = cub::DeviceRadixSort::SortPairs(temp, n, b.keys, b.keys_alt, b.idx, reinterpret_cast<int32_t *>(b.res + b.list_at()), b.max_voxels,
                                            0, fr_key_bits(b.max_clusters), s);
    }
    if (!temp) *bytes = n;
    return e;
}

// the CUB scratch the job needs for its sizes (the buffers' pointers may still be null); 0 on a CUB error
static size_t fr_temp_bytes(const DsmFrontier &b)
{
    size_t most = 1;
    for (int which = 0; which < 4; which++)
    {
        if (which >= 2 && b.max_clusters == 0) continue;                  // no table
        if (which == 3 && b.max_voxels == 0) continue;                    // no list
        size_t n = 0;
        if (fr_cub(b, nullptr, &n, nullptr, which) != cudaSuccess) return 0;
        most = n > most ? n : most;
    }
    return most;
}

extern "C" int dsm_frontier_enable(dsm_ctx *ctx, int max_clusters, int max_voxels)
{
    if (!ctx) return DSM_E_INVALID;
    const DsmField *f = ctx->field.get();
    if (!f || !ctx->views || ctx->frontier) return DSM_E_STATE;
    for (int n : {max_clusters, max_voxels})
        if (n < 0 || n > DSM_FRONTIER_MAX_CAPACITY) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    auto fr = std::make_unique<DsmFrontier>();
    DsmFrontier &b = *fr;
    const int *n = f->g.n;
    b.voxels = (int)f->voxels;
    // every 2x2x2 block of voxels is 26-connected, so it meets at most one component
    b.max_comp = ((n[0] + 1) / 2) * ((n[1] + 1) / 2) * ((n[2] + 1) / 2);
    b.max_clusters = max_clusters, b.max_voxels = max_voxels;
    const size_t cl = (size_t)std::max(max_clusters, 1), vx = (size_t)std::max(max_voxels, 1);
    const size_t sel = (size_t)fr_sel_blocks(b.voxels);
    const size_t res = fr_res_bytes(b);
    CudaOwner &o = fr->own;
    o.device(&b.label, f->voxels);
    for (int32_t **p : {&b.roots, &b.count, &b.cmap, &b.cid}) o.device(p, (size_t)b.max_comp);
    for (int32_t **p : {&b.slot_comp, &b.sizes, &b.offs}) o.device(p, cl);
    o.device(&b.acc, cl);
    o.device(&b.idx, vx);
    o.device(&b.keys, vx);
    o.device(&b.keys_alt, vx);
    o.device(&b.blk, sel);
    o.device(&b.blk_ofs, sel);
    o.device(&b.res, res);
    o.host(&fr->res_host, res);
    o.event(&fr->ev);
    b.temp_bytes = fr_temp_bytes(b);
    if (b.temp_bytes) o.device(reinterpret_cast<uint8_t **>(&b.temp), b.temp_bytes);
    return keep(ctx->frontier, fr, b.temp_bytes != 0);
}

// Enqueue only: the job on the state grid of the latest (known) field request with that request's origin, one D2H copy
// of the result capacity and the event.  A later field request clears that grid only behind the job, in stream order.
extern "C" int dsm_frontier_enqueue(dsm_ctx *ctx, int min_voxels)
{
    if (!ctx) return DSM_E_INVALID;
    DsmFrontier *fr = ctx->frontier.get();
    const DsmField *f = known_field(ctx);
    if (!fr || !f || fr->in_flight) return DSM_E_STATE;
    if (min_voxels < 1) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    const DsmFrontier &b = *fr;
    const DsmFieldGrid &g = f->g;
    const uint8_t *state = f->occ;
    const cudaStream_t s = ctx->stream;
    int32_t *hdr = reinterpret_cast<int32_t *>(b.res);
    auto *table = reinterpret_cast<dsm_frontier_cluster_t *>(b.res + DsmFrontier::table_at());
    CK(cudaMemsetAsync(b.res, 0, 4 * DSM_FRONTIER_WORDS, s));
    const int rows = g.n[1] * g.n[2];
    k_frontier_mark<<<(unsigned)(rows + FR_ROW_WARPS - 1) / FR_ROW_WARPS, 32 * FR_ROW_WARPS, 0, s>>>(g, state, f->dist + dsm_field_header(f->voxels),
                                                                                                 b.label, hdr);
    const dim3 tiles((g.n[0] + FR_TX - 1) / FR_TX, (g.n[1] + FR_TY - 1) / FR_TY, (g.n[2] + FR_TZ - 1) / FR_TZ);
    k_frontier_tile<<<tiles, FR_TILE, 0, s>>>(g, b.label);
    k_frontier_seam<<<tiles, FR_TILE, 0, s>>>(g, b.label);
    k_frontier_flatten<<<fr_blocks(b.voxels), FR_BLOCK, 0, s>>>(b.label, b.voxels);
    CK(cudaGetLastError());
    CK(fr_select(b, FrIsRoot{b.label}, b.roots, hdr + DSM_FRONTIER_N_COMPONENTS, s));
    k_frontier_number<<<fr_blocks(b.max_comp), FR_BLOCK, 0, s>>>(b.label, b.roots, b.count, hdr);
    k_frontier_count<<<fr_blocks(b.voxels), FR_BLOCK, 0, s>>>(b.label, b.voxels, b.count);
    k_frontier_keep<<<fr_blocks(b.max_comp), FR_BLOCK, 0, s>>>(b.count, b.max_comp, min_voxels, b.cmap, hdr);
    CK(cudaGetLastError());
    CK(fr_cub(b, b.temp, nullptr, s, 1));
    if (b.max_clusters > 0) CK(cudaMemsetAsync(b.sizes, 0, 4 * (size_t)b.max_clusters, s));
    k_frontier_slot<<<fr_blocks(b.max_comp), FR_BLOCK, 0, s>>>(b.count, b.cmap, b.cid, b.max_clusters, b.slot_comp, b.sizes, b.acc, hdr);
    CK(cudaGetLastError());
    if (b.max_clusters > 0)
    {
        k_frontier_reduce<<<fr_blocks(b.voxels), FR_BLOCK, 0, s>>>(g, state, b.label, b.cmap, b.acc);
        CK(cudaGetLastError());
        CK(fr_cub(b, b.temp, nullptr, s, 2));
        k_frontier_table<<<fr_blocks(b.max_clusters), FR_BLOCK, 0, s>>>(g, b.roots, b.slot_comp, b.sizes, b.offs, b.acc, b.max_clusters,
                                                                        b.max_voxels, table, hdr);
        CK(cudaGetLastError());
        if (b.max_voxels > 0)
        {
            CK(fr_select(b, FrIsListed{b.label, b.cmap, hdr}, b.idx, hdr + DSM_FRONTIER_N_SELECTED, s));
            k_frontier_keys<<<fr_blocks(b.max_voxels), FR_BLOCK, 0, s>>>(b.label, b.cmap, b.idx, b.keys, b.max_voxels, (uint32_t)b.max_clusters,
                                                                         hdr);
            CK(cudaGetLastError());
            CK(fr_cub(b, b.temp, nullptr, s, 3));
        }
    }
    return submit(ctx, *fr, b.res, fr_res_bytes(b), f->requests);
}

extern "C" int dsm_frontier_wait(dsm_ctx *ctx, const dsm_frontier_cluster_t **clusters, const int32_t **voxels, dsm_frontier_counts_t *counts)
{
    if (!ctx) return DSM_E_INVALID;
    DsmFrontier *fr = ctx->frontier.get();
    const int rc = wait_head(ctx, fr);
    if (rc != DSM_OK) return rc;
    const int32_t *h = fr->words();
    if (clusters) *clusters = reinterpret_cast<const dsm_frontier_cluster_t *>(fr->res_host + DsmFrontier::table_at());
    if (voxels) *voxels = reinterpret_cast<const int32_t *>(fr->res_host + fr->list_at());
    if (counts) std::memcpy(counts, h, sizeof(dsm_frontier_counts_t));
    return capacity(ctx, h, DSM_FRONTIER_ERR_TAG, "dsm_frontier_wait", "the field the job read");
}
