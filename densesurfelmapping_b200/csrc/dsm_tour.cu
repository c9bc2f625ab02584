// Exploration tour (dsm_tour_*, DESIGN.md §8.14): the order in which to visit n sites, by a deterministic multi-start
// local search for the asymmetric TSP over a travel-cost matrix, all in int64.
//
//   k_tour_search  one CTA of 256 threads per start, the tour in shared memory.  The construction fills one position
//                  per step with a block minimum over packed u64 keys w << 10 | j (42 + 10 bits), taken once for each
//                  candidate up to the one the start draws.  Each pass scans the forward and backward leg weights with
//                  cub::BlockScan (int64, four legs per thread); warps stride over the rows of the neighbourhood (a 2-opt
//                  row per i, an Or-opt row per (L, i)), lanes over j or q, each thread keeping its least (delta, code);
//                  a warp shuffle and a pass over the warps' minima give every thread the pass's move, and the block
//                  applies it through the second tour buffer.  The start's tour and record go to global memory.
//   k_tour_best    one CTA: the least (cost, start), the best tour's order and legs priced P, and the header.
// The matrix is read through the read-only path: at 4 n^2 bytes (4 MB at n = 1024) it stays in L2.  The kernels carry
// no error gate and are launched without PDL, as the field jobs' kernels.  The job's C ABI calls (dsm_tour_enable,
// _enqueue and _wait) follow them; its packed result (D2H) is
//   dsm_tour_info_t | dsm_tour_start_t starts[n_starts] | int32 order[n]
#include "dsm_ctx.hpp"
#include <climits>
#include <cub/block/block_scan.cuh>

#define TOUR_BLOCK 256
#define TOUR_WARPS (TOUR_BLOCK / 32)
#define TOUR_ITEMS (DSM_TOUR_MAX_SITES / TOUR_BLOCK) // the legs each thread scans

static_assert(sizeof(dsm_tour_info_t) == 64 && sizeof(dsm_tour_start_t) == 16, "dsm_tour layouts");
static_assert(DSM_TOUR_MAX_SITES == TOUR_ITEMS * TOUR_BLOCK && DSM_TOUR_MAX_SITES <= 1024, "a site or position fits 10 bits");

typedef cub::BlockScan<long long, TOUR_BLOCK> TourScan;

// w(a, b) of include/dsm.h
struct TourWeight
{
    const uint32_t *M;
    int n, open;
    __device__ __forceinline__ long long operator()(int a, int b) const
    {
        if (a == b || (open && b == 0)) return 0;
        const uint32_t x = __ldg(M + (size_t)a * n + b);
        return x == 0xffffffffu ? DSM_TOUR_P : (long long)x;
    }
};

__device__ __forceinline__ unsigned long long tour_splitmix64(unsigned long long z)
{
    z += 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

// (d, c) becomes the lesser of itself and (od, oc)
__device__ __forceinline__ void tour_take(long long od, uint32_t oc, long long &d, uint32_t &c)
{
    if (od < d || (od == d && oc < c)) d = od, c = oc;
}

// the least (d, c) of the block, in every thread
__device__ __forceinline__ void tour_block_least(long long &d, uint32_t &c, long long *s_d, uint32_t *s_c)
{
    for (int o = 16; o; o >>= 1)
    {
        const long long od = __shfl_xor_sync(0xffffffffu, d, o);
        const uint32_t oc = __shfl_xor_sync(0xffffffffu, c, o);
        tour_take(od, oc, d, c);
    }
    if ((threadIdx.x & 31) == 0) s_d[threadIdx.x >> 5] = d, s_c[threadIdx.x >> 5] = c;
    __syncthreads();
    for (int k = 0; k < TOUR_WARPS; k++) tour_take(s_d[k], s_c[k], d, c);
    __syncthreads(); // s_d and s_c are free again
}

// m, the included sites (0 and every j >= 1 with M[0][j] finite), in every thread; left[j] (if given) flags them
__device__ __forceinline__ int tour_included(const uint32_t *M, int n, uint8_t *left)
{
    int m = 0;
    for (int r = 0; r < TOUR_ITEMS; r++)
    {
        const int j = r * TOUR_BLOCK + threadIdx.x;
        const bool in = j < n && (j == 0 || __ldg(M + j) != 0xffffffffu);
        if (left && j < n) left[j] = in;
        m += __syncthreads_count(in);
    }
    return m;
}

// F[k] and B[k], k in [0, DSM_TOUR_MAX_SITES]: the sums of the forward legs w(t_l, t_{l+1}) and the backward legs
// w(t_{l+1}, t_l) over l < k, with t_m = t_0 = site 0 (legs from position m on weigh 0).  Returns the cost F[m].
__device__ __forceinline__ long long tour_prefix(const TourWeight &w, const int32_t *t, int m, long long *F, long long *B,
                                                 TourScan::TempStorage &tmp)
{
    long long f[TOUR_ITEMS], b[TOUR_ITEMS];
    for (int u = 0; u < TOUR_ITEMS; u++)
    {
        const int k = threadIdx.x * TOUR_ITEMS + u;
        const int x = k < m ? t[k] : 0, y = k + 1 < m ? t[k + 1] : 0;
        f[u] = k < m ? w(x, y) : 0;
        b[u] = k < m ? w(y, x) : 0;
    }
    long long cf, cb;
    TourScan(tmp).ExclusiveSum(f, f, cf);
    __syncthreads();
    TourScan(tmp).ExclusiveSum(b, b, cb);
    for (int u = 0; u < TOUR_ITEMS; u++) F[threadIdx.x * TOUR_ITEMS + u] = f[u], B[threadIdx.x * TOUR_ITEMS + u] = b[u];
    if (threadIdx.x == 0) F[DSM_TOUR_MAX_SITES] = cf, B[DSM_TOUR_MAX_SITES] = cb;
    __syncthreads();
    return cf;
}

__global__ void __launch_bounds__(TOUR_BLOCK) k_tour_search(const uint32_t *__restrict__ M, int n, int open, int max_passes,
                                                            unsigned long long seed, int32_t *__restrict__ tours,
                                                            dsm_tour_start_t *__restrict__ starts)
{
    __shared__ int32_t s_t[2][DSM_TOUR_MAX_SITES];
    __shared__ long long s_F[DSM_TOUR_MAX_SITES + 1], s_B[DSM_TOUR_MAX_SITES + 1];
    __shared__ uint8_t s_left[DSM_TOUR_MAX_SITES];
    __shared__ TourScan::TempStorage s_scan;
    __shared__ long long s_d[TOUR_WARPS];
    __shared__ uint32_t s_c[TOUR_WARPS];
    const TourWeight w{M, n, open};
    const int s = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int m = tour_included(M, n, s_left); // s_left[j]: j is included and not yet in the tour
    if (tid == 0) s_left[0] = 0, s_t[0][0] = 0;
    __syncthreads();

    // construction: position k takes candidate `pick` of the c least keys w(t_{k-1}, j) << 10 | j (keys >= 1: j >= 1)
    for (int k = 1; k < m; k++)
    {
        const int prev = s_t[0][k - 1], c = min(3, m - k);
        const int pick = s == 0 ? 0 : (int)(tour_splitmix64(seed ^ ((unsigned long long)s << 32) ^ (unsigned long long)k) % (unsigned)c);
        unsigned long long lo = 0;
        for (int r = 0; r <= pick; r++)
        {
            long long best = LLONG_MAX;
            for (int j = tid; j < n; j += TOUR_BLOCK)
                if (s_left[j])
                {
                    const long long key = w(prev, j) << 10 | j;
                    if ((unsigned long long)key > lo && key < best) best = key;
                }
            uint32_t unused = 0;
            tour_block_least(best, unused, s_d, s_c);
            lo = (unsigned long long)best;
        }
        if (tid == 0) s_t[0][k] = (int)(lo & 1023), s_left[lo & 1023] = 0;
        __syncthreads();
    }

    // passes: rows 0..r2-1 are 2-opt rows i = r + 1; then m - L Or-opt rows i = 1..m-L for each L = 1, 2, 3
    int cur = 0, passes = 0, converged = 0;
    const int r2 = max(m - 2, 0), rows = r2 + max(m - 1, 0) + max(m - 2, 0) + max(m - 3, 0);
    for (int p = 0; p < max_passes; p++)
    {
        const int32_t *t = s_t[cur];
        tour_prefix(w, t, m, s_F, s_B, s_scan);
        long long bd = 0;
        uint32_t bc = 0xffffffffu;
        for (int r = warp; r < rows; r += TOUR_WARPS)
            if (r < r2)
            {
                // reverse [i, j]: w(t_{i-1}, t_j) + w(t_i, t_{j+1}) - f_{i-1} - f_j + (B_j - B_i) - (F_j - F_i)
                const int i = r + 1, a = t[i - 1], b = t[i];
                const long long base = s_F[i - 1] - s_B[i];
                for (int j = i + 1 + lane; j < m; j += 32)
                {
                    const int tj = t[j], tj1 = j + 1 < m ? t[j + 1] : 0;
                    const long long d = base + w(a, tj) + w(b, tj1) - (s_F[j + 1] - s_F[j]) + s_B[j] - s_F[j];
                    tour_take(d, (uint32_t)(i << 12 | j), bd, bc);
                }
            }
            else
            {
                // move [i, e] after q: w(t_{i-1}, t_{e+1}) + w(t_q, t_i) + w(t_e, t_{q+1}) - f_{i-1} - f_e - f_q
                int i = r - r2, L = 1;
                while (i >= m - L) i -= m - L, L++;
                i += 1;
                const int e = i + L - 1, a = t[i - 1], b = t[i], c = t[e], d1 = e + 1 < m ? t[e + 1] : 0;
                const long long base = w(a, d1) - (s_F[i] - s_F[i - 1]) - (s_F[e + 1] - s_F[e]);
                for (int q = lane; q < m; q += 32)
                {
                    if (q >= i - 1 && q <= e) continue;
                    const int tq = t[q], tq1 = q + 1 < m ? t[q + 1] : 0;
                    const long long d = base + w(tq, b) + w(c, tq1) - (s_F[q + 1] - s_F[q]);
                    tour_take(d, (uint32_t)(1u << 22 | i << 12 | L << 10 | q), bd, bc);
                }
            }
        tour_block_least(bd, bc, s_d, s_c);
        if (bd >= 0)
        {
            converged = 1;
            break;
        }
        const int i = bc >> 12 & 1023, x = bc & 1023, L = bc >> 10 & 3;
        int32_t *nt = s_t[cur ^ 1];
        for (int q = tid; q < m; q += TOUR_BLOCK)
        {
            int src = q;
            if (!(bc >> 22))
                src = q >= i && q <= x ? i + x - q : q;
            else if (x < i)
                src = q > x && q <= x + L ? i + (q - x - 1) : q > x + L && q < i + L ? q - L : q;
            else
                src = q >= i && q <= x - L ? q + L : q > x - L && q <= x ? i + (q - (x - L + 1)) : q;
            nt[q] = t[src];
        }
        __syncthreads();
        cur ^= 1;
        passes++;
    }
    const long long C = tour_prefix(w, s_t[cur], m, s_F, s_B, s_scan);
    for (int q = tid; q < m; q += TOUR_BLOCK) tours[(size_t)s * n + q] = s_t[cur][q];
    if (tid == 0)
    {
        dsm_tour_start_t r;
        r.cost = C;
        r.passes = passes;
        r.converged = converged;
        starts[s] = r;
    }
}

__global__ void __launch_bounds__(TOUR_BLOCK) k_tour_best(const uint32_t *__restrict__ M, int n, int open, int n_starts, int max_passes,
                                                          unsigned long long seed, const int32_t *__restrict__ tours, uint8_t *__restrict__ res)
{
    __shared__ long long s_d[TOUR_WARPS];
    __shared__ uint32_t s_c[TOUR_WARPS];
    const TourWeight w{M, n, open};
    const auto *starts = reinterpret_cast<const dsm_tour_start_t *>(res + 64);
    int32_t *order = reinterpret_cast<int32_t *>(res + 64 + 16 * (size_t)n_starts);
    long long C = LLONG_MAX;
    uint32_t best = 0xffffffffu;
    for (int s = threadIdx.x; s < n_starts; s += TOUR_BLOCK) tour_take(starts[s].cost, (uint32_t)s, C, best);
    tour_block_least(C, best, s_d, s_c);
    const int m = tour_included(M, n, nullptr);
    const int32_t *t = tours + (size_t)best * n;
    int n_inf = 0;
    for (int r = 0; r < TOUR_ITEMS; r++)
    {
        const int k = r * TOUR_BLOCK + threadIdx.x;
        n_inf += __syncthreads_count(k < m && w(t[k], k + 1 < m ? t[k + 1] : 0) == DSM_TOUR_P);
        if (k < n) order[k] = k < m ? t[k] : -1;
    }
    if (threadIdx.x == 0)
    {
        dsm_tour_info_t h;
        memset(&h, 0, sizeof(h));
        h.n_sites = n, h.n_included = m, h.open = open, h.n_starts = n_starts, h.max_passes = max_passes;
        h.best_start = (int32_t)best, h.best_cost = C, h.seed = seed, h.n_infinite = n_inf;
        *reinterpret_cast<dsm_tour_info_t *>(res) = h;
    }
}

// byte offsets of the result's order and its end
static size_t tour_order_at(int n_starts) { return sizeof(dsm_tour_info_t) + sizeof(dsm_tour_start_t) * (size_t)n_starts; }
static size_t tour_res_bytes(int n_starts, int n) { return tour_order_at(n_starts) + 4 * (size_t)n; }

extern "C" int dsm_tour_enable(dsm_ctx *ctx, int max_sites, int max_starts)
{
    if (!ctx) return DSM_E_INVALID;
    if (ctx->tour) return DSM_E_STATE;
    if (max_sites < 1 || max_sites > DSM_TOUR_MAX_SITES || max_starts < 1 || max_starts > DSM_TOUR_MAX_STARTS) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    auto tr = std::make_unique<DsmTour>();
    tr->max_sites = max_sites, tr->max_starts = max_starts;
    const size_t entries = (size_t)max_sites * max_sites, res = tour_res_bytes(max_starts, max_sites);
    CudaOwner &o = tr->own;
    o.host(&tr->matrix_host, entries);
    o.device(&tr->matrix, entries);
    o.device(&tr->tours, (size_t)max_starts * max_sites);
    o.device(&tr->res, res);
    o.host(&tr->res_host, res);
    o.event(&tr->ev);
    return keep(ctx->tour, tr);
}

// Enqueue only: the matrix staged and copied, the kernels, one D2H copy of the used result and the event.
extern "C" int dsm_tour_enqueue(dsm_ctx *ctx, const uint32_t *matrix, int n, int open, int n_starts, int max_passes, uint64_t seed)
{
    if (!ctx) return DSM_E_INVALID;
    DsmTour *tr = ctx->tour.get();
    if (!tr || tr->in_flight) return DSM_E_STATE;
    if (!matrix || n < 1 || n > tr->max_sites || n_starts < 1 || n_starts > tr->max_starts || (open != 0 && open != 1) ||
        max_passes < 0 || max_passes > DSM_TOUR_MAX_PASSES ||
        (unsigned long long)n_starts * (unsigned long long)max_passes * (unsigned long long)n * (unsigned long long)n > DSM_TOUR_MAX_WORK)
        return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    // the previous job's copy out of this staging ended before its wait, which no job in flight implies
    const size_t bytes = 4 * (size_t)n * n;
    std::memcpy(tr->matrix_host, matrix, bytes);
    CK(cudaMemcpyAsync(tr->matrix, tr->matrix_host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    k_tour_search<<<n_starts, TOUR_BLOCK, 0, ctx->stream>>>(tr->matrix, n, open, max_passes, seed, tr->tours,
                                                            reinterpret_cast<dsm_tour_start_t *>(tr->res + sizeof(dsm_tour_info_t)));
    k_tour_best<<<1, TOUR_BLOCK, 0, ctx->stream>>>(tr->matrix, n, open, n_starts, max_passes, seed, tr->tours, tr->res);
    CK(cudaGetLastError());
    tr->n = n, tr->n_starts = n_starts;
    return submit(ctx, *tr, tr->res, tour_res_bytes(n_starts, n), 0);
}

extern "C" int dsm_tour_wait(dsm_ctx *ctx, dsm_tour_info_t *info, const dsm_tour_start_t **starts, const int32_t **order)
{
    if (!ctx) return DSM_E_INVALID;
    DsmTour *tr = ctx->tour.get();
    const int rc = wait_head(ctx, tr);
    if (rc != DSM_OK) return rc;
    if (info) std::memcpy(info, tr->res_host, sizeof(dsm_tour_info_t));
    if (starts) *starts = reinterpret_cast<const dsm_tour_start_t *>(tr->res_host + sizeof(dsm_tour_info_t));
    if (order) *order = reinterpret_cast<const int32_t *>(tr->res_host + tour_order_at(tr->n_starts));
    return DSM_OK;
}
