// Hand-written sm_90a kernels for the DenseSurfelMapping per-frame hot path: input repack, seed initialisation,
// surfel fuse / initialise and the GPU-resident pool kernels.  The superpixel and plane-fit kernels live in dsm_tile.cu.
//
// Every kernel takes the frame index from the grid so a batch of independent frames is one launch.  No tensor cores:
// there is no dense contraction anywhere on this path (largest "matrix" is a 4x4 fp64 solve per superpixel).
//
// EXACTNESS CONTRACT (SURVEY.md §7 H1-H4): superpixel labels must be bit-identical to the
// serialised reference.  Therefore this file is compiled with -fmad=false (the reference is
// built for baseline x86-64: SSE2, no FMA contraction), keeps IEEE division / sqrt
// (-prec-div/-prec-sqrt defaults, no fast-math, no FTZ) and spells out every float<->double
// promotion exactly where the reference's C++ expressions have them.  All citations
// ":NNN" refer to the reference's surfel_fusion/src/fusion_functions.cpp.
#include "dsm_exact.cuh"
#include <cuda_pipeline.h>
#include <climits>
#include <type_traits>

// -------------------------------------------------------------------------------------------
// Kin  repack — the caller's tightly packed [n][H][W] gray / depth arrive by ONE contiguous H2D copy
// each (a strided 2-D copy of 1226-byte rows runs at less than half the PCIe rate) and are laid
// out here into the 16-byte-aligned pitched device format every other kernel relies on.
// One thread per 4 output pixels; reads are unaligned scalars (coalesced), writes are vectors.
// -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_repack(const __grid_constant__ DsmDev d, const uint8_t *gray_packed, const float *depth_packed)
{
    const int b = d.frame0 + blockIdx.z; // device frame slot; the packed source holds this chunk's frames from 0
    const int x4 = (blockIdx.x * 64 + threadIdx.x) * 4;
    const int y = blockIdx.y * 4 + threadIdx.y;
    if (x4 >= d.Wp || y >= d.H) return;
    const size_t src = ((size_t)blockIdx.z * d.H + y) * d.W + x4;
    const size_t dst = (size_t)b * d.px_stride + (size_t)y * d.Wp + x4;
    uchar4 g = make_uchar4(0, 0, 0, 0);
    float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    if (x4 + 3 < d.W)
    {
        g = make_uchar4(gray_packed[src], gray_packed[src + 1], gray_packed[src + 2], gray_packed[src + 3]);
        z = make_float4(depth_packed[src], depth_packed[src + 1], depth_packed[src + 2], depth_packed[src + 3]);
    }
    else
    {
        if (x4 < d.W) g.x = gray_packed[src], z.x = depth_packed[src];
        if (x4 + 1 < d.W) g.y = gray_packed[src + 1], z.y = depth_packed[src + 1];
        if (x4 + 2 < d.W) g.z = gray_packed[src + 2], z.z = depth_packed[src + 2];
    }
    *reinterpret_cast<uchar4 *>(const_cast<uint8_t *>(d.gray) + dst) = g;
    *reinterpret_cast<float4 *>(const_cast<float *>(d.depth) + dst) = z;
}

// -------------------------------------------------------------------------------------------
// K0  seed_init   — initialize_seeds_kernel (:577-629) + the per-frame clears (:963-965)
// one thread per seed
// -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_seed_init(const __grid_constant__ DsmDev d)
{
    pdl_enter();
    const int b = d.frame0 + blockIdx.y;
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    if (blockIdx.x == 0 && threadIdx.x == 0)
    {
        d.nlist[b] = 0;
        d.nnew[b] = 0;
        d.errflag[b] = 0;
        d.done[b] = 0;
    }
    const int W = d.W, H = d.H, Wp = d.Wp;
    const uint8_t *gray = d.gray + (size_t)b * d.px_stride;
    const float *depth = d.depth + (size_t)b * d.px_stride;
    const bool live = s < d.S;
    const int sp_x = live ? s % d.spw : 0, sp_y = live ? s / d.spw : 0;
    int ix = sp_x * DSM_SP + DSM_SP / 2, iy = sp_y * DSM_SP + DSM_SP / 2;
    ix = ix < W - 1 ? ix : W - 1;
    iy = iy < H - 1 ? iy : H - 1;
    float md = live ? depth[iy * Wp + ix] : 1.0f;
    // seeds sitting on a hole: first depth > 0.01 in raster order of the clamped END-EXCLUSIVE window
    // (:602-625).  The warp serves its hole seeds one at a time, 32 window pixels per step.
    unsigned todo = __ballot_sync(FULL, live && (double)md < 0.01);
    while (todo)
    {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const int hx = __shfl_sync(FULL, sp_x, src), hy = __shfl_sync(FULL, sp_y, src);
        int xb = hx * DSM_SP + DSM_SP / 2 - DSM_SP, yb = hy * DSM_SP + DSM_SP / 2 - DSM_SP;
        int xe = xb + DSM_SP * 2, ye = yb + DSM_SP * 2;
        xb = xb > 0 ? xb : 0;
        yb = yb > 0 ? yb : 0;
        xe = xe < W - 1 ? xe : W - 1;
        ye = ye < H - 1 ? ye : H - 1;
        const int ww = xe - xb, n = ww * (ye - yb);
        float found = 0.f;
        bool got = false;
        for (int base = 0; base < n && !got; base += 32)
        {
            const int i = base + lane;
            float t = 0.f;
            if (i < n) t = depth[(yb + i / ww) * Wp + xb + i % ww];
            const unsigned hit = __ballot_sync(FULL, (double)t > 0.01);
            if (hit)
            {
                found = __shfl_sync(FULL, t, __ffs(hit) - 1);
                got = true;
            }
        }
        if (got && lane == src) md = found;
    }
    if (!live) return;
    const size_t o = (size_t)b * d.S + s;
    store_seed(d, o, (float)ix, (float)iy, (float)gray[iy * Wp + ix], md, false); // stable = false
    d.fused[o] = 0;                                                                 // fused = false
}

// -------------------------------------------------------------------------------------------
// Staging of a contiguous run of 44-byte surfel records through shared memory for the streaming pool
// kernels (k_fuse, k_pool_transform).  When the run is 16-byte aligned and a multiple of 16 bytes it
// moves as ONE TMA 1-D bulk copy each way (cp.async.bulk: UBLKCP in SASS, completion on an mbarrier for
// the load, a bulk async-group for the store) issued by a single thread -- no per-thread address math,
// no register staging; otherwise (unaligned slice start, ragged tail) coalesced 4-byte accesses.
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ bool stage_in(float *sm, const float *g, int cnt, uint64_t *bar, int nthreads)
{
    const unsigned bytes = (unsigned)cnt * 44u;
    const bool bulk = (bytes % 16u == 0u) && ((reinterpret_cast<uintptr_t>(g) & 15u) == 0u);
    if (bulk)
    {
        const unsigned b = smem_u32(bar);
        if (threadIdx.x == 0)
        {
            mbar_init(b, 1);
            mbar_expect_tx(b, bytes);
            bulk_load(smem_u32(sm), g, bytes, b);
        }
        __syncthreads(); // barrier initialised before anybody polls it
        mbar_wait(b, 0);
    }
    else
    {
        for (int i = threadIdx.x; i < cnt * 11; i += nthreads) sm[i] = g[i];
        __syncthreads();
    }
    return bulk;
}

__device__ __forceinline__ void stage_out(float *g, const float *sm, int cnt, bool bulk, int nthreads)
{
    if (bulk)
    {
        fence_proxy_async_smem();
        __syncthreads();
        if (threadIdx.x == 0) bulk_store(g, smem_u32(sm), (unsigned)cnt * 44u);
    }
    else
    {
        __syncthreads();
        for (int i = threadIdx.x; i < cnt * 11; i += nthreads) g[i] = sm[i];
    }
}

// A resident view whose error word is set (a frame of dsm_fuse_stream_window was rejected): the pool stays as it is.
// Read after pdl_enter, i.e. after the kernel that may have set it has completed.
__device__ __forceinline__ bool gated(const DsmDev &d) { return d.gate && *(volatile const int32_t *)d.gate != 0; }

// -------------------------------------------------------------------------------------------
// K5  surfel_fuse — fuse_surfels_kernel (:190-313).  Pure map over the frame's pool slice.
// The AoS pool (44 B/element, ABI layout) is staged through shared memory with fully coalesced
// 4-byte accesses; each thread then works on its element at stride 11 words (conflict-free).
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ void mat4_mul(const float *m, float x, float y, float z, float w, float *o)
{ // column-major, column-by-column accumulation (matches the oracle's Eigen stand-in)
#pragma unroll
    for (int i = 0; i < 4; i++) o[i] = ((m[i] * x + m[4 + i] * y) + m[8 + i] * z) + m[12 + i] * w;
}
__device__ __forceinline__ void mat3_mul(const float *m, float x, float y, float z, float *o)
{
#pragma unroll
    for (int i = 0; i < 3; i++) o[i] = (m[i] * x + m[4 + i] * y) + m[8 + i] * z;
}
__device__ __forceinline__ float get_weight(float depth)
{ // std::min(1.0 / depth / depth, 1.0) (:99-102); std::min(a,b) = (b < a) ? b : a
    const double w = 1.0 / (double)depth / (double)depth;
    return (float)((1.0 < w) ? 1.0 : w);
}

#define FUSE_BLOCK 256
__global__ void __launch_bounds__(FUSE_BLOCK) k_fuse(const __grid_constant__ DsmDev d)
{
    pdl_enter();
    if (gated(d)) return;
    __shared__ alignas(128) float sm[FUSE_BLOCK * 11];
    __shared__ float s_pose[32];
    __shared__ uint64_t bar;
    const int b = d.frame0 + blockIdx.y;
    const int begin = d.poolofs[b], end = d.poolofs[b + 1];
    const int first = begin + blockIdx.x * FUSE_BLOCK;
    if (first >= end) return;
    const int cnt = min(FUSE_BLOCK, end - first);
    float *g = reinterpret_cast<float *>(d.pool + first);
    if (threadIdx.x < 16) s_pose[threadIdx.x] = d.pose[b * 16 + threadIdx.x];
    else if (threadIdx.x < 32) s_pose[threadIdx.x] = d.ipose[b * 16 + threadIdx.x - 16];
    const bool bulk = stage_in(sm, g, cnt, &bar, FUSE_BLOCK);
    __syncthreads(); // s_pose
    if (threadIdx.x < cnt)
    {
        float *e = sm + threadIdx.x * 11;
        const float *pose = s_pose, *inv_pose = s_pose + 16;
        const int ref = d.refidx[b];
        const int W = d.W, H = d.H, Wp = d.Wp;
        const size_t fo = (size_t)b * d.px_stride, so = (size_t)b * d.S;
        int update_times = __float_as_int(e[9]);
        const int last_update = __float_as_int(e[10]);
        do
        {
            if (ref - last_update > 5 && update_times < 5)
            { // remove unstable (:207-211)
                e[9] = __int_as_float(0);
                break;
            }
            if (update_times == 0) break;
            float pc[4];
            mat4_mul(inv_pose, e[0], e[1], e[2], 1.0f, pc);
            if (pc[2] < d.fuse_near || pc[2] > d.fuse_far) break;
            float nc[3];
            mat3_mul(inv_pose, e[3], e[4], e[5], nc);
            const float pu = pc[0] * d.fx / pc[2] + d.cx;
            const float pv = pc[1] * d.fy / pc[2] + d.cy;
            const int ui = (int)((double)pu + 0.5), vi = (int)((double)pv + 0.5);
            if (ui < 1 || ui > W - 2 || vi < 1 || vi > H - 2) break;
            if ((double)pc[2] < (double)d.depth[fo + (size_t)vi * Wp + ui] - 1.0)
            { // occluding the measurement (:239-243)
                e[9] = __int_as_float(0);
                break;
            }
            const int sp = dsm_code_seed(d.code[fo + (size_t)vi * Wp + ui], ui, vi, d.spw);
            const float4 *pl = d.plane + (so + sp) * 3;
            const float4 r0 = pl[0]; // n, view_cos
            if (r0.x == 0 && r0.y == 0 && r0.z == 0) break;
            if ((double)r0.w < MAX_ANGLE_COS) break;
            const float4 r1 = pl[1]; // posi, mean_depth
            const float4 r2 = pl[2]; // size, I
            float tol = (float)((double)(pc[2] * pc[2]) / (d.baseline * (double)d.camera_f) * d.disparity_error);
            tol = (double)tol < d.min_tolerate_diff ? (float)d.min_tolerate_diff : tol;
            if (pc[2] < r1.w - tol) break;
            if (pc[2] > r1.w + tol) break;
            const float ndc = nc[0] * r0.x + nc[1] * r0.y + nc[2] * r0.z;
            if ((double)ndc < MAX_ANGLE_COS)
            {
                e[9] = __int_as_float(0);
                break;
            }
            const float ow = e[8];
            const float nw = get_weight(r1.w);
            const float sw = ow + nw;
            float pw[4];
            mat4_mul(pose, r1.x, r1.y, r1.z, 1.0f, pw);
            const float fpx = (e[0] * ow + nw * pw[0]) / sw;
            const float fpy = (e[1] * ow + nw * pw[1]) / sw;
            const float fpz = (e[2] * ow + nw * pw[2]) / sw;
            float fnx = nc[0] * ow + nw * r0.x;
            float fny = nc[1] * ow + nw * r0.y;
            float fnz = nc[2] * ow + nw * r0.z;
            const double nl = (double)sqrtf(fnx * fnx + fny * fny + fnz * fnz);
            fnx = (float)((double)fnx / nl);
            fny = (float)((double)fny / nl);
            fnz = (float)((double)fnz / nl);
            float nwd[3];
            mat3_mul(pose, fnx, fny, fnz, nwd);
            e[0] = fpx, e[1] = fpy, e[2] = fpz;
            e[3] = nwd[0], e[4] = nwd[1], e[5] = nwd[2];
            e[8] = sw;
            e[7] = r2.y;
            const float new_size = (float)((double)r2.x * fabs((double)(r1.w / (d.camera_f * r0.w))));
            if (new_size < e[6]) e[6] = new_size;
            e[10] = __int_as_float(ref);
            e[9] = __int_as_float(update_times + 1);
            d.fused[so + sp] = 1; // idempotent multi-writer store (:311)
        } while (0);
    }
    stage_out(g, sm, cnt, bulk, FUSE_BLOCK);
}

// Block rank (ballot -> per-warp count -> prefix over the warps): the position of this thread among the CTA's threads
// with `live` set, in thread order.  s_warp (shared, one int per warp) holds every warp's count when it returns.
__device__ __forceinline__ int block_rank(bool live, int *s_warp)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned bal = __ballot_sync(FULL, live);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int pos = 0;
    for (int w = 0; w < warp; w++) pos += s_warp[w];
    return pos + __popc(bal & ((1u << lane) - 1));
}

// -------------------------------------------------------------------------------------------
// K6  surfel_init — initialize_surfels (:315-361).  new_surfels come out in seed-index order exactly like the
// reference's serial push_back loop, with several CTAs per frame and no inter-CTA communication: CTA j owns
// seeds [1024 j, 1024 j + 1024) and finds its output offset without any inter-CTA communication by re-evaluating
// the cheap emit predicate over the seeds before its range (<= 36 B per seed, L2-resident), then scans its own
// range.  Same predicate, same per-surfel arithmetic, same order: byte-identical output.
__device__ __forceinline__ bool init_emits(const DsmDev &d, size_t so, int s)
{
    const float4 *pl = d.plane + (so + s) * 3;
    const float4 r0 = pl[0];
    const float md = pl[1].w;
    return !(md == 0) && !d.fused[so + s] && !((double)r0.w < MAX_ANGLE_COS) && !(r0.x == 0 && r0.y == 0 && r0.z == 0);
}
__global__ void __launch_bounds__(1024) k_init_surfels(const __grid_constant__ DsmDev d)
{
    pdl_enter();
    if (gated(d)) return;
    __shared__ int s_warp[32];
    __shared__ int s_before[32];
    __shared__ float s_pose[16];
    const int b = d.frame0 + blockIdx.y;
    const size_t so = (size_t)b * d.S;
    if (threadIdx.x < 16) s_pose[threadIdx.x] = d.pose[b * 16 + threadIdx.x];
    const int first = blockIdx.x * 1024;
    // emitted surfels before this CTA's range
    int before = 0;
    for (int s = threadIdx.x; s < first; s += 1024) before += init_emits(d, so, s) ? 1 : 0;
    before = __reduce_add_sync(FULL, before);
    const int s = first + threadIdx.x;
    const bool e = s < d.S && init_emits(d, so, s);
    if ((threadIdx.x & 31) == 0) s_before[threadIdx.x >> 5] = before; // read after block_rank's barrier
    int pos = block_rank(e, s_warp), total = 0;
    for (int w = 0; w < 32; w++)
    {
        pos += s_before[w];
        total += s_before[w] + s_warp[w];
    }
    if (e)
    {
        const float4 *pl = d.plane + (so + s) * 3;
        const float4 r0 = pl[0], r1 = pl[1], r2 = pl[2];
        float pw[4], nw[3];
        mat4_mul(s_pose, r1.x, r1.y, r1.z, 1.0f, pw);
        mat3_mul(s_pose, r0.x, r0.y, r0.z, nw);
        dsm_surfel_t o;
        o.px = pw[0], o.py = pw[1], o.pz = pw[2];
        o.nx = nw[0], o.ny = nw[1], o.nz = nw[2];
        o.size = (float)((double)r2.x * fabs((double)(r1.w / (d.camera_f * r0.w))));
        o.color = r2.y;
        o.weight = get_weight(r1.w);
        o.update_times = 1;
        o.last_update = d.refidx[b];
        d.newsurf[so + pos] = o;
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) d.nnew[b] = total;
}

// -------------------------------------------------------------------------------------------
// GPU-resident pool (SURVEY.md §8f rows 1-2): what SurfelMap does to `local_surfels` between and
// after the hot-path calls, kept on the device so a stream never round-trips its pool.
//
// k_pool_count / k_pool_scan / k_pool_scatter — ordered selection over a pool range (retire, exports, and the hole list of
//   the post-step below).
// k_pool_recycle — the post-fusion step of SurfelMap::fuse_map (surfel_map.cpp:1077-1109) in place, slot for slot: new
//   surfels fill the dead slots from the highest index down, the rest are appended; leftover holes are filled from the
//   back (see the kernel).
// k_pool_transform — warp_active_surfels_cpu_kernel (surfel_map.cpp:750-789): p <- W p, n <- R_W n
//   for every surfel of the pool after a loop closure.  Pure streaming over the 44-byte records,
//   staged through shared memory like k_fuse.
// -------------------------------------------------------------------------------------------
// selection predicate of the pool kernels: mode 0 = dead slots (update_times == 0, fuse_map post-step, surfel_map.cpp:1081);
// mode 1 = live surfels last updated by keyframe `key` (move_add_surfels, surfel_map.cpp:1479-1497);
// mode 2 = surfels with update_times >= key (the publish/save filters, surfel_map.cpp:1158, :1243, :1406, :1429)
__device__ __forceinline__ bool pool_pred(const dsm_surfel_t &e, int mode, int key)
{
    if (mode == 2) return e.update_times >= key;
    return mode == 0 ? (e.update_times == 0) : (e.update_times > 0 && e.last_update == key);
}

__global__ void __launch_bounds__(256) k_pool_count(const __grid_constant__ DsmDev d, int b, int *blkcnt, int mode, int key)
{
    pdl_enter();
    if (gated(d)) return;
    const int begin = d.poolofs[b], end = d.poolofs[b + 1];
    const int i = begin + blockIdx.x * 256 + threadIdx.x;
    const bool live = i < end && pool_pred(d.pool[i], mode, key);
    const int c = __syncthreads_count(live);
    if (threadIdx.x == 0) blkcnt[blockIdx.x] = (begin + blockIdx.x * 256 < end) ? c : 0;
}

__global__ void __launch_bounds__(1024) k_pool_scan(const __grid_constant__ DsmDev d, int b, const int *blkcnt, int *blkofs, int *nsel)
{
    pdl_enter();
    if (gated(d)) return;
    __shared__ int s_warp[32];
    __shared__ int s_run;
    const int begin = d.poolofs[b], end = d.poolofs[b + 1];
    const int nblk = (end - begin + 255) / 256;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_run = 0;
    __syncthreads();
    for (int base = 0; base < nblk; base += 1024)
    {
        const int i = base + threadIdx.x;
        const int v = i < nblk ? blkcnt[i] : 0;
        int wtot;
        const int wex = warp_excl_scan(v, lane, wtot);
        if (lane == 31) s_warp[warp] = wtot;
        __syncthreads();
        const int run = s_run;
        int wofs = 0, tot = 0;
        for (int w = 0; w < 32; w++)
        {
            const int c = s_warp[w];
            if (w < warp) wofs += c;
            tot += c;
        }
        if (i < nblk) blkofs[i] = run + wofs + wex;
        __syncthreads();
        if (threadIdx.x == 0) s_run = run + tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) *nsel = s_run; // selected surfels in the range
}

// The selected surfels of the CTA's 256 pool entries, in pool order, to dst + blkofs[CTA].  Rec is the output record:
// the whole 44-byte surfel (retire, surfel export), its pool index (the hole list of k_pool_recycle) or, for the
// point-cloud builders of SurfelMap (publish_active_pointcloud surfel_map.cpp:1398-1417, publish_all_pointcloud :1419-1454,
// publish_neighbor_pointcloud :1284-1300, save_cloud :1153-1173), one PointXYZI float4 {px, py, pz, intensity = color}
// like the serial push_back loops.
template <typename Rec>
__global__ void __launch_bounds__(256) k_pool_scatter(const __grid_constant__ DsmDev d, int b, const int *blkofs, Rec *dst, int mode, int key)
{
    pdl_enter();
    if (gated(d)) return;
    __shared__ int s_warp[8];
    const int begin = d.poolofs[b], end = d.poolofs[b + 1];
    const int i = begin + blockIdx.x * 256 + threadIdx.x;
    if (begin + blockIdx.x * 256 >= end) return;
    dsm_surfel_t e;
    bool live = false;
    if (i < end)
    {
        e = d.pool[i];
        live = pool_pred(e, mode, key);
        if (live && mode == 1) d.pool[i].update_times = 0; // "delete the surfel from the local point" (surfel_map.cpp:1496)
    }
    const int rank = block_rank(live, s_warp);
    if (!live) return;
    const int pos = blkofs[blockIdx.x] + rank;
    if constexpr (std::is_same<Rec, float4>::value)
        dst[pos] = make_float4(e.px, e.py, e.pz, e.color);
    else if constexpr (std::is_same<Rec, int32_t>::value)
        dst[pos] = i;
    else
        dst[pos] = e;
}

// -------------------------------------------------------------------------------------------
// k_pool_recycle — the post-step of SurfelMap::fuse_map (surfel_map.cpp:1077-1109) on the resident pool [0, N), in place.
// The reference, with D = d_0 < ... < d_{m-1} the slots with update_times == 0 and K new surfels:
//   for k < K:  if D is not empty: local[D.back()] = new[k], D.pop_back()   else push_back(new[k])
//   while D is not empty: local[D.back()] = local.back(), D.pop_back(), local.pop_back()
// so the new size is N' = N - m + K and
//   fill:  new[k] -> slot d_{m-1-k} for k < min(K, m); new[k] -> slot N + k - m for k >= m (then there is no tail).
//   tail:  (K < m) the q = m - K lowest holes d_0..d_{q-1} remain.  Iteration j of the while loop reads the back,
//          position N-1-j, and writes hole d_{q-1-j}: hole d_t reads position N' + t ("tail offset" t, t < q).  A hole d_t
//          >= N' lies inside the tail and is popped later; one below N' is a final slot.  What tail offset t holds when
//          it is read: position N'+t itself if it was occupied after the fill (a live surfel, or new[m-1-i] when it is
//          the filled hole d_i, i >= q); otherwise N'+t is a leftover hole d_s, which an earlier iteration wrote with
//          what tail offset s held (s > t: that iteration read position N'+s = p + u(p), u(p) = occupied positions in
//          (p, N) = (N-1-p) - (q-1-s) >= 0, and s == t only for a hole that is the back when it is read, whose own read
//          no final slot ever follows).
// So src(t) = t's own surfel if occupied, else src(s): pointer chains over the tail that only go up, of any length up to
// q.  They are resolved by pointer doubling in shared memory within segments of RC_SEG tail offsets, and across segments
// by taking the segments from the top down: a CTA draws a ticket (atomic) for each segment it takes, so every segment
// above it belongs to a CTA that is already running; it waits for the completion flags of the segments its remaining
// pointers leave to and reads their resolved sources.  No CTA waits for one that may not have started: no co-residency assumption.
// Every destination (fill, final slot) lies below N' or at an append slot >= N, every source at or above N' (or in
// newsurf): nothing is read after another thread of the grid wrote it.  The last CTA to finish stores N' in ofs_out[1]
// (every CTA has read N from it before) and clears the tickets and flags for the next call.
// holes: d_0..d_{m-1} ascending, *nhole = m (k_pool_scatter<int32_t> over mode 0); src: [capacity] resolved sources;
// sync: [2 + capacity / RC_SEG + 1] = {ticket, done, segment flags}, zero between calls.
// -------------------------------------------------------------------------------------------
#define RC_SEG DSM_RECYCLE_SEG
#define RC_LOG 10 // log2(RC_SEG): doubling rounds that collapse any chain inside a segment
static_assert(RC_SEG == 1 << RC_LOG, "RC_LOG");
#define RC_MIN_GRID 16 // CTAs beyond the fill's: tail segments are taken by ticket, so any grid resolves any tail
__global__ void __launch_bounds__(RC_SEG) k_pool_recycle(const __grid_constant__ DsmDev d, int b, const int *nhole, const int32_t *holes,
                                                         int32_t *src, int32_t *sync, int32_t *ofs_out)
{
    pdl_enter();
    if (gated(d)) return; // uniform over the grid: no ticket is drawn, nothing to reset
    __shared__ int s_val[RC_SEG];
    __shared__ int s_ticket;
    const int N = d.poolofs[b + 1]; // the resident pool starts at 0
    const int m = *nhole, K = d.nnew[b];
    const int Np = N - m + K;
    const dsm_surfel_t *newsurf = d.newsurf + (size_t)b * d.S;
    for (int k = blockIdx.x * RC_SEG + threadIdx.x; k < K; k += gridDim.x * RC_SEG)
    { // fill: a hole at or above N' is popped, its new surfel is read from newsurf by the tail
        if (k < m)
        {
            const int h = holes[m - 1 - k];
            if (h < Np) d.pool[h] = newsurf[k];
        }
        else
            d.pool[N + k - m] = newsurf[k];
    }
    const int q = m - K;
    const int nseg = q > 0 ? (q + RC_SEG - 1) / RC_SEG : 0;
    while (nseg > 0)
    {
        if (threadIdx.x == 0) s_ticket = atomicAdd(&sync[0], 1);
        __syncthreads();
        const int ticket = s_ticket;
        __syncthreads();
        if (ticket >= nseg) break;
        const int seg = nseg - 1 - ticket, t0 = seg * RC_SEG, t = t0 + threadIdx.x;
        const bool mine = t < q;
        // v >= 0: pointer to tail offset v; v < 0: resolved, source -1 - v (a pool position in [N', N), or N + k for new[k])
        int v = 0;
        if (mine)
        {
            const int p = Np + t;
            if (d.pool[p].update_times != 0)
                v = -1 - p;
            else
            { // p is a hole d_i; the holes >= N' are the last entries of D, at most q of them: i is in [K, m)
                int lo = K, hi = m - 1;
                while (lo < hi)
                {
                    const int mid = (lo + hi) >> 1;
                    if (holes[mid] < p) lo = mid + 1;
                    else hi = mid;
                }
                if (lo >= q) v = -1 - (N + m - 1 - lo); // filled with new[m-1-i]
                else v = lo == t ? -1 - p : lo;         // leftover hole: what tail offset i held (i == t: never read)
            }
        }
        s_val[threadIdx.x] = v;
        if (__syncthreads_or(mine && v >= 0))
        {
#pragma unroll 1
            for (int r = 0; r < RC_LOG; r++)
            {
                const int nv = (mine && v >= 0 && v < t0 + RC_SEG) ? s_val[v - t0] : v;
                __syncthreads();
                s_val[threadIdx.x] = v = nv;
                __syncthreads();
            }
        }
        if (mine && v >= 0)
        { // leaves the segment upwards: that segment's CTA holds an earlier ticket
            const volatile int32_t *flag = sync + 2 + v / RC_SEG;
            while (*flag == 0) __nanosleep(32);
            __threadfence();
            v = __ldcg(src + v);
        }
        if (mine)
        {
            src[t] = v;
            const int h = holes[t];
            if (h < Np)
            {
                const int s = -1 - v;
                d.pool[h] = s >= N ? newsurf[s - N] : d.pool[s];
            }
        }
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) atomicExch(&sync[2 + seg], 1);
    }
    __shared__ bool s_last;
    if (threadIdx.x == 0)
    {
        __threadfence();
        s_last = atomicAdd(&sync[1], 1) == (int)gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    for (int i = threadIdx.x; i < nseg; i += RC_SEG) sync[2 + i] = 0;
    if (threadIdx.x == 0)
    {
        sync[0] = 0;
        sync[1] = 0;
        ofs_out[1] = Np;
    }
}

// p <- W p, n <- R_W n of one surfel record e, in place (the per-surfel body of both warp kernels of the reference)
__device__ __forceinline__ void transform_surfel(const float *W, float *e)
{
    float pw[4], nw[3];
    mat4_mul(W, e[0], e[1], e[2], 1.0f, pw);
    mat3_mul(W, e[3], e[4], e[5], nw);
    e[0] = pw[0], e[1] = pw[1], e[2] = pw[2];
    e[3] = nw[0], e[4] = nw[1], e[5] = nw[2];
}

#define XF_BLOCK 256
__global__ void __launch_bounds__(XF_BLOCK) k_pool_transform(const __grid_constant__ DsmDev d, int b, const float *Wm)
{
    __shared__ alignas(128) float sm[XF_BLOCK * 11];
    __shared__ float s_w[16];
    __shared__ uint64_t bar;
    const int begin = d.poolofs[b], end = d.poolofs[b + 1];
    const int first = begin + blockIdx.x * XF_BLOCK;
    if (first >= end) return;
    const int cnt = min(XF_BLOCK, end - first);
    float *g = reinterpret_cast<float *>(d.pool + first);
    if (threadIdx.x < 16) s_w[threadIdx.x] = Wm[threadIdx.x];
    const bool bulk = stage_in(sm, g, cnt, &bar, XF_BLOCK);
    __syncthreads(); // s_w
    if (threadIdx.x < cnt) transform_surfel(s_w, sm + threadIdx.x * 11);
    stage_out(g, sm, cnt, bulk, XF_BLOCK);
}

// two-entry offset table {a, b} written in stream order (the pool kernels take their range from device memory)
__global__ void k_set2(int32_t *p, int a, int b)
{
    p[0] = a;
    p[1] = b;
}
void dsm_launch_set2(int32_t *p, int a, int b, cudaStream_t s) { k_set2<<<1, 1, 0, s>>>(p, a, b); }

// -------------------------------------------------------------------------------------------
// Window step of dsm_fuse_stream_window: SurfelMap::move_add_surfels (surfel_map.cpp:1473-1594) for one frame, on the
// resident pool and the inactive store, with every count on the device.  The store is dense in retirement order and
// described by the segment table (keyframe, offset, count) in the same order; hdr holds its size and length.
//   k_win_plan     (reactivation) the listed keyframes' segments: their total, the pool slot each one goes to (list
//                  order, store order within a keyframe) and the offset every other segment will have after the holes
//                  close, kept in the segments' scratch field (< 0: -1 - pool slot; >= 0: new offset)
//   k_win_count    (retire) per 256-slot block of the pool, how many live surfels each listed keyframe owns
//   k_win_commit   capacity check of the whole frame (store after the retire, pool after the reactivation plus one
//                  frame of new surfels); a frame that does not fit sets the error word and nothing of it is applied.
//                  Otherwise: the block counts become store offsets (key-major scan), one segment per non-empty key is
//                  appended
//   k_win_scatter  (retire) the selected surfels to their store slots, flagged dead in the pool
//   k_win_copy     (reactivation) the listed segments to their pool slots
//   k_win_compact  (reactivation) the store's remaining surfels move down over the holes, order kept
//   k_win_finish   (reactivation) segment table compacted, store and pool sizes updated, compaction flags cleared
// Every kernel exits at once while the error word is set.  Surfels of a keyframe are selected by last_update: a
// surfel matches at most one listed keyframe, so one pass over the pool equals the reference's loop over the list.
// -------------------------------------------------------------------------------------------
#define WIN_MAX DSM_WINDOW_MAX_KEYS
__device__ __forceinline__ int win_list(const DsmWin &w, bool react, const int32_t **keys)
{
    const int32_t *o = w.tab + (react ? w.B + 1 : 0);
    const int a = o[w.t];
    *keys = w.tab + (react ? w.tab[2 * w.B + 3] : DSM_WIN_KEYS(w.B)) + a;
    return o[w.t + 1] - a;
}
__device__ __forceinline__ int win_rank(const int *s_key, int n, int kf)
{
    for (int r = 0; r < n; r++)
        if (s_key[r] == kf) return r;
    return -1;
}
__device__ __forceinline__ bool win_failed(const DsmWin &w) { return *(volatile const int32_t *)(w.res + 2) != 0; }
// exclusive prefix of v over a CTA of 32 * nwarp threads; total over the CTA in *tot (s_warp: 32 ints, reused)
__device__ __forceinline__ int cta_excl_scan(int v, int *s_warp, int &tot)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int wtot;
    const int ex = warp_excl_scan(v, lane, wtot);
    __syncthreads();
    if (lane == 31) s_warp[warp] = wtot;
    __syncthreads();
    int before = 0;
    tot = 0;
    for (int k = 0; k < nw; k++)
    {
        const int c = s_warp[k];
        before += k < warp ? c : 0;
        tot += c;
    }
    return before + ex;
}

__global__ void __launch_bounds__(1024) k_win_plan(const DsmWin w)
{
    pdl_enter();
    if (win_failed(w)) return;
    __shared__ int s_key[WIN_MAX], s_run[WIN_MAX], s_warp[32];
    __shared__ int s_lo, s_carry, s_sel[1024];
    const int32_t *keys;
    const int na = win_list(w, true, &keys);
    for (int r = threadIdx.x; r < na; r += blockDim.x) s_key[r] = keys[r], s_run[r] = 0;
    if (threadIdx.x == 0) s_lo = INT_MAX, s_carry = 0;
    __syncthreads();
    const int nseg = w.hdr[1], N = w.res[1];
    for (int j = threadIdx.x; j < nseg; j += blockDim.x)
    {
        const int4 s = w.seg[j];
        const int r = win_rank(s_key, na, s.x);
        if (r >= 0)
        {
            atomicAdd(&s_run[r], s.z);
            atomicMin(&s_lo, s.y);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0)
    { // s_run: first pool slot of each listed keyframe (list order)
        int run = 0;
        for (int r = 0; r < na; r++)
        {
            const int c = s_run[r];
            s_run[r] = N + run;
            run += c;
        }
        w.hdr[2] = run;
        w.hdr[3] = s_lo;
    }
    __syncthreads();
    for (int base = 0; base < nseg; base += blockDim.x)
    {
        const int j = base + threadIdx.x;
        int4 s = make_int4(0, 0, 0, 0);
        int r = -1;
        if (j < nseg)
        {
            s = w.seg[j];
            r = win_rank(s_key, na, s.x);
        }
        int tot;
        const int gone = s_carry + cta_excl_scan(r >= 0 ? s.z : 0, s_warp, tot); // reactivated surfels below this segment
        if (j < nseg && r < 0) w.seg[j].w = s.y - gone;
        int nsel;
        const int k = cta_excl_scan(r >= 0 ? 1 : 0, s_warp, nsel);
        if (r >= 0) s_sel[k] = j;
        __syncthreads();
        if (threadIdx.x == 0)
        { // the chunk's listed segments in store order: pool slots in order within each keyframe
            for (int q = 0; q < nsel; q++)
            {
                const int4 t = w.seg[s_sel[q]];
                const int rr = win_rank(s_key, na, t.x);
                w.seg[s_sel[q]].w = -1 - s_run[rr];
                s_run[rr] += t.z;
            }
            s_carry += tot;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_win_count(const __grid_constant__ DsmDev d, const DsmWin w)
{
    pdl_enter();
    if (win_failed(w)) return;
    __shared__ int s_key[WIN_MAX], s_cnt[WIN_MAX];
    const int32_t *keys;
    const int nr = win_list(w, false, &keys);
    const int N = w.res[1];
    if (blockIdx.x * 256 >= N) return; // the commit scans the blocks below N only
    for (int r = threadIdx.x; r < nr; r += 256) s_key[r] = keys[r], s_cnt[r] = 0;
    __syncthreads();
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < N && d.pool[i].update_times > 0)
    {
        const int r = win_rank(s_key, nr, d.pool[i].last_update);
        if (r >= 0) atomicAdd(&s_cnt[r], 1);
    }
    __syncthreads();
    for (int r = threadIdx.x; r < nr; r += 256) w.blk[(size_t)r * w.blk_stride + blockIdx.x] = s_cnt[r];
}

__global__ void __launch_bounds__(1024) k_win_commit(const DsmWin w, int nr, int na)
{
    pdl_enter();
    if (win_failed(w)) return;
    __shared__ int s_start[WIN_MAX + 1], s_warp[32], s_carry;
    const int32_t *keys;
    win_list(w, false, &keys);
    const int N = w.res[1], nblk = (N + 255) / 256, size = w.hdr[0];
    for (int r = threadIdx.x; r <= nr; r += blockDim.x) s_start[r] = 0;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    const int E = nr * nblk; // key-major: the surfels of key 0 in pool order, then key 1, ...
    for (int base = 0; base < E; base += blockDim.x)
    {
        const int e = base + threadIdx.x;
        const int r = nblk ? e / nblk : 0, b = nblk ? e - r * nblk : 0;
        int32_t *c = w.blk + (size_t)r * w.blk_stride + b;
        const int v = e < E ? *c : 0;
        int tot;
        const int ex = s_carry + cta_excl_scan(v, s_warp, tot);
        if (e < E)
        {
            *c = size + ex;
            if (b == 0) s_start[r] = ex;
        }
        __syncthreads();
        if (threadIdx.x == 0) s_carry += tot;
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    const int moved = s_carry, react = na > 0 ? w.hdr[2] : 0;
    s_start[nr] = moved;
    if ((long long)size + moved > w.store_cap || (long long)N + react + w.S > w.pool_cap)
    { // the frame does not fit: it and every later one are not applied
        w.res[3] = w.t;
        __threadfence();
        w.res[2] = w.tab[2 * w.B + 2];
        return;
    }
    int nseg = w.hdr[1];
    for (int r = 0; r < nr; r++)
    {
        const int c = s_start[r + 1] - s_start[r];
        if (c > 0) w.seg[nseg++] = make_int4(keys[r], size + s_start[r], c, size + s_start[r] - react);
    }
    w.hdr[0] = size + moved;
    w.hdr[1] = nseg;
}

__global__ void __launch_bounds__(256) k_win_scatter(const __grid_constant__ DsmDev d, const DsmWin w)
{
    pdl_enter();
    if (win_failed(w)) return;
    __shared__ int s_key[WIN_MAX], s_wc[8][WIN_MAX];
    const int32_t *keys;
    const int nr = win_list(w, false, &keys);
    const int N = w.res[1];
    if (blockIdx.x * 256 >= N) return;
    for (int r = threadIdx.x; r < nr; r += 256) s_key[r] = keys[r];
    for (int q = threadIdx.x; q < 8 * nr; q += 256) s_wc[q / nr][q % nr] = 0;
    __syncthreads();
    const int i = blockIdx.x * 256 + threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    dsm_surfel_t e;
    int r = -1;
    if (i < N)
    {
        e = d.pool[i];
        if (e.update_times > 0) r = win_rank(s_key, nr, e.last_update);
    }
    // position among the block's surfels of the same key, in pool order: within the warp, then over the warps before
    const unsigned peers = __match_any_sync(FULL, r);
    if (r >= 0 && lane == __ffs(peers) - 1) s_wc[warp][r] = __popc(peers);
    __syncthreads();
    if (r < 0) return;
    int pos = w.blk[(size_t)r * w.blk_stride + blockIdx.x] + __popc(peers & ((1u << lane) - 1));
    for (int q = 0; q < warp; q++) pos += s_wc[q][r];
    w.store[pos] = e;
    d.pool[i].update_times = 0; // "delete the surfel from the local point" (surfel_map.cpp:1496)
}

__global__ void __launch_bounds__(256) k_win_copy(const __grid_constant__ DsmDev d, const DsmWin w)
{
    pdl_enter();
    if (win_failed(w) || w.hdr[2] == 0) return;
    __shared__ int4 s_list[256];
    __shared__ int s_n;
    const int nseg = w.hdr[1];
    for (int base = 0; base < nseg; base += 256)
    {
        __syncthreads();
        if (threadIdx.x == 0) s_n = 0;
        __syncthreads();
        const int j = base + threadIdx.x;
        if (j < nseg)
        {
            const int4 s = w.seg[j];
            if (s.w < 0) s_list[atomicAdd(&s_n, 1)] = s;
        }
        __syncthreads();
        for (int q = 0; q < s_n; q++)
        {
            const int4 s = s_list[q];
            dsm_surfel_t *dst = d.pool + (-1 - s.w);
            for (int k = blockIdx.x * 256 + threadIdx.x; k < s.z; k += gridDim.x * 256) dst[k] = w.store[s.y + k];
        }
    }
}

// In place, downwards, order kept.  The range [lo, size) is cut into chunks of DSM_WIN_CHUNK surfels that CTAs take by
// ticket in ascending order.  A CTA reads its chunk into shared memory, raises the chunk's flag, then waits for the
// flags of the chunks its destinations fall into (all of them below or at its own: every destination is below its
// source) before it writes.  It only ever waits for chunks with earlier tickets, whose CTAs are running and raise
// their flags without waiting for anything: no co-residency is assumed and no store-sized scratch is used.
__global__ void __launch_bounds__(DSM_WIN_CHUNK) k_win_compact(const DsmWin w)
{
    pdl_enter();
    if (win_failed(w) || w.hdr[2] == 0) return;
    __shared__ dsm_surfel_t s_e[DSM_WIN_CHUNK];
    __shared__ int s_ticket, s_dmin;
    const int size = w.hdr[0], lo = w.hdr[3], nseg = w.hdr[1];
    const int nchunk = (size - lo + DSM_WIN_CHUNK - 1) / DSM_WIN_CHUNK;
    for (;;)
    {
        __syncthreads();
        if (threadIdx.x == 0)
        {
            s_ticket = atomicAdd(&w.sync[0], 1);
            s_dmin = INT_MAX;
        }
        __syncthreads();
        const int k = s_ticket;
        if (k >= nchunk) break;
        const int p = lo + k * DSM_WIN_CHUNK + threadIdx.x;
        int dst = -1;
        if (p < size)
        { // the segment holding p: the last one starting at or below it
            int a = 0, b = nseg - 1;
            while (a < b)
            {
                const int m = (a + b + 1) >> 1;
                if (w.seg[m].y <= p) a = m;
                else b = m - 1;
            }
            const int4 s = w.seg[a];
            if (s.w >= 0)
            {
                dst = s.w + (p - s.y);
                s_e[threadIdx.x] = w.store[p];
                atomicMin(&s_dmin, dst);
            }
        }
        __syncthreads();
        if (threadIdx.x == 0)
        {
            __threadfence();
            atomicExch(&w.sync[2 + k], 1);
            if (s_dmin != INT_MAX)
                for (int j = (s_dmin - lo) / DSM_WIN_CHUNK; j < k; j++)
                {
                    const volatile int32_t *flag = w.sync + 2 + j;
                    while (*flag == 0) __nanosleep(32);
                }
            __threadfence();
        }
        __syncthreads();
        if (dst >= 0) w.store[dst] = s_e[threadIdx.x];
    }
}

__global__ void __launch_bounds__(1024) k_win_finish(const DsmWin w)
{
    pdl_enter();
    if (win_failed(w)) return;
    __shared__ int s_warp[32], s_carry;
    const int react = w.hdr[2], size = w.hdr[0], lo = w.hdr[3], nseg = w.hdr[1];
    if (react == 0) return; // nothing was stored for the listed keyframes: no compaction ran
    const int nchunk = (size - lo + DSM_WIN_CHUNK - 1) / DSM_WIN_CHUNK;
    for (int i = threadIdx.x; i < nchunk; i += blockDim.x) w.sync[2 + i] = 0;
    if (threadIdx.x == 0) w.sync[0] = 0, s_carry = 0;
    __syncthreads();
    for (int base = 0; base < nseg; base += blockDim.x)
    { // entries only move down, and a chunk is read before any of it is written
        const int j = base + threadIdx.x;
        int4 s = make_int4(0, 0, 0, -1);
        if (j < nseg) s = w.seg[j];
        int tot;
        const int k = s_carry + cta_excl_scan(s.w >= 0 ? 1 : 0, s_warp, tot);
        __syncthreads();
        if (j < nseg && s.w >= 0) w.seg[k] = make_int4(s.x, s.w, s.z, 0);
        __syncthreads();
        if (threadIdx.x == 0) s_carry += tot;
        __syncthreads();
    }
    __syncthreads();
    if (threadIdx.x == 0)
    {
        w.hdr[0] = size - react;
        w.hdr[1] = s_carry;
        w.res[1] += react;
    }
}

// warp_inactive_surfels_cpu_kernel (surfel_map.cpp:704-733) on the segments of keyframe kf, found in the device table,
// one surfel per thread
__global__ void __launch_bounds__(256) k_inactive_transform(const DsmWin w, int kf, const float *Wm)
{
    __shared__ float s_w[16];
    __shared__ int2 s_list[256];
    __shared__ int s_n;
    if (threadIdx.x < 16) s_w[threadIdx.x] = Wm[threadIdx.x];
    const int nseg = w.hdr[1];
    for (int base = 0; base < nseg; base += 256)
    {
        __syncthreads();
        if (threadIdx.x == 0) s_n = 0;
        __syncthreads();
        const int j = base + threadIdx.x;
        if (j < nseg)
        {
            const int4 s = w.seg[j];
            if (s.x == kf) s_list[atomicAdd(&s_n, 1)] = make_int2(s.y, s.z);
        }
        __syncthreads();
        for (int q = 0; q < s_n; q++)
            for (int k = blockIdx.x * 256 + threadIdx.x; k < s_list[q].y; k += gridDim.x * 256)
                transform_surfel(s_w, reinterpret_cast<float *>(w.store + s_list[q].x + k));
    }
}

// -------------------------------------------------------------------------------------------
// k_cloud_mirror — the inactive cloud of dsm_publish_enqueue, incrementally.  `shadow` holds the cloud as the host
// mirror last received it, [0, state[0]) of it being published.  CTA c forms the points {px, py, pz, color} of the
// stored surfels [256 c, 256 c + 256) below the store size (device header), compares them bit for bit with the shadow,
// and if one differs, or the chunk reaches beyond the previously published size, writes the chunk to the shadow and,
// through the device alias of the pinned host buffer, to the mirror at the same offset: 16 bytes per thread, whole
// 128-byte lines per quarter-warp, and only changed chunks cross PCIe.  Nothing upstream marks what it changed: the
// compare finds it whatever kernel wrote the store.  The surfels are staged like k_pool_transform's (one TMA bulk copy
// per chunk, stride-11 words); the pass reads 44 + 16 bytes per stored surfel and writes 32 per forwarded point.
// The last CTA to finish writes the header (PUB_* words) and prepares `state` {published size, lowest changed index,
// chunks forwarded, CTAs done} for the next snapshot.  A context without a store runs one CTA on size 0.
// -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(DSM_PUB_CHUNK) k_cloud_mirror(const dsm_surfel_t *store, const int32_t *size_word, const int32_t *res,
                                                                float4 *shadow, float4 *mirror, int32_t *state, int32_t *header)
{
    __shared__ alignas(128) float sm[DSM_PUB_CHUNK * 11];
    __shared__ uint64_t bar;
    __shared__ int s_low;
    __shared__ bool s_last;
    const int size = store ? *size_word : 0, prev = state[0];
    const int nchunk = max(1, (size + DSM_PUB_CHUNK - 1) / DSM_PUB_CHUNK);
    if ((int)blockIdx.x >= nchunk) return; // the grid is sized from the host's upper bound of the store
    const int first = blockIdx.x * DSM_PUB_CHUNK, cnt = min(DSM_PUB_CHUNK, size - first);
    if (threadIdx.x == 0) s_low = INT_MAX;
    if (cnt > 0)
    {
        stage_in(sm, reinterpret_cast<const float *>(store + first), cnt, &bar, DSM_PUB_CHUNK);
        const int i = first + threadIdx.x;
        float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
        bool differs = false;
        if (threadIdx.x < cnt)
        {
            const float *e = sm + threadIdx.x * 11;
            p = make_float4(e[0], e[1], e[2], e[7]);
            differs = i >= prev;
            if (!differs)
            {
                const float4 o = shadow[i];
                differs = __float_as_uint(o.x) != __float_as_uint(p.x) || __float_as_uint(o.y) != __float_as_uint(p.y) ||
                          __float_as_uint(o.z) != __float_as_uint(p.z) || __float_as_uint(o.w) != __float_as_uint(p.w);
            }
            if (differs) atomicMin(&s_low, i);
        }
        if (__syncthreads_or(differs))
        {
            if (threadIdx.x < cnt)
            {
                shadow[i] = p;
                mirror[i] = p;
            }
            if (threadIdx.x == 0)
            {
                atomicMin(&state[1], s_low);
                atomicAdd(&state[2], 1);
            }
        }
    }
    __syncthreads(); // the chunk's stores come before the count of finished CTAs
    if (threadIdx.x == 0)
    {
        __threadfence();
        s_last = atomicAdd(&state[3], 1) == nchunk - 1;
    }
    __syncthreads();
    if (!s_last || threadIdx.x != 0) return;
    __threadfence();
    const volatile int32_t *st = state;
    header[DSM_PUB_N_INACTIVE] = size;
    header[DSM_PUB_PREV] = prev;
    header[DSM_PUB_CHANGED_FROM] = min(st[1], size);
    header[DSM_PUB_CHUNKS] = st[2];
    header[DSM_PUB_ERR_TAG] = res[2];
    header[DSM_PUB_ERR_FRAME] = res[3];
    state[0] = size;
    state[1] = INT_MAX;
    state[2] = 0;
    state[3] = 0;
}

// -------------------------------------------------------------------------------------------
// k_map_snapshot — the map of dsm_checkpoint_enqueue at its position in the stream, into the checkpoint's device image
// (DsmSnapLayout).  The live sizes exist on the device only (res_ofs[1], win_hdr), so the copy is sized here: CTA c
// < pool_grid copies pool surfels [256 c, 256 c + 256) below the pool size, CTA pool_grid + c stored surfels
// [256 c, 256 c + 256) below the store size and the segments with the same indices (a segment holds >= 1 surfel, so
// every live segment falls to a live CTA), packed from int4 to int32[3].  The surfels are staged like
// k_pool_transform's: source and destination chunks start 11264 * c bytes from 128-byte aligned bases, so every whole
// chunk moves as one TMA bulk copy each way and only the ragged last chunk of a section goes word by word.  CTA 0 writes
// the header, the error word included: the snapshot does not wait on it (it records it, as k_cloud_mirror does).
// Launched without PDL: it begins after everything enqueued before it has completed.
// -------------------------------------------------------------------------------------------
#define SNAP_CHUNK 256
__global__ void __launch_bounds__(SNAP_CHUNK) k_map_snapshot(const dsm_surfel_t *pool, const int32_t *res, int pool_grid,
                                                             const dsm_surfel_t *store, const int4 *seg, const int32_t *hdr,
                                                             uint8_t *image, const DsmSnapLayout lay)
{
    __shared__ alignas(128) float sm[SNAP_CHUNK * 11];
    __shared__ uint64_t bar;
    const int n_pool = res[1], n_store = store ? hdr[0] : 0, n_seg = store ? hdr[1] : 0;
    if (blockIdx.x == 0 && threadIdx.x == 0)
    {
        int32_t *h = reinterpret_cast<int32_t *>(image);
        h[DSM_SNAP_N_POOL] = n_pool;
        h[DSM_SNAP_N_STORE] = n_store;
        h[DSM_SNAP_N_SEGMENTS] = n_seg;
        h[DSM_SNAP_ERR_TAG] = res[2];
        h[DSM_SNAP_ERR_FRAME] = res[3];
    }
    const bool in_pool = (int)blockIdx.x < pool_grid;
    const int first = (in_pool ? blockIdx.x : blockIdx.x - pool_grid) * SNAP_CHUNK;
    const int n = in_pool ? n_pool : n_store;
    if (first >= n) return;
    const int cnt = min(SNAP_CHUNK, n - first);
    if (!in_pool && first + (int)threadIdx.x < n_seg)
    {
        const int i = first + threadIdx.x;
        const int4 g = seg[i];
        int32_t *t = reinterpret_cast<int32_t *>(image + lay.table) + 3 * (size_t)i;
        t[0] = g.x, t[1] = g.y, t[2] = g.z;
    }
    const float *src = reinterpret_cast<const float *>((in_pool ? pool : store) + first);
    float *dst = reinterpret_cast<float *>(image + (in_pool ? lay.pool : lay.store)) + (size_t)first * 11;
    const bool bulk = stage_in(sm, src, cnt, &bar, SNAP_CHUNK); // dst is 16-byte aligned whenever src is
    stage_out(dst, sm, cnt, bulk, SNAP_CHUNK);
}

// -------------------------------------------------------------------------------------------
// k_map_drain — the live part of the checkpoint image to its pinned host twin through the device alias, on a side
// stream after k_map_snapshot: the header line and the whole 128-byte lines that hold each section's live bytes (the
// sections are line-aligned and sized in lines, so the last line of a section stays inside it).  16 bytes per thread,
// a quarter-warp per line; a small fixed grid, since the copy is bound by PCIe and must leave the SMs to the stream's
// kernels.
// -------------------------------------------------------------------------------------------
#define DRAIN_BLOCK 256
__global__ void __launch_bounds__(DRAIN_BLOCK) k_map_drain(const uint8_t *image, uint8_t *host, const DsmSnapLayout lay)
{
    const int32_t *h = reinterpret_cast<const int32_t *>(image);
    const size_t lp = ((size_t)h[DSM_SNAP_N_POOL] * 44 + 127) / 128, ls = ((size_t)h[DSM_SNAP_N_STORE] * 44 + 127) / 128;
    const size_t lt = ((size_t)h[DSM_SNAP_N_SEGMENTS] * 12 + 127) / 128;
    const size_t words = 8 * (1 + lp + ls + lt);
    for (size_t w = (size_t)blockIdx.x * DRAIN_BLOCK + threadIdx.x; w < words; w += (size_t)gridDim.x * DRAIN_BLOCK)
    {
        size_t line = w >> 3, ofs;
        if (line == 0) ofs = 0;
        else if ((line -= 1) < lp) ofs = lay.pool + line * 128;
        else if ((line -= lp) < ls) ofs = lay.store + line * 128;
        else ofs = lay.table + (line - ls) * 128;
        ofs += (w & 7) * 16;
        *reinterpret_cast<int4 *>(host + ofs) = __ldg(reinterpret_cast<const int4 *>(image + ofs));
    }
}

// -------------------------------------------------------------------------------------------
// k_map_delta — the map of dsm_checkpoint_enqueue_incremental at its position in the stream, into the same device image,
// which already holds the map of the last checkpoint (DESIGN.md §8.6).  k_map_snapshot's grid and chunks: CTA c <
// pool_grid stages pool chunk c, CTA pool_grid + c store chunk c (and writes the segments with the same indices), each
// staged like k_pool_transform's.  A chunk is changed if one of its live words differs from the image's, or if it
// reaches beyond the image's size of its section (k_map_snapshot writes nothing past the live sizes); only a changed
// chunk is written into the image.  Each live CTA writes its chunk's flag, so the set of flags depends on the two maps
// alone.  The image's sizes are read at the start of every CTA; the last CTA to finish rewrites the header (new sizes,
// previous sizes, error word) once every other has read them.  Launched without PDL, like k_map_snapshot.
// -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SNAP_CHUNK) k_map_delta(const dsm_surfel_t *pool, const int32_t *res, int pool_grid,
                                                          const dsm_surfel_t *store, const int4 *seg, const int32_t *hdr,
                                                          uint8_t *image, const DsmSnapLayout lay, int pool_chunks)
{
    __shared__ alignas(128) float sm[SNAP_CHUNK * 11];
    __shared__ uint64_t bar;
    __shared__ bool s_last;
    int32_t *h = reinterpret_cast<int32_t *>(image);
    const int n_pool = res[1], n_store = store ? hdr[0] : 0, n_seg = store ? hdr[1] : 0;
    const bool in_pool = (int)blockIdx.x < pool_grid;
    const int c = in_pool ? blockIdx.x : blockIdx.x - pool_grid, first = c * SNAP_CHUNK;
    const int n = in_pool ? n_pool : n_store;
    const int prev = h[in_pool ? DSM_SNAP_N_POOL : DSM_SNAP_N_STORE];
    bool changed = false;
    if (first < n)
    {
        const int cnt = min(SNAP_CHUNK, n - first);
        if (!in_pool && first + (int)threadIdx.x < n_seg)
        {
            const int i = first + threadIdx.x;
            const int4 g = seg[i];
            int32_t *t = reinterpret_cast<int32_t *>(image + lay.table) + 3 * (size_t)i;
            t[0] = g.x, t[1] = g.y, t[2] = g.z;
        }
        const float *src = reinterpret_cast<const float *>((in_pool ? pool : store) + first);
        float *dst = reinterpret_cast<float *>(image + (in_pool ? lay.pool : lay.store)) + (size_t)first * 11;
        const bool bulk = stage_in(sm, src, cnt, &bar, SNAP_CHUNK);
        bool differs = first + cnt > prev;
        if (!differs)
        {
            const uint32_t *old = reinterpret_cast<const uint32_t *>(dst);
            for (int i = threadIdx.x; i < cnt * 11; i += SNAP_CHUNK) differs |= __float_as_uint(sm[i]) != old[i];
        }
        changed = __syncthreads_or(differs);
        if (changed) stage_out(dst, sm, cnt, bulk, SNAP_CHUNK);
    }
    if (threadIdx.x == 0) image[lay.bytes + (in_pool ? c : pool_chunks + c)] = changed ? 1 : 0;
    __syncthreads();
    if (threadIdx.x == 0)
    {
        __threadfence();
        s_last = atomicAdd(&h[DSM_DELTA_DONE], 1) == (int)gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last || threadIdx.x != 0) return;
    __threadfence();
    volatile int32_t *v = h;
    v[DSM_DELTA_PREV_POOL] = v[DSM_SNAP_N_POOL];
    v[DSM_DELTA_PREV_STORE] = v[DSM_SNAP_N_STORE];
    v[DSM_SNAP_N_POOL] = n_pool;
    v[DSM_SNAP_N_STORE] = n_store;
    v[DSM_SNAP_N_SEGMENTS] = n_seg;
    v[DSM_SNAP_ERR_TAG] = res[2];
    v[DSM_SNAP_ERR_FRAME] = res[3];
    v[DSM_DELTA_DONE] = 0;
}

// -------------------------------------------------------------------------------------------
// k_map_drain_delta — k_map_drain for k_map_delta's image: the header line, the flag lines and the live table lines
// whole, then one warp per live chunk that copies the chunk's live 128-byte lines if its flag is set (a chunk of 256
// surfels is 88 lines, and each section starts on a line).  The same small fixed grid as k_map_drain.
// -------------------------------------------------------------------------------------------
#define CHUNK_LINES (SNAP_CHUNK * 44 / 128)
__global__ void __launch_bounds__(DRAIN_BLOCK) k_map_drain_delta(const uint8_t *image, uint8_t *host, const DsmSnapLayout lay,
                                                                 int pool_chunks, int store_chunks)
{
    const int32_t *h = reinterpret_cast<const int32_t *>(image);
    const int n_pool = h[DSM_SNAP_N_POOL], n_store = h[DSM_SNAP_N_STORE];
    const size_t lp = ((size_t)n_pool * 44 + 127) / 128, ls = ((size_t)n_store * 44 + 127) / 128;
    const size_t lt = ((size_t)h[DSM_SNAP_N_SEGMENTS] * 12 + 127) / 128, lf = ((size_t)pool_chunks + store_chunks + 127) / 128;
    const size_t words = 8 * (1 + lf + lt);
    for (size_t w = (size_t)blockIdx.x * DRAIN_BLOCK + threadIdx.x; w < words; w += (size_t)gridDim.x * DRAIN_BLOCK)
    {
        size_t line = w >> 3, ofs;
        if (line == 0) ofs = 0;
        else if ((line -= 1) < lf) ofs = lay.bytes + line * 128;
        else ofs = lay.table + (line - lf) * 128;
        ofs += (w & 7) * 16;
        *reinterpret_cast<int4 *>(host + ofs) = __ldg(reinterpret_cast<const int4 *>(image + ofs));
    }
    const uint8_t *flags = image + lay.bytes;
    const int cp = (n_pool + SNAP_CHUNK - 1) / SNAP_CHUNK, cs = (n_store + SNAP_CHUNK - 1) / SNAP_CHUNK;
    const int warps = gridDim.x * (DRAIN_BLOCK / 32), lane = threadIdx.x & 31;
    for (int q = blockIdx.x * (DRAIN_BLOCK / 32) + (threadIdx.x >> 5); q < cp + cs; q += warps)
    {
        const bool in_pool = q < cp;
        const int c = in_pool ? q : q - cp;
        if (!flags[in_pool ? c : pool_chunks + c]) continue;
        const size_t base = in_pool ? lay.pool : lay.store, l0 = (size_t)c * CHUNK_LINES;
        const size_t l1 = min(l0 + CHUNK_LINES, in_pool ? lp : ls);
        for (size_t w = l0 * 8 + lane; w < l1 * 8; w += 32)
        {
            const size_t ofs = base + w * 16;
            *reinterpret_cast<int4 *>(host + ofs) = __ldg(reinterpret_cast<const int4 *>(image + ofs));
        }
    }
}

// -------------------------------------------------------------------------------------------
// parity readback: rebuild the reference's 60-byte Superpixel_seed records for one frame
// -------------------------------------------------------------------------------------------
__global__ void k_seeds_export(const __grid_constant__ DsmDev d, int b, dsm_seed_t *out, int raw_md)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= d.S) return;
    const size_t o = (size_t)b * d.S + s;
    const float4 sd = d.seed[o];
    const float4 *pl = d.plane + o * 3;
    const float4 r0 = pl[0], r1 = pl[1], r2 = pl[2];
    dsm_seed_t e;
    e.x = sd.x, e.y = sd.y;
    e.size = r2.x;
    e.norm_x = r0.x, e.norm_y = r0.y, e.norm_z = r0.z;
    e.posi_x = r1.x, e.posi_y = r1.y, e.posi_z = r1.z;
    e.view_cos = r0.w;
    e.mean_depth = raw_md ? sd.w : r1.w; // raw_md: clustering state before the plane fit (debug staging)
    e.mean_intensity = sd.z;
    e.fused = d.fused[o] ? 1 : 0;
    e.stable = (d.tstable[o] == DSM_STABLE) ? 1 : 0;
    e._pad[0] = e._pad[1] = 0;
    e.min_eigen_value = 0.f;
    e.max_eigen_value = 0.f;
    out[s] = e;
}

// parity readback: the reference's int32 superpixel_index of one frame, from the label codes
__global__ void k_labels_export(const __grid_constant__ DsmDev d, int b)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= d.W) return;
    const size_t o = (size_t)b * d.px_stride + (size_t)y * d.Wp + x;
    d.labels[o] = dsm_code_seed(d.code[o], x, y, d.spw);
}

// -------------------------------------------------------------------------------------------
// raw cloud — publish_raw_pointcloud (surfel_map.cpp:1115-1151): every pixel of one frame back-projected into the world,
// intensity = gray.  The reference loops column-outer (point k = i*H + j) while the planes are row-major, so a CTA
// transposes a 32-column x 32-row tile through shared memory: coalesced row reads, points computed in registers and
// staged as float4 (row pitch 33: conflict-free both ways), then each column's run of up to 32 points is stored as
// contiguous 16-byte points (512 B per warp and column).  Float operations in the reference's order; with -fmad=false
// and IEEE division the points are bit-identical to the serial loop (holes included: depth 0 maps to T).
// -------------------------------------------------------------------------------------------
#define RAW_TILE 32
__global__ void __launch_bounds__(256) k_raw_cloud(const __grid_constant__ DsmDev d, int b, const DsmRawPose P, float4 *out)
{
    __shared__ float4 tile[RAW_TILE][RAW_TILE + 1]; // [column][row]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int i0 = blockIdx.x * RAW_TILE, j0 = blockIdx.y * RAW_TILE;
    const int i = i0 + lane;
    const float ci = (float)i - d.cx; // (i - cam_cx): int promoted to float
    const size_t base = (size_t)b * d.px_stride;
#pragma unroll
    for (int r = warp; r < RAW_TILE; r += 8)
    {
        const int j = j0 + r;
        if (i >= d.W || j >= d.H) continue;
        const size_t o = base + (size_t)j * d.Wp + i;
        const float z = d.depth[o];
        const float c0 = ci * z / d.fx;
        const float c1 = ((float)j - d.cy) * z / d.fy;
        float4 p;
        p.x = ((P.R[0] * c0 + P.R[1] * c1) + P.R[2] * z) + P.T[0];
        p.y = ((P.R[3] * c0 + P.R[4] * c1) + P.R[5] * z) + P.T[1];
        p.z = ((P.R[6] * c0 + P.R[7] * c1) + P.R[8] * z) + P.T[2];
        p.w = (float)d.gray[o];
        tile[lane][r] = p;
    }
    __syncthreads();
    const int rows = min(RAW_TILE, d.H - j0);
    if (lane >= rows) return;
#pragma unroll
    for (int c = warp; c < RAW_TILE; c += 8)
        if (i0 + c < d.W) out[(size_t)(i0 + c) * d.H + j0 + lane] = tile[c][lane];
}

// -------------------------------------------------------------------------------------------
// superpixel image — FusionFunctions::debug_show (fusion_functions.cpp:977-1006) of one frame: every pixel painted with
// |normal| * 255 of its superpixel (cv::Vec3b order {|nx|, |ny|, |nz|}), black where the right or the lower neighbour has
// another label.  A thread covers 4 consecutive pixels of a row: one u32 of codes, the u32 below it and the code right of
// its last pixel (both L1/L2 hits of neighbouring threads' rows); its 12 output bytes go through a per-warp staging row
// so that the warp stores 96 consecutive 32-bit words.  Output rows have a pitch of 3*Wp bytes; pixels >= W are 0.
// -------------------------------------------------------------------------------------------
// `uchar = fabs(n) * 255` (:986-988) as the reference's x86-64 build computes it: fabs of the float promoted to double,
// the product exact in double (24-bit mantissa x 255 < 2^32), then a truncating conversion through int32 whose low byte
// is kept; NaN (and anything >= 2^31) converts to INT_MIN, i.e. byte 0
__device__ __forceinline__ uint32_t sp_channel(float n)
{
    const double v = fabs((double)n) * 255.0;
    return v < 2147483648.0 ? (uint32_t)(int)v & 0xffu : 0u;
}

#define SPI_PX 4                    // pixels per thread
#define SPI_WARPS 4                 // rows per CTA (one warp each)
#define SPI_SPAN (32 * SPI_PX)      // pixels per warp
__global__ void __launch_bounds__(32 * SPI_WARPS) k_superpixel_image(const __grid_constant__ DsmDev d, int b, uint32_t *out)
{
    __shared__ uint32_t stage[SPI_WARPS][3 * 32]; // a warp's 384 output bytes; lane l writes words 3l..3l+2 (conflict-free)
    const int lane = threadIdx.x, y = blockIdx.y * SPI_WARPS + threadIdx.y;
    if (y >= d.H) return; // whole warps: the rows of a CTA are its warps
    const int x0 = blockIdx.x * SPI_SPAN, x = x0 + lane * SPI_PX;
    uint32_t px[SPI_PX] = {0u, 0u, 0u, 0u}; // 24-bit {b0, b1, b2} per pixel
    if (x < d.W)
    { // x + 3 < Wp (Wp is a multiple of 16): the u32 reads stay inside the pitched row
        const size_t o = (size_t)b * d.px_stride + (size_t)y * d.Wp + x;
        const uint32_t c = *reinterpret_cast<const uint32_t *>(d.code + o);
        const uint32_t cd = y + 1 < d.H ? *reinterpret_cast<const uint32_t *>(d.code + o + d.Wp) : 0u;
        const int right = x + SPI_PX < d.W ? dsm_code_seed(d.code[o + SPI_PX], x + SPI_PX, y, d.spw) : -1;
        const float4 *pl = d.plane + (size_t)b * d.S * 3;
        int s = dsm_code_seed(c & 0xff, x, y, d.spw);
#pragma unroll
        for (int i = 0; i < SPI_PX; i++)
        {
            const int xi = x + i;
            if (xi >= d.W) break;
            // right neighbour: the next pixel of this thread, or the first pixel of the next group
            const int sr = i + 1 < SPI_PX ? dsm_code_seed((c >> (8 * (i + 1))) & 0xff, xi + 1, y, d.spw) : right;
            const bool edge = (xi + 1 < d.W && sr != s) || (y + 1 < d.H && dsm_code_seed((cd >> (8 * i)) & 0xff, xi, y + 1, d.spw) != s);
            if (!edge)
            {
                const float4 n = pl[(size_t)s * 3];
                px[i] = sp_channel(n.x) | sp_channel(n.y) << 8 | sp_channel(n.z) << 16;
            }
            s = sr;
        }
    }
    uint32_t *st = stage[threadIdx.y];
    st[3 * lane + 0] = px[0] | px[1] << 24;
    st[3 * lane + 1] = px[1] >> 8 | px[2] << 16;
    st[3 * lane + 2] = px[2] >> 16 | px[3] << 8;
    __syncwarp();
    // the row holds 3*Wp/4 words (Wp is a multiple of 16); this warp's run starts at word 3*x0/4
    const int row_words = 3 * d.Wp / 4, w0 = 3 * x0 / 4;
    uint32_t *dst = out + (size_t)y * row_words + w0;
#pragma unroll
    for (int k = 0; k < 3; k++)
        if (w0 + 32 * k + lane < row_words) dst[32 * k + lane] = st[32 * k + lane];
}

// -------------------------------------------------------------------------------------------
// launchers
// -------------------------------------------------------------------------------------------
void dsm_launch_repack(const DsmDev &d, int nb, const uint8_t *gray_packed, const float *depth_packed, cudaStream_t s)
{
    dim3 block(64, 4);
    dim3 grid((d.Wp + 255) / 256, (d.H + 3) / 4, nb);
    k_repack<<<grid, block, 0, s>>>(d, gray_packed, depth_packed);
}
void dsm_launch_seed_init(const DsmDev &d, int nb, cudaStream_t s)
{
    dim3 grid((d.S + 255) / 256, nb);
    pdl_launch(k_seed_init, grid, dim3(256), 0, s, d);
}
void dsm_launch_fuse(const DsmDev &d, int nb, cudaStream_t s)
{
    if (d.max_pool_per_frame <= 0) return;
    dim3 grid((d.max_pool_per_frame + FUSE_BLOCK - 1) / FUSE_BLOCK, nb);
    pdl_launch(k_fuse, grid, dim3(FUSE_BLOCK), 0, s, d);
}
void dsm_launch_init_surfels(const DsmDev &d, int nb, cudaStream_t s)
{
    dim3 grid((d.S + 1023) / 1024, nb);
    pdl_launch(k_init_surfels, grid, dim3(1024), 0, s, d);
}
void dsm_launch_seeds_export(const DsmDev &d, int frame, dsm_seed_t *out_dev, int raw_md, cudaStream_t s)
{
    k_seeds_export<<<(d.S + 255) / 256, 256, 0, s>>>(d, frame, out_dev, raw_md);
}
void dsm_launch_labels_export(const DsmDev &d, int frame, cudaStream_t s)
{
    k_labels_export<<<dim3((d.W + 255) / 256, d.H), 256, 0, s>>>(d, frame);
}

template <typename... KArgs, typename... Args>
static void sel_launch(bool pdl, void (*kern)(KArgs...), int grid, int block, cudaStream_t s, Args &&...args)
{
    if (pdl) pdl_launch(kern, dim3(grid), dim3(block), 0, s, args...);
    else kern<<<grid, block, 0, s>>>(args...);
}
void dsm_launch_pool_select(const DsmDev &d, int frame, int upper, int mode, int key, DsmRec rec, void *dst, int *blkcnt,
                            int *blkofs, int *nsel, cudaStream_t s, int flags)
{
    const int nblk = (upper + 255) / 256;
    const bool pdl = flags & DSM_SEL_PDL;
    if (!(flags & DSM_SEL_SCATTER_ONLY))
    {
        if (nblk > 0) sel_launch(pdl, k_pool_count, nblk, 256, s, d, frame, blkcnt, mode, key);
        sel_launch(pdl, k_pool_scan, 1, 1024, s, d, frame, (const int *)blkcnt, blkofs, nsel);
    }
    if (nblk == 0 || !dst) return;
    const int *ofs = blkofs;
    if (rec == DSM_REC_INDEX) sel_launch(pdl, k_pool_scatter<int32_t>, nblk, 256, s, d, frame, ofs, static_cast<int32_t *>(dst), mode, key);
    else if (rec == DSM_REC_POINT) sel_launch(pdl, k_pool_scatter<float4>, nblk, 256, s, d, frame, ofs, static_cast<float4 *>(dst), mode, key);
    else sel_launch(pdl, k_pool_scatter<dsm_surfel_t>, nblk, 256, s, d, frame, ofs, static_cast<dsm_surfel_t *>(dst), mode, key);
}

// the fuse_map post-step on the resident pool of frame slot `frame` (whose offset table is ofs_out = {0, N}): hole list,
// then k_pool_recycle, whose last CTA stores the new size in ofs_out[1].  upper >= N bounds the grids.
void dsm_launch_pool_recycle(const DsmDev &d, int frame, int upper, int *blkcnt, int *blkofs, int *nsel, int32_t *holes, int32_t *src,
                             int32_t *sync, int32_t *ofs_out, cudaStream_t s)
{
    dsm_launch_pool_select(d, frame, upper, 0, 0, DSM_REC_INDEX, holes, blkcnt, blkofs, nsel, s, DSM_SEL_PDL);
    // Sized by the fill (K <= S), not by `upper`, which can be far above the pool size: in the common frame there is no
    // tail and every further 1024-thread CTA only waits for a free SM next to the other stream's kernels.  A long tail
    // (after a large retire) is worked through by these CTAs segment after segment.
    const int grid = (d.S + RC_SEG - 1) / RC_SEG;
    pdl_launch(k_pool_recycle, dim3(grid > RC_MIN_GRID ? grid : RC_MIN_GRID), dim3(RC_SEG), 0, s, d, frame, (const int *)nsel,
               (const int32_t *)holes, src, sync, ofs_out);
}
void dsm_launch_raw_cloud(const DsmDev &d, int frame, const DsmRawPose &pose, float4 *out, cudaStream_t s)
{
    dim3 grid((d.W + RAW_TILE - 1) / RAW_TILE, (d.H + RAW_TILE - 1) / RAW_TILE);
    k_raw_cloud<<<grid, 256, 0, s>>>(d, frame, pose, out);
}
void dsm_launch_superpixel_image(const DsmDev &d, int frame, uint8_t *out, cudaStream_t s)
{
    dim3 grid((d.W + SPI_SPAN - 1) / SPI_SPAN, (d.H + SPI_WARPS - 1) / SPI_WARPS);
    k_superpixel_image<<<grid, dim3(32, SPI_WARPS), 0, s>>>(d, frame, reinterpret_cast<uint32_t *>(out));
}
void dsm_launch_pool_transform(const DsmDev &d, int frame, int upper, const float *Wm_dev, cudaStream_t s)
{
    if (upper <= 0) return;
    k_pool_transform<<<(upper + XF_BLOCK - 1) / XF_BLOCK, XF_BLOCK, 0, s>>>(d, frame, Wm_dev);
}

// one frame's window step (see k_win_plan): `upper` >= pool size sizes the two pool passes; the compaction and the copy
// run on a fixed grid and take their sizes from the device
#define WIN_GRID 264
void dsm_launch_window_step(const DsmDev &d, const DsmWin &w, int upper, int nr, int na, cudaStream_t s)
{
    const int nblk = (upper + 255) / 256;
    if (na > 0) pdl_launch(k_win_plan, dim3(1), dim3(1024), 0, s, w);
    if (nr > 0 && nblk > 0) pdl_launch(k_win_count, dim3(nblk), dim3(256), 0, s, d, w);
    pdl_launch(k_win_commit, dim3(1), dim3(1024), 0, s, w, nr, na);
    if (nr > 0 && nblk > 0) pdl_launch(k_win_scatter, dim3(nblk), dim3(256), 0, s, d, w);
    if (na == 0) return;
    pdl_launch(k_win_copy, dim3(WIN_GRID), dim3(256), 0, s, d, w);
    pdl_launch(k_win_compact, dim3(WIN_GRID), dim3(DSM_WIN_CHUNK), 0, s, w);
    pdl_launch(k_win_finish, dim3(1), dim3(1024), 0, s, w);
}
void dsm_launch_inactive_transform(const DsmWin &w, int kf, const float *Wm_dev, cudaStream_t s)
{
    k_inactive_transform<<<WIN_GRID, 256, 0, s>>>(w, kf, Wm_dev);
}
void dsm_launch_cloud_mirror(const dsm_surfel_t *store, const int32_t *size_word, const int32_t *res, int upper, float4 *shadow,
                             float4 *mirror, int32_t *state, int32_t *header, cudaStream_t s)
{
    const int grid = store ? (upper + DSM_PUB_CHUNK - 1) / DSM_PUB_CHUNK : 1;
    k_cloud_mirror<<<grid > 1 ? grid : 1, DSM_PUB_CHUNK, 0, s>>>(store, size_word, res, shadow, mirror, state, header);
}
void dsm_launch_map_snapshot(const dsm_surfel_t *pool, const int32_t *res, int pool_upper, const dsm_surfel_t *store, const int4 *seg,
                             const int32_t *hdr, int store_upper, uint8_t *image, const DsmSnapLayout &lay, cudaStream_t s)
{
    const int pool_chunks = (pool_upper + SNAP_CHUNK - 1) / SNAP_CHUNK;
    const int pool_grid = pool_chunks > 1 ? pool_chunks : 1; // CTA 0 exists and writes the header
    const int store_grid = store ? (store_upper + SNAP_CHUNK - 1) / SNAP_CHUNK : 0;
    k_map_snapshot<<<pool_grid + store_grid, SNAP_CHUNK, 0, s>>>(pool, res, pool_grid, store, seg, hdr, image, lay);
}
void dsm_launch_map_drain(const uint8_t *image, uint8_t *host_dev, const DsmSnapLayout &lay, int ctas, cudaStream_t s)
{
    k_map_drain<<<ctas, DRAIN_BLOCK, 0, s>>>(image, host_dev, lay);
}
void dsm_launch_map_delta(const dsm_surfel_t *pool, const int32_t *res, int pool_upper, const dsm_surfel_t *store, const int4 *seg,
                          const int32_t *hdr, int store_upper, uint8_t *image, const DsmSnapLayout &lay, int pool_chunks, cudaStream_t s)
{
    static_assert(DSM_SNAP_CHUNK == SNAP_CHUNK && DSM_DELTA_WORDS <= 32, "the image's chunks and header line");
    const int pool_grid = std::max(dsm_snap_chunks(pool_upper), 1); // as k_map_snapshot's: CTA 0 exists
    const int store_grid = store ? dsm_snap_chunks(store_upper) : 0;
    k_map_delta<<<pool_grid + store_grid, SNAP_CHUNK, 0, s>>>(pool, res, pool_grid, store, seg, hdr, image, lay, pool_chunks);
}
void dsm_launch_map_drain_delta(const uint8_t *image, uint8_t *host_dev, const DsmSnapLayout &lay, int pool_chunks, int store_chunks,
                                int ctas, cudaStream_t s)
{
    k_map_drain_delta<<<ctas, DRAIN_BLOCK, 0, s>>>(image, host_dev, lay, pool_chunks, store_chunks);
}
