// Host side of the C ABI declared in include/dsm.h: context, HBM allocation, the per-frame
// kernel schedule (mirrors FusionFunctions::fuse_initialize_map / generate_super_pixels,
// fusion_functions.cpp:30-83, :960-975) and the copies either side of it; the batch and stream paths, the resident pool
// and the inactive store, publishing, the distance field with its captured views, checkpoints and the debug readers.
// Each planner job's entry points live beside its kernels (dsm_field.cu for the queries, dsm_frontier.cu, ...).
// No CPU implementation of any phase lives here: if CUDA is unavailable every call fails.
#include "dsm_ctx.hpp"
#include "dsm_map_state.h"
#include <cmath>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <cstdint>
#include <algorithm>
#include <new>
#include <vector>

static const char *kKernelNames[DSM_NUM_KERNELS] = {"seed_init", "slic_assign_first", "slic_assign", "slic_gather", "slic_newton",
                                                     "plane_gather", "plane_solve", "surfel_fuse", "surfel_init", "repack"};

extern "C" int dsm_version(void) { return DSM_VERSION; }

extern "C" const char *dsm_strerror(int code)
{
    switch (code)
    {
    case DSM_OK: return "ok";
    case DSM_E_INVALID: return "invalid argument";
    case DSM_E_SHAPE: return "unsupported image shape (W%8 or H%8 > 4, or smaller than 24x24)";
    case DSM_E_NODEVICE: return "no usable CUDA device (sm_90 required)";
    case DSM_E_CUDA: return "CUDA error";
    case DSM_E_NOMEM: return "out of memory";
    case DSM_E_CAPACITY: return "surfel capacity exceeded";
    case DSM_E_STATE: return "invalid call sequence";
    case DSM_E_NCCL: return "NCCL error";
    case DSM_E_IO: return "file could not be opened or written";
    default: return "unknown error";
    }
}

extern "C" const char *dsm_last_error(const dsm_ctx *ctx) { return ctx ? ctx->err : "null context"; }
extern "C" const char *dsm_kernel_name(int id) { return (id >= 0 && id < DSM_NUM_KERNELS) ? kKernelNames[id] : "?"; }
extern "C" int dsm_num_seeds(const dsm_ctx *ctx) { return ctx ? ctx->d.S : DSM_E_INVALID; }

extern "C" void dsm_destroy(dsm_ctx *ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    ctx->ckpt.reset(); // a pending checkpoint is written first, then its thread ends
    dsm_comm_destroy(ctx);
    // an asynchronous batch may still be in flight on any of the context's streams: drain them before the buffers go
    for (auto &s : ctx->own.streams) cudaStreamSynchronize(s.get());
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    delete ctx; // releases every buffer, stream, event and captured graph the context owns
}

// TMA descriptors for the tile kernels: each per-pixel array as a [B][H][Wp] tensor, box = one 8x4-seed tile plus
// halo (DSM_TILE_W x DSM_TILE_H elements; out-of-image parts of a box are zero-filled by the copy engine).
// cuTensorMapEncodeTiled is a driver entry point; it is resolved through the runtime so the library keeps linking
// against cudart only.
// smallest float >= c: (double)x < c  <=>  x < ceil_float(c) for every float x
static float ceil_float(double c)
{
    float f = (float)c;
    if ((double)f < c) f = nextafterf(f, INFINITY);
    return f;
}
static void apply_constants(DsmDev &d, const dsm_constants &k)
{
    d.huber = k.huber_range;
    d.huber_hi = ceil_float(k.huber_range);
    d.baseline = k.baseline;
    d.disparity_error = k.disparity_error;
    d.min_tolerate_diff = k.min_tolerate_diff;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static int make_tile_maps(dsm_ctx *ctx)
{
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    if (!fn || qres != cudaDriverEntryPointSuccess)
    {
        snprintf(ctx->err, sizeof(ctx->err), "cuTensorMapEncodeTiled is not available in this driver");
        return DSM_E_CUDA;
    }
    PFN_encodeTiled enc = (PFN_encodeTiled)fn;
    const DsmDev &d = ctx->d;
    struct
    {
        CUtensorMap *map;
        void *base;
        CUtensorMapDataType type;
        unsigned esize, boxw;
    } specs[3] = {{&ctx->maps.cod, d.code, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, DSM_TILE_GW},
                  {&ctx->maps.dep, ctx->depth, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, DSM_TILE_W},
                  {&ctx->maps.gry, ctx->gray, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, DSM_TILE_GW}};
    for (auto &sp : specs)
    {
        const cuuint64_t dims[3] = {(cuuint64_t)d.Wp, (cuuint64_t)d.H, (cuuint64_t)d.B};
        const cuuint64_t strides[2] = {(cuuint64_t)d.Wp * sp.esize, (cuuint64_t)d.px_stride * sp.esize}; // bytes, multiples of 16 (Wp % 16 == 0)
        const cuuint32_t box[3] = {sp.boxw, DSM_TILE_H, 1};
        const cuuint32_t estr[3] = {1, 1, 1};
        const CUresult r = enc(sp.map, sp.type, 3, sp.base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS)
        {
            snprintf(ctx->err, sizeof(ctx->err), "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
            return DSM_E_CUDA;
        }
    }
    return DSM_OK;
}

extern "C" int dsm_create(const dsm_params *params, int device, void *cuda_stream, dsm_ctx **out)
{
    if (!params || !out) return DSM_E_INVALID;
    *out = nullptr;
    const int W = params->width, H = params->height;
    if (params->max_batch < 1 || params->max_local_surfels < 0) return DSM_E_INVALID;
    if (W < 3 * DSM_SP || H < 3 * DSM_SP || W % DSM_SP > 4 || H % DSM_SP > 4) return DSM_E_SHAPE;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) return DSM_E_NODEVICE;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return DSM_E_NODEVICE;
    if (prop.major != 9 || prop.minor != 0) return DSM_E_NODEVICE; // the only code in this library is sm_90a SASS
    if (cudaSetDevice(device) != cudaSuccess) return DSM_E_NODEVICE;

    dsm_ctx *ctx = new (std::nothrow) dsm_ctx();
    if (!ctx) return DSM_E_NOMEM;
    ctx->p = *params;
    ctx->device = device;
    {
        const char *e = getenv("DSM_GRAPHS");
        ctx->use_graphs = !(e && e[0] == '0');
    }
    ctx->stream = (cudaStream_t)cuda_stream;
    if (!ctx->stream && ctx->own.stream(&ctx->stream) != cudaSuccess)
    {
        delete ctx;
        return DSM_E_CUDA;
    }
    const int B = params->max_batch;
    const int Wp = (W + 15) / 16 * 16;
    const int spw = W / DSM_SP, sph = H / DSM_SP, S = spw * sph;
    const size_t px = (size_t)H * Wp;
    DsmDev &d = ctx->d;
    d.W = W, d.H = H, d.Wp = Wp, d.spw = spw, d.sph = sph, d.S = S, d.B = B;
    d.Sp = (S + 31) / 32 * 32;
    d.fx = params->fx, d.fy = params->fy, d.cx = params->cx, d.cy = params->cy;
    d.fuse_far = params->fuse_far, d.fuse_near = params->fuse_near;
    d.camera_f = (float)((fabs((double)params->fx) + fabs((double)params->fy)) / 2.0); // (:250)
    {
        const dsm_constants drive = DSM_CONSTANTS_DRIVE;
        apply_constants(d, drive);
    }
    d.px_stride = px;
    const size_t npool = (size_t)(params->max_local_surfels > 0 ? params->max_local_surfels : 1);
    cudaError_t e = cudaSuccess;
    // +64 bytes/elements of slack so the 16-byte vector accesses on the last pitched row stay in bounds
#define ALLOC(ptr, n)                        \
    if (e == cudaSuccess) e = ctx->own.device(&(ptr), (size_t)(n), true)
    ALLOC(ctx->gray, B * px + 64);
    ALLOC(ctx->depth, B * px + 64);
    ALLOC(d.labels, B * px + 64);
    ALLOC(d.seed, (size_t)B * S);
    ALLOC(d.inv_md, (size_t)B * S);
    ALLOC(d.invd, B * px + 64);
    ALLOC(d.code, B * px + 64);
    ALLOC(d.seed_hl, (size_t)B * S);
    ALLOC(d.done, (size_t)B);
    ALLOC(d.hardq, (size_t)B * S);
    ALLOC(d.nhard, (size_t)B);
    ALLOC(d.hrec, (size_t)B * S * 24);
    ALLOC(d.tstable, (size_t)B * S);
    ALLOC(d.und, (size_t)B * S);
    ALLOC(d.dlist, (size_t)B * S * 232);
    ALLOC(d.errflag, (size_t)B);
    ALLOC(d.qlist, (size_t)B * S * 3 * 232);
    ALLOC(d.pfsum, (size_t)B * S * 2);
    ALLOC(d.plane, (size_t)B * S * 3);
    ALLOC(d.fused, (size_t)B * S);
    ALLOC(d.list, B * px);
    ALLOC(d.nlist, (size_t)B);
    ALLOC(d.pool, npool);
    ALLOC(ctx->pool_snap, npool);
    ALLOC(ctx->poolofs, (size_t)B + 1);
    ALLOC(d.newsurf, (size_t)B * S);
    ALLOC(d.nnew, (size_t)B);
    ALLOC(ctx->pose, (size_t)B * 16);
    ALLOC(ctx->ipose, (size_t)B * 16);
    ALLOC(ctx->refidx, (size_t)B);
    ALLOC(ctx->seed_export, (size_t)S);
    ALLOC(ctx->kx, (size_t)Wp + 16);
    ALLOC(ctx->ky, (size_t)H + 16);
    ALLOC(ctx->gray_packed, (size_t)B * H * W + 64);
    ALLOC(ctx->depth_packed, (size_t)B * H * W + 64);
    ALLOC(ctx->blkcnt, npool / 256 + 64);
    ALLOC(ctx->blkofs, npool / 256 + 64);
    ALLOC(ctx->nsel, 1);
    ALLOC(ctx->holes, npool);
    ALLOC(ctx->rc_src, npool);
    ALLOC(ctx->rc_sync, dsm_recycle_sync_len((int)npool));
    ALLOC(ctx->wmat, 16);
    ALLOC(ctx->res_ofs, 4);
    ALLOC(ctx->win_hdr, 4);
    ctx->win_len = (size_t)DSM_WIN_KEYS(B) + (size_t)2 * B * DSM_WINDOW_MAX_KEYS;
    ALLOC(ctx->d_win, 2 * ctx->win_len);
#undef ALLOC
    if (e == cudaSuccess) e = ctx->own.host(&ctx->h_pose, (size_t)2 * B * 32);
    if (e == cudaSuccess) e = ctx->own.host(&ctx->h_ofs, (size_t)B + 1);
    if (e == cudaSuccess) e = ctx->own.host(&ctx->h_ref, (size_t)2 * B);
    if (e == cudaSuccess) e = ctx->own.host(&ctx->h_win, 2 * ctx->win_len);
    if (e == cudaSuccess) e = ctx->own.host(&ctx->h_sync, 8);
    int least = 0, greatest = 0;
    if (e == cudaSuccess) e = cudaDeviceGetStreamPriorityRange(&least, &greatest);
    if (e == cudaSuccess) e = ctx->own.stream(&ctx->s_hi, greatest);
    if (e == cudaSuccess) e = ctx->own.stream(&ctx->s_h2d);
    if (e == cudaSuccess) e = ctx->own.stream(&ctx->s_d2h);
    for (cudaStream_t &s : ctx->s_comp)
        if (e == cudaSuccess) e = ctx->own.stream(&s);
    for (cudaEvent_t *ev : {&ctx->ev_start, &ctx->ev_fork, &ctx->ev_p2})
        if (e == cudaSuccess) e = ctx->own.event(ev);
    for (int i = 0; i < DSM_MAX_CHUNKS; i++)
        for (cudaEvent_t *ev : {&ctx->ev_join[i], &ctx->ev_h2d[i], &ctx->ev_done[i]})
            if (e == cudaSuccess) e = ctx->own.event(ev);
    for (int h = 0; h < 2; h++)
        for (cudaEvent_t *ev : {&ctx->half_h2d[h], &ctx->half_free[h]})
            if (e == cudaSuccess) e = ctx->own.event(ev);
    if (e == cudaSuccess)
    { // back-projection factor tables: the same float ops as back_project (fusion_functions.cpp:94-95)
        std::vector<float> hx((size_t)Wp + 16), hy((size_t)H + 16);
        for (int u = 0; u < Wp + 16; u++) hx[u] = ((float)u - params->cx) / params->fx;
        for (int v = 0; v < H + 16; v++) hy[v] = ((float)v - params->cy) / params->fy;
        e = cudaMemcpy(ctx->kx, hx.data(), hx.size() * sizeof(float), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(ctx->ky, hy.data(), hy.size() * sizeof(float), cudaMemcpyHostToDevice);
    }
    if (e != cudaSuccess)
    {
        dsm_destroy(ctx);
        return e == cudaErrorMemoryAllocation ? DSM_E_NOMEM : DSM_E_CUDA;
    }
    d.gray = ctx->gray;
    d.depth = ctx->depth;
    d.poolofs = ctx->poolofs;
    d.pose = ctx->pose;
    d.ipose = ctx->ipose;
    d.refidx = ctx->refidx;
    d.kx = ctx->kx;
    d.ky = ctx->ky;
    if (make_tile_maps(ctx) != DSM_OK || dsm_tile_setup() != 0)
    {
        dsm_destroy(ctx);
        return DSM_E_CUDA;
    }
    *out = ctx;
    return DSM_OK;
}

// general 4x4 float inverse (adjugate / determinant) of a column-major matrix: stands in for
// Eigen's `pose.inverse()` (fusion_functions.cpp:59); same formula as the oracle's Eigen stand-in.
static void inverse4f(const float *m, float *out)
{
    float inv[16];
    inv[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
    inv[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
    inv[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
    inv[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
    inv[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
    inv[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
    inv[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
    inv[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
    inv[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
    inv[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
    inv[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
    inv[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
    inv[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
    inv[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
    inv[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
    inv[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
    float det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12];
    float inv_det = 1.0f / det;
    for (int i = 0; i < 16; i++) out[i] = inv[i] * inv_det;
}

// ---- profiling helpers ----
static cudaEvent_t prof_event(dsm_ctx *ctx)
{
    if (!ctx->ev_free.empty())
    {
        cudaEvent_t e = ctx->ev_free.back();
        ctx->ev_free.pop_back();
        return e;
    }
    cudaEvent_t e = nullptr;
    ctx->own.event(&e, cudaEventDefault); // recycled through ev_free, released with the context
    ctx->own.take();                       // a failure leaves e null; the next call tries again
    return e;
}
struct ProfScope
{
    dsm_ctx *ctx;
    int id;
    cudaEvent_t e0, e1;
    bool on;
    cudaStream_t st;
    ProfScope(dsm_ctx *c, int k, cudaStream_t stream = nullptr) : ctx(c), id(k), on((c->prof_mask >> k) & 1u), st(stream ? stream : c->stream)
    {
        if (on)
        {
            e0 = prof_event(ctx);
            e1 = prof_event(ctx);
            cudaEventRecord(e0, st);
        }
    }
    ~ProfScope()
    {
        if (on)
        {
            cudaEventRecord(e1, st);
            ctx->prof_pending.push_back(ProfRec{id, e0, e1});
        }
    }
};

extern "C" int dsm_profile_enable(dsm_ctx *ctx, uint32_t mask)
{
    if (!ctx) return DSM_E_INVALID;
    ctx->prof_mask = mask;
    return DSM_OK;
}
static int prof_drain(dsm_ctx *ctx, bool accumulate)
{
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    for (auto &r : ctx->prof_pending)
    {
        if (accumulate)
        {
            float ms = 0.f;
            CK(cudaEventElapsedTime(&ms, r.e0, r.e1));
            ctx->prof_ms[r.id] += ms;
            ctx->prof_n[r.id] += 1;
        }
        ctx->ev_free.push_back(r.e0);
        ctx->ev_free.push_back(r.e1);
    }
    ctx->prof_pending.clear();
    return DSM_OK;
}
extern "C" int dsm_profile_reset(dsm_ctx *ctx)
{
    if (!ctx) return DSM_E_INVALID;
    int rc = prof_drain(ctx, false);
    memset(ctx->prof_ms, 0, sizeof(ctx->prof_ms));
    memset(ctx->prof_n, 0, sizeof(ctx->prof_n));
    return rc;
}
extern "C" int dsm_profile_read(dsm_ctx *ctx, float *ms_total, int32_t *launches)
{
    if (!ctx || !ms_total || !launches) return DSM_E_INVALID;
    int rc = prof_drain(ctx, true);
    if (rc != DSM_OK) return rc;
    memcpy(ms_total, ctx->prof_ms, sizeof(ctx->prof_ms));
    memcpy(launches, ctx->prof_n, sizeof(ctx->prof_n));
    return DSM_OK;
}

// ---- batch stages ----
// The per-frame tables of n frames: pose, its inverse and the reference index go to the pinned rows [row, row + n) of
// h_pose / h_ref, then to the device slots [slot, slot + n) of pose / ipose / refidx on `st` (pose and inverse are
// interleaved on the host: two strided copies).  The caller makes sure earlier copies out of these rows have completed.
static int stage_tables(dsm_ctx *ctx, size_t row, int slot, int n, const float *poses, const int32_t *ref, cudaStream_t st)
{
    float *hp = ctx->h_pose + row * 32;
    for (int b = 0; b < n; b++)
    {
        memcpy(hp + (size_t)b * 32, poses + (size_t)b * 16, 16 * sizeof(float));
        inverse4f(poses + (size_t)b * 16, hp + (size_t)b * 32 + 16);
        ctx->h_ref[row + b] = ref[b];
    }
    CK(cudaMemcpy2DAsync(ctx->pose + (size_t)slot * 16, 16 * sizeof(float), hp, 32 * sizeof(float), 16 * sizeof(float), n, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpy2DAsync(ctx->ipose + (size_t)slot * 16, 16 * sizeof(float), hp + 16, 32 * sizeof(float), 16 * sizeof(float), n, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->refidx + slot, ctx->h_ref + row, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    return DSM_OK;
}

// Batch-mode tables of frames [0, n) on the main stream (first pinned half): per-frame pool offsets `ofs`, validated.
static int upload_tables(dsm_ctx *ctx, int n, const int32_t *ref, const float *poses, const int32_t *ofs)
{
    if (ofs[0] != 0) return DSM_E_INVALID;
    int maxper = 0;
    for (int b = 0; b <= n; b++) ctx->h_ofs[b] = ofs[b];
    for (int b = 0; b < n; b++)
    {
        int c = ofs[b + 1] - ofs[b];
        if (c < 0) return DSM_E_INVALID;
        if (c > maxper) maxper = c;
    }
    if (ofs[n] > ctx->p.max_local_surfels) return DSM_E_CAPACITY;
    ctx->n_pool = ofs[n];
    ctx->d.max_pool_per_frame = maxper;
    CK(cudaMemcpyAsync(ctx->poolofs, ctx->h_ofs, ((size_t)n + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
    return stage_tables(ctx, 0, 0, n, poses, ref, ctx->stream);
}

// The images of n frames, rows gray_pitch / depth_pitch bytes apart, into the packed staging from frame slot `slot` on
// `st`: packed rows in one contiguous copy per array, padded rows in one 2-D copy.  k_repack then lays them out in the
// pitched planes, the same for both.
static int stage_images(dsm_ctx *ctx, int slot, int n, const uint8_t *gray, size_t gray_pitch, const float *depth,
                        size_t depth_pitch, cudaStream_t st)
{
    const size_t W = ctx->p.width, rows = (size_t)n * ctx->p.height, row0 = (size_t)slot * ctx->p.height;
    uint8_t *gp = ctx->gray_packed + row0 * W;
    float *dp = ctx->depth_packed + row0 * W;
    if (gray_pitch == W)
        CK(cudaMemcpyAsync(gp, gray, rows * W, cudaMemcpyHostToDevice, st));
    else
        CK(cudaMemcpy2DAsync(gp, W, gray, gray_pitch, W, rows, cudaMemcpyHostToDevice, st));
    if (depth_pitch == W * 4)
        CK(cudaMemcpyAsync(dp, depth, rows * W * 4, cudaMemcpyHostToDevice, st));
    else
        CK(cudaMemcpy2DAsync(dp, W * 4, depth, depth_pitch, W * 4, rows, cudaMemcpyHostToDevice, st));
    return DSM_OK;
}

// Launches of the schedule up to and including the plane fit: seed init, 3 x (assign, gather, Newton), plane gather, solve.
static const int kPlaneFitSteps = 12;
// the schedule enqueued now runs at least through the plane fit (dsm_debug_stop_after does not cut it short before)
static bool schedule_fits(const dsm_ctx *ctx) { return ctx->stop_after <= 0 || ctx->stop_after >= kPlaneFitSteps; }

// The frames the context holds: slots [slot0, slot0 + n) hold the images of the latest call that took images, and the
// batch calls' frames are [0, nb).  `ran`: their schedule has been enqueued (through the plane fit unless
// dsm_debug_stop_after cuts it).
static void hold_frames(dsm_ctx *ctx, int slot0, int n, bool ran)
{
    ctx->nb = slot0 + n;
    ctx->uploaded = true;
    ctx->ran = ran;
    ctx->img_slot0 = slot0, ctx->img_n = n;
    ctx->img_fit = ran && schedule_fits(ctx);
}

extern "C" int dsm_batch_upload(dsm_ctx *ctx, int n, const int32_t *ref, const uint8_t *gray, const float *depth,
                                const float *poses, const dsm_surfel_t *local, const int32_t *ofs)
{
    if (!ctx || !ref || !gray || !depth || !poses || !ofs) return DSM_E_INVALID;
    if (n < 1 || n > ctx->p.max_batch) return DSM_E_INVALID;
    if (ofs[n] > 0 && !local) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    // the pinned tables are reused: make sure the previous batch's copies have drained
    CK(cudaStreamSynchronize(ctx->stream));
    int rc = upload_tables(ctx, n, ref, poses, ofs);
    if (rc != DSM_OK) return rc;
    rc = stage_images(ctx, 0, n, gray, (size_t)ctx->p.width, depth, (size_t)ctx->p.width * 4, ctx->stream);
    if (rc != DSM_OK) return rc;
    {
        DsmDev d = ctx->d;
        d.frame0 = 0;
        ProfScope p(ctx, DSM_K_REPACK);
        dsm_launch_repack(d, n, ctx->gray_packed, ctx->depth_packed, ctx->stream);
    }
    if (ctx->n_pool > 0)
    {
        CK(cudaMemcpyAsync(ctx->d.pool, local, (size_t)ctx->n_pool * sizeof(dsm_surfel_t), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(ctx->pool_snap, ctx->d.pool, (size_t)ctx->n_pool * sizeof(dsm_surfel_t), cudaMemcpyDeviceToDevice, ctx->stream));
    }
    hold_frames(ctx, 0, n, false);
    ctx->res_active = false;
    return DSM_OK;
}

extern "C" int dsm_batch_restore_pool(dsm_ctx *ctx)
{
    if (!ctx) return DSM_E_INVALID;
    if (!ctx->uploaded) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    if (ctx->n_pool > 0)
        CK(cudaMemcpyAsync(ctx->d.pool, ctx->pool_snap, (size_t)ctx->n_pool * sizeof(dsm_surfel_t), cudaMemcpyDeviceToDevice, ctx->stream));
    return DSM_OK;
}

// The per-frame schedule: generate_super_pixels (:960-975) then fuse (:58-71) then initialise (:79), enqueued for the
// frame slots [d.frame0, d.frame0 + nb) of the view `d` (its pool, poolofs and max_pool_per_frame).
// phase bit 0: the pose- and pool-independent part (superpixels, pixel normals, plane fit); bit 1: fuse + initialise.
static int launch_schedule(dsm_ctx *ctx, const DsmDev &d, int nb, cudaStream_t st, int phase)
{
    int budget = ctx->stop_after > 0 ? ctx->stop_after : 1 << 30;
#define STEP(ID, CALL)                  \
    if (budget-- > 0)                   \
    {                                   \
        ProfScope p(ctx, ID, st);       \
        CALL;                           \
    }
    if (phase & 1)
    { // generate_super_pixels (:960-975): seed init, 3 x (assign [+ stable relaxation], gather, Newton), plane fit
        STEP(DSM_K_SEED_INIT, dsm_launch_seed_init(d, nb, st));
        for (int it = 0; it < 3; it++) // ITERATION_NUM (fusion_functions.h:8)
        {
            STEP(it == 0 ? DSM_K_ASSIGN_FIRST : DSM_K_ASSIGN, dsm_launch_assign2(d, nb, it == 0, st));
            STEP(DSM_K_GATHER, dsm_launch_gather(d, ctx->maps, nb, st));
            STEP(DSM_K_NEWTON, dsm_launch_newton2(d, nb, st));
        }
        STEP(DSM_K_PLANE_GATHER, dsm_launch_plane_gather(d, ctx->maps, nb, st));
        STEP(DSM_K_PLANE_SOLVE, dsm_launch_gn_solve(d, nb, st));
    }
    if (phase & 2)
    {
        if (d.max_pool_per_frame > 0)
        {
            STEP(DSM_K_FUSE, dsm_launch_fuse(d, nb, st));
        }
        STEP(DSM_K_INIT_SURFELS, dsm_launch_init_surfels(d, nb, st));
    }
#undef STEP
    CK(cudaGetLastError());
    return DSM_OK;
}

// Enqueue the schedule for the view `v` (frames [v.frame0, v.frame0 + nf)).  Phase 2 (the resident stream's fuse /
// initialise on its pool) ends with the pool's fuse_map post-step (in place, slot for slot as the reference); phase 3
// (the batch calls) and phase 1 have none.
// The 14-18 launches are captured once per distinct parameter set into a CUDA graph and replayed: the
// per-launch CPU cost and inter-kernel gaps matter for single frames and small chunks.  Profiling
// (event pairs around kernels) and the debug kernel budget use plain launches.
static int enqueue_schedule(dsm_ctx *ctx, const DsmDev &v, int nf, cudaStream_t st, int phase = 3)
{
    // grids over the pool are sized from max_pool_per_frame rounded up to 4 Ki surfels (the kernels take the true
    // ranges from poolofs on the device, surplus blocks exit at once), so that callers whose pool size
    // changes a little from call to call keep hitting the same captured graph
    DsmDev d = v;
    if (d.max_pool_per_frame > 0) d.max_pool_per_frame = (d.max_pool_per_frame + 4095) & ~4095;
    auto plain = [&]() -> int
    {
        int rc = launch_schedule(ctx, d, nf, st, phase);
        if (rc != DSM_OK) return rc;
        if (phase == 2)
            dsm_launch_pool_recycle(d, d.frame0, d.max_pool_per_frame, ctx->blkcnt, ctx->blkofs, ctx->nsel, ctx->holes, ctx->rc_src,
                                    ctx->rc_sync, ctx->res_ofs, st);
        return DSM_OK;
    };
    if (!ctx->use_graphs || ctx->prof_mask != 0 || ctx->stop_after > 0) return plain();
    for (auto &g : ctx->graphs)
        if (g.f0 == d.frame0 && g.nf == nf && g.maxper == d.max_pool_per_frame && g.pool == d.pool && g.poolofs == d.poolofs &&
            g.gate == d.gate && g.phase == phase)
        {
            CK(cudaGraphLaunch(g.exec.get(), st));
            return DSM_OK;
        }
    cudaGraph_t graph = nullptr;
    if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) != cudaSuccess)
    {
        cudaGetLastError();
        return plain();
    }
    int rc = plain();
    cudaError_t ce = cudaStreamEndCapture(st, &graph);
    if (rc != DSM_OK || ce != cudaSuccess || !graph)
    {
        cudaGetLastError();
        if (graph) cudaGraphDestroy(graph);
        ctx->use_graphs = false; // capture is not possible in this environment: fall back to plain launches
        return rc != DSM_OK ? rc : plain();
    }
    cudaGraphExec_t exec = nullptr;
    ce = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess || !exec)
    {
        cudaGetLastError();
        ctx->use_graphs = false;
        return plain();
    }
    if (ctx->graphs.size() >= 64) ctx->graphs.erase(ctx->graphs.begin()); // bounded cache
    ctx->graphs.push_back(GraphEntry{d.frame0, nf, d.max_pool_per_frame, phase, d.pool, d.poolofs, d.gate, GraphExecPtr(exec)});
    CK(cudaGraphLaunch(exec, st));
    return DSM_OK;
}

// Frames [0, n) in `parts` even parts, part i on s_comp[i], forked from the main stream and joined back into it (a
// single part runs on the main stream itself).  part(i, f0, nf, st) enqueues part i, frames [f0, f0 + nf), on st.
template <typename Part>
static int run_parts(dsm_ctx *ctx, int n, int parts, Part part)
{
    if (parts <= 1) return part(0, 0, n, ctx->stream);
    CK(cudaEventRecord(ctx->ev_fork, ctx->stream));
    for (int i = 0, f0 = 0; i < parts; i++)
    {
        const int nf = (n - f0 + (parts - i) - 1) / (parts - i);
        CK(cudaStreamWaitEvent(ctx->s_comp[i], ctx->ev_fork, 0));
        const int rc = part(i, f0, nf, ctx->s_comp[i]);
        if (rc != DSM_OK) return rc;
        CK(cudaEventRecord(ctx->ev_join[i], ctx->s_comp[i]));
        CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_join[i], 0));
        f0 += nf;
    }
    return DSM_OK;
}

extern "C" int dsm_batch_run(dsm_ctx *ctx)
{
    if (!ctx) return DSM_E_INVALID;
    if (!ctx->uploaded) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    // The frames of a batch are independent, and most kernels of the schedule are issue- or latency-bound rather than
    // DRAM-bound: two sub-batches run CONCURRENTLY on two streams fill each other's tails and stalls.  With two resident
    // contexts alternating (bench.py) the gain on an H100 at 400 W is small: 1.150 / 1.163 ms per 32-frame step with two
    // sub-batches against 1.153 / 1.168 ms with one (two runs each); three or four sub-batches were slower.
    const int parts = (ctx->stop_after > 0 || ctx->nb < 8) ? 1 : (ctx->run_split < ctx->nb ? ctx->run_split : ctx->nb);
    const int rc = run_parts(ctx, ctx->nb, parts, [&](int, int f0, int nf, cudaStream_t st) {
        DsmDev v = ctx->d; // batch view: per-frame pool slices at poolofs, frames from slot 0
        v.frame0 = f0;
        return enqueue_schedule(ctx, v, nf, st);
    });
    if (rc != DSM_OK) return rc;
    hold_frames(ctx, ctx->img_slot0, ctx->img_n, true); // the same frames (nb == img_slot0 + img_n), now run
    return DSM_OK;
}

extern "C" int dsm_set_concurrency(dsm_ctx *ctx, int sub_batches)
{
    if (!ctx || sub_batches < 1 || sub_batches > 4) return DSM_E_INVALID;
    ctx->run_split = sub_batches;
    return DSM_OK;
}

extern "C" int dsm_set_constants(dsm_ctx *ctx, const dsm_constants *k)
{
    if (!ctx || !k) return DSM_E_INVALID;
    if (!(k->huber_range > 0.0) || !(k->baseline > 0.0) || !(k->disparity_error > 0.0) || !(k->min_tolerate_diff >= 0.0)) return DSM_E_INVALID;
    if (ctx->in_flight) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->graphs.clear(); // captured schedules embed the kernel parameters
    apply_constants(ctx->d, *k);
    dsm_checkpoint_map_replaced(ctx); // an incremental checkpoint's base carries the constants
    return DSM_OK;
}

extern "C" int dsm_debug_stop_after(dsm_ctx *ctx, int n)
{
    if (!ctx) return DSM_E_INVALID;
    ctx->stop_after = n;
    return DSM_OK;
}

extern "C" int dsm_debug_invariant_violations(dsm_ctx *ctx, int *count)
{
    if (!ctx || !count) return DSM_E_INVALID;
    if (!ctx->ran) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    std::vector<int32_t> h((size_t)ctx->nb);
    CK(cudaMemcpyAsync(h.data(), ctx->d.errflag, (size_t)ctx->nb * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    int c = 0;
    for (int v : h) c += v;
    *count = c;
    return DSM_OK;
}

extern "C" int dsm_batch_download(dsm_ctx *ctx, dsm_surfel_t *local_out, dsm_surfel_t *new_out, int32_t *n_new)
{
    if (!ctx) return DSM_E_INVALID;
    if (!ctx->ran) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    if (local_out && ctx->n_pool > 0)
        CK(cudaMemcpyAsync(local_out, ctx->d.pool, (size_t)ctx->n_pool * sizeof(dsm_surfel_t), cudaMemcpyDeviceToHost, ctx->stream));
    if (new_out)
        CK(cudaMemcpyAsync(new_out, ctx->d.newsurf, (size_t)ctx->nb * ctx->d.S * sizeof(dsm_surfel_t), cudaMemcpyDeviceToHost, ctx->stream));
    if (n_new)
        CK(cudaMemcpyAsync(n_new, ctx->d.nnew, (size_t)ctx->nb * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    return DSM_OK;
}

extern "C" int dsm_sync(dsm_ctx *ctx)
{
    if (!ctx) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    return DSM_OK;
}

// End-to-end batch call with host buffers (dsm_fuse_batch = dsm_fuse_batch_async + dsm_batch_wait).  The batch is cut into chunks of frames; chunk c's H2D
// (copy stream), kernels (compute stream) and D2H (second copy stream) overlap with the neighbouring
// chunks, so the call costs about max(PCIe time, kernel time) instead of their sum.  Host buffers
// should be pinned for the copies to be truly asynchronous (pageable memory works, staged by the driver).
extern "C" int dsm_batch_wait(dsm_ctx *ctx)
{
    if (!ctx) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->s_h2d));
    for (cudaStream_t s : ctx->s_comp) CK(cudaStreamSynchronize(s));
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaStreamSynchronize(ctx->s_d2h));
    CK(cudaGetLastError());
    ctx->in_flight = false;
    return DSM_OK;
}

// an in-flight dsm_fuse_batch_async batch copies and runs on the context's side streams: finish it first
static int finish_batch(dsm_ctx *ctx) { return ctx->in_flight ? dsm_batch_wait(ctx) : DSM_OK; }

// dsm_fuse_batch_async, with rows of the n images gray_pitch / depth_pitch bytes apart
static int fuse_batch_async(dsm_ctx *ctx, int n, const int32_t *ref, const uint8_t *gray, size_t gray_pitch, const float *depth,
                            size_t depth_pitch, const float *poses, dsm_surfel_t *local, const int32_t *ofs,
                            dsm_surfel_t *new_out, int32_t *n_new)
{
    if (!ctx || !ref || !gray || !depth || !poses || !ofs) return DSM_E_INVALID;
    if (n < 1 || n > ctx->p.max_batch) return DSM_E_INVALID;
    if (ofs[n] > 0 && !local) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    int rc = finish_batch(ctx); // one batch per context at a time
    if (rc != DSM_OK) return rc;
    CK(cudaStreamSynchronize(ctx->stream));
    rc = upload_tables(ctx, n, ref, poses, ofs); // small tables, on the main stream
    if (rc != DSM_OK) return rc;
    const int H = ctx->p.height, S = ctx->d.S;
    const size_t fpx = (size_t)H * ctx->p.width;
    // copies must not start before earlier work on the main stream (previous users of the buffers) is done
    CK(cudaEventRecord(ctx->ev_start, ctx->stream));
    CK(cudaStreamWaitEvent(ctx->s_h2d, ctx->ev_start, 0));
    CK(cudaStreamWaitEvent(ctx->s_d2h, ctx->ev_start, 0));
    // even chunks (a smaller first chunk was tried: no gain, the kernels of small chunks are less efficient); the kernels
    // of each chunk run on their own compute stream, so the latency-bound per-seed kernels of one chunk overlap the wide
    // kernels of its neighbours instead of leaving SMs idle
    const int nchunks = n >= 16 ? 4 : (n >= 4 ? 2 : 1);
    rc = run_parts(ctx, n, nchunks, [&](int c, int f0, int nf, cudaStream_t cs) {
        const int p0 = ofs[f0], p1 = ofs[f0 + nf];
        int maxper = 0;
        for (int b = f0; b < f0 + nf; b++) maxper = (ofs[b + 1] - ofs[b] > maxper) ? ofs[b + 1] - ofs[b] : maxper;
        // H2D of this chunk
        int r = stage_images(ctx, f0, nf, gray + (size_t)f0 * H * gray_pitch, gray_pitch,
                             (const float *)((const char *)depth + (size_t)f0 * H * depth_pitch), depth_pitch, ctx->s_h2d);
        if (r != DSM_OK) return r;
        if (p1 > p0)
            CK(cudaMemcpyAsync(ctx->d.pool + p0, local + p0, (size_t)(p1 - p0) * sizeof(dsm_surfel_t), cudaMemcpyHostToDevice, ctx->s_h2d));
        CK(cudaEventRecord(ctx->ev_h2d[c], ctx->s_h2d));
        CK(cudaStreamWaitEvent(cs, ctx->ev_h2d[c], 0));
        DsmDev v = ctx->d; // batch view of this chunk
        v.frame0 = f0;
        v.max_pool_per_frame = maxper;
        {
            ProfScope p(ctx, DSM_K_REPACK, cs);
            dsm_launch_repack(v, nf, ctx->gray_packed + (size_t)f0 * fpx, ctx->depth_packed + (size_t)f0 * fpx, cs);
        }
        r = enqueue_schedule(ctx, v, nf, cs);
        if (r != DSM_OK) return r;
        CK(cudaEventRecord(ctx->ev_done[c], cs));
        // D2H of this chunk
        CK(cudaStreamWaitEvent(ctx->s_d2h, ctx->ev_done[c], 0));
        if (p1 > p0)
            CK(cudaMemcpyAsync(local + p0, ctx->d.pool + p0, (size_t)(p1 - p0) * sizeof(dsm_surfel_t), cudaMemcpyDeviceToHost, ctx->s_d2h));
        if (new_out)
            CK(cudaMemcpyAsync(new_out + (size_t)f0 * S, ctx->d.newsurf + (size_t)f0 * S, (size_t)nf * S * sizeof(dsm_surfel_t), cudaMemcpyDeviceToHost, ctx->s_d2h));
        if (n_new)
            CK(cudaMemcpyAsync(n_new + f0, ctx->d.nnew + f0, (size_t)nf * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->s_d2h));
        return DSM_OK;
    });
    if (rc != DSM_OK) return rc;
    hold_frames(ctx, 0, n, true);
    ctx->in_flight = true;
    ctx->res_active = false; // the pool buffer now holds this batch's slices: a resident pool (if any) is gone
    CK(cudaGetLastError());
    return DSM_OK;
}

extern "C" int dsm_fuse_batch_async(dsm_ctx *ctx, int n, const int32_t *ref, const uint8_t *gray, const float *depth,
                                    const float *poses, dsm_surfel_t *local, const int32_t *ofs,
                                    dsm_surfel_t *new_out, int32_t *n_new)
{
    if (!ctx) return DSM_E_INVALID;
    return fuse_batch_async(ctx, n, ref, gray, (size_t)ctx->p.width, depth, (size_t)ctx->p.width * 4, poses, local, ofs,
                            new_out, n_new);
}

extern "C" int dsm_fuse_batch(dsm_ctx *ctx, int n, const int32_t *ref, const uint8_t *gray, const float *depth,
                              const float *poses, dsm_surfel_t *local, const int32_t *ofs,
                              dsm_surfel_t *new_out, int32_t *n_new)
{
    int rc = dsm_fuse_batch_async(ctx, n, ref, gray, depth, poses, local, ofs, new_out, n_new);
    if (rc != DSM_OK) return rc;
    return dsm_batch_wait(ctx);
}

// one frame of fuse_batch_async with the caller's row pitches, then its wait
extern "C" int dsm_fuse_frame(dsm_ctx *ctx, int ref_idx, const uint8_t *gray, size_t gray_pitch,
                              const float *depth, size_t depth_pitch, const float pose[16],
                              dsm_surfel_t *local, int n_local, dsm_surfel_t *new_out, int new_cap, int *n_new)
{
    if (!ctx || !gray || !depth || !pose || n_local < 0 || new_cap < 0 || !n_new) return DSM_E_INVALID;
    if (new_cap > 0 && !new_out) return DSM_E_INVALID;
    if (gray_pitch < (size_t)ctx->p.width || depth_pitch < (size_t)ctx->p.width * 4) return DSM_E_INVALID;
    const int32_t ref = ref_idx, ofs[2] = {0, n_local};
    int32_t cnt = 0;
    int rc = fuse_batch_async(ctx, 1, &ref, gray, gray_pitch, depth, depth_pitch, pose, local, ofs, nullptr, &cnt);
    if (rc == DSM_OK) rc = dsm_batch_wait(ctx);
    if (rc != DSM_OK) return rc;
    *n_new = cnt;
    const int ncopy = cnt < new_cap ? cnt : new_cap;
    if (ncopy > 0)
    {
        CK(cudaMemcpyAsync(new_out, ctx->d.newsurf, (size_t)ncopy * sizeof(dsm_surfel_t), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    return DSM_OK;
}

// ---- GPU-resident pool (stream mode) ----
// The resident pool is described by res_ofs = {0, n} on the device; its frames run in the frame slots of the staging
// half their call uses (stream_run).
// The view of frame slot `slot`: grids over the pool are sized from its upper bound rounded up to 64 Ki surfels and
// clamped to the capacity, so that the captured graph stays valid while the pool grows (surplus blocks exit at once:
// the kernels read the true range from the device).
static DsmDev resident_view(dsm_ctx *ctx, int slot)
{
    DsmDev d = ctx->d;
    d.frame0 = slot;
    d.poolofs = ctx->res_ofs - slot; // kernels read poolofs[b], poolofs[b+1] with b == slot
    const int upq = (ctx->res_upper + 65535) / 65536 * 65536;
    d.max_pool_per_frame = upq < ctx->p.max_local_surfels ? upq : ctx->p.max_local_surfels;
    // the error word exists for dsm_fuse_stream_window only: a context that has never run it reads no gate
    d.gate = ctx->win_tag > 0 ? ctx->res_ofs + 2 : nullptr;
    return d;
}

// The synchronisation point of the device-side state: after a window step, the pool size, the store size, the segment
// table and the error word are known only on the device.  Waits for the stream, refreshes the host bounds and the
// segment mirror, and reports (and clears) a rejected frame as DSM_E_CAPACITY.  A no-op when no window step has run
// since the last one.  The first nseg_hint table entries are read with the header; only a longer table takes a second
// round trip.
static int res_sync(dsm_ctx *ctx, int nseg_hint = 0)
{
    if (!ctx->win_pending) return DSM_OK;
    CK(cudaSetDevice(ctx->device));
    int32_t *h = ctx->h_sync, *hdr = ctx->h_sync + 4; // pinned, so these copies do not wait for the stream one by one
    InactStore *store = ctx->inact.get();
    std::vector<int4> t(store ? (size_t)std::min(nseg_hint, store->cap) : 0);
    CK(cudaMemcpyAsync(h, ctx->res_ofs, 4 * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(hdr, ctx->win_hdr, 4 * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    if (!t.empty()) CK(cudaMemcpyAsync(t.data(), store->seg, t.size() * sizeof(int4), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    if (store)
    {
        const size_t read = t.size();
        t.resize((size_t)hdr[1]);
        if (t.size() > read)
        {
            CK(cudaMemcpyAsync(t.data() + read, store->seg + read, (t.size() - read) * sizeof(int4), cudaMemcpyDeviceToHost, ctx->stream));
            CK(cudaStreamSynchronize(ctx->stream));
        }
        store->segs.clear();
        for (const int4 &g : t) store->segs.push_back(InactStore::Seg{g.x, g.y, g.z});
        store->size = store->upper = hdr[0];
    }
    ctx->res_upper = h[1];
    ctx->win_pending = false;
    if (h[2] == 0) return DSM_OK;
    CK(cudaMemsetAsync(ctx->res_ofs + 2, 0, 2 * sizeof(int32_t), ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    snprintf(ctx->err, sizeof(ctx->err), "dsm_fuse_stream_window: frame %d of a call did not fit the pool or the store; "
             "the map holds the frames before it", h[3]);
    return DSM_E_CAPACITY;
}

// the device-side view of the store and the window tables; `half` selects the staging half of the window lists, S is
// the room for new surfels the capacity check keeps in the pool (a fused frame's seeds; 0 for a step without a fuse)
static DsmWin window_view(dsm_ctx *ctx, int half, int t, int S)
{
    DsmWin w{};
    w.tab = ctx->d_win + (size_t)half * ctx->win_len;
    w.t = t, w.B = ctx->p.max_batch;
    w.hdr = ctx->win_hdr;
    w.res = ctx->res_ofs;
    w.pool_cap = ctx->p.max_local_surfels;
    w.S = S;
    if (const InactStore *s = ctx->inact.get())
    {
        w.store = s->surfels, w.seg = s->seg, w.blk = s->blk, w.sync = s->sync;
        w.blk_stride = s->blk_stride, w.store_cap = s->cap;
    }
    return w;
}

// The per-frame window lists of dsm_fuse_stream_window (a null offset array: empty lists)
struct WinLists
{
    const int32_t *rk, *ro, *ak, *ao;
};

// The lists of n frames into staging half `half` (table layout: DsmWin), copied on `st` like the pose tables: the
// device reads them when the window step runs, so a captured schedule never depends on their contents
static int stage_window(dsm_ctx *ctx, int half, int n, const WinLists &w, int tag, cudaStream_t st)
{
    const int B = ctx->p.max_batch, KR = DSM_WIN_KEYS(B);
    int32_t *h = ctx->h_win + (size_t)half * ctx->win_len;
    for (int t = 0; t <= n; t++)
    {
        h[t] = w.ro ? w.ro[t] - w.ro[0] : 0;
        h[B + 1 + t] = w.ao ? w.ao[t] - w.ao[0] : 0;
    }
    const int nr = h[n], na = h[B + 1 + n];
    if (nr > 0) memcpy(h + KR, w.rk + w.ro[0], (size_t)nr * sizeof(int32_t));
    if (na > 0) memcpy(h + KR + nr, w.ak + w.ao[0], (size_t)na * sizeof(int32_t));
    h[2 * B + 2] = tag;
    h[2 * B + 3] = KR + nr;
    CK(cudaMemcpyAsync(ctx->d_win + (size_t)half * ctx->win_len, h, (size_t)(KR + nr + na) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    return DSM_OK;
}

// The entry of the calls on the resident pool and the inactive store, after their own argument checks: the state they
// need (`need`: NEED_POOL, NEED_STORE), then res_sync, then the device
enum { NEED_POOL = 1, NEED_STORE = 2 };
static int res_enter(dsm_ctx *ctx, int need)
{
    if (((need & NEED_POOL) && !ctx->res_active) || ((need & NEED_STORE) && !ctx->inact)) return DSM_E_STATE;
    const int rs = res_sync(ctx);
    if (rs != DSM_OK) return rs;
    CK(cudaSetDevice(ctx->device));
    return DSM_OK;
}

// res_ofs = {0, n} after the copies already on the stream; waits, so the caller's source buffers are free on return
static int set_pool_size(dsm_ctx *ctx, int n)
{
    ctx->h_ofs[0] = 0;
    ctx->h_ofs[1] = n;
    CK(cudaMemcpyAsync(ctx->res_ofs, ctx->h_ofs, 2 * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->res_upper = n;
    return DSM_OK;
}

// The ordered selection (mode / key as pool_pred) over the range of view d into pool_snap, and its first min(cap, n)
// records to `out`, n being its count.  With n_out, n is read back into *n_out and the call waits for the copy.  Without
// it, the caller knows that all `cap` records of the range are selected, and nothing waits.  Mode 1 (retire) flags what
// it selects dead, so it scatters only after the count has been checked against cap: DSM_E_CAPACITY leaves the pool as
// it was.
static int select_out(dsm_ctx *ctx, const DsmDev &d, int upper, int mode, int key, DsmRec rec, void *out, int cap, int *n_out)
{
    const bool retire = mode == 1;
    dsm_launch_pool_select(d, 0, upper, mode, key, rec, retire ? nullptr : ctx->pool_snap, ctx->blkcnt, ctx->blkofs, ctx->nsel, ctx->stream);
    int n = cap;
    if (n_out)
    {
        CK(cudaMemcpyAsync(&n, ctx->nsel, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        CK(cudaGetLastError());
        *n_out = n;
    }
    if (retire)
    {
        if (n > cap) return DSM_E_CAPACITY; // call again with cap >= *n_out
        dsm_launch_pool_select(d, 0, upper, mode, key, rec, ctx->pool_snap, ctx->blkcnt, ctx->blkofs, ctx->nsel, ctx->stream,
                               DSM_SEL_SCATTER_ONLY);
        CK(cudaGetLastError());
    }
    const int c = std::min(n, cap);
    if (c <= 0) return DSM_OK;
    const size_t bytes = (size_t)c * (rec == DSM_REC_POINT ? sizeof(dsm_point_t) : sizeof(dsm_surfel_t));
    CK(cudaMemcpyAsync(out, ctx->pool_snap, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    if (n_out) CK(cudaStreamSynchronize(ctx->stream));
    return DSM_OK;
}

extern "C" int dsm_pool_upload(dsm_ctx *ctx, const dsm_surfel_t *local, int n)
{
    if (!ctx || n < 0 || (n > 0 && !local)) return DSM_E_INVALID;
    if (n > ctx->p.max_local_surfels) return DSM_E_CAPACITY;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->s_h2d));
    const int rs = res_sync(ctx); // the new pool replaces whatever a rejected windowed frame left: its error is dropped
    if (rs != DSM_OK && rs != DSM_E_CAPACITY) return rs;
    CK(cudaStreamSynchronize(ctx->stream));
    if (n > 0) CK(cudaMemcpyAsync(ctx->d.pool, local, (size_t)n * sizeof(dsm_surfel_t), cudaMemcpyHostToDevice, ctx->stream));
    const int rc = set_pool_size(ctx, n); // `local` may be pageable / reused by the caller
    if (rc != DSM_OK) return rc;
    ctx->res_active = true;
    ctx->n_pool = n;
    return DSM_OK;
}

extern "C" int dsm_pool_size(dsm_ctx *ctx, int *n)
{
    if (!ctx || !n) return DSM_E_INVALID;
    const int rc = res_enter(ctx, NEED_POOL);
    if (rc != DSM_OK) return rc;
    int32_t h[2] = {0, 0};
    CK(cudaMemcpyAsync(h, ctx->res_ofs, 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    *n = h[1];
    ctx->res_upper = h[1];
    return DSM_OK;
}

extern "C" int dsm_pool_download(dsm_ctx *ctx, dsm_surfel_t *out, int cap, int *n)
{
    if (!ctx || !n || cap < 0 || (cap > 0 && !out)) return DSM_E_INVALID;
    int rc = dsm_pool_size(ctx, n);
    if (rc != DSM_OK) return rc;
    const int c = *n < cap ? *n : cap;
    if (c > 0)
    {
        CK(cudaMemcpyAsync(out, ctx->d.pool, (size_t)c * sizeof(dsm_surfel_t), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    return DSM_OK;
}

// retire (mode 1) and the publish_*_pointcloud / save_cloud / save_mesh filters (mode 2) on the resident pool (see
// include/dsm.h), ordered through select_out
static int pool_select(dsm_ctx *ctx, int mode, int key, DsmRec rec, void *out, int cap, int *n_out)
{
    if (!ctx || !n_out || cap < 0 || (cap > 0 && !out)) return DSM_E_INVALID;
    const int rc = res_enter(ctx, NEED_POOL);
    return rc != DSM_OK ? rc : select_out(ctx, resident_view(ctx, 0), ctx->res_upper, mode, key, rec, out, cap, n_out);
}
extern "C" int dsm_pool_retire(dsm_ctx *ctx, int kf, dsm_surfel_t *out, int cap, int *n_out)
{
    return pool_select(ctx, 1, kf, DSM_REC_SURFEL, out, cap, n_out);
}
extern "C" int dsm_pool_export_cloud(dsm_ctx *ctx, int min_update_times, dsm_point_t *out, int cap, int *n_out)
{
    return pool_select(ctx, 2, min_update_times, DSM_REC_POINT, out, cap, n_out);
}
extern "C" int dsm_pool_export_surfels(dsm_ctx *ctx, int min_update_times, dsm_surfel_t *out, int cap, int *n_out)
{
    return pool_select(ctx, 2, min_update_times, DSM_REC_SURFEL, out, cap, n_out);
}

extern "C" int dsm_pool_append(dsm_ctx *ctx, const dsm_surfel_t *surfels, int n)
{
    if (!ctx || n < 0 || (n > 0 && !surfels)) return DSM_E_INVALID;
    int cur = 0;
    int rc = dsm_pool_size(ctx, &cur);
    if (rc != DSM_OK) return rc;
    if (cur + n > ctx->p.max_local_surfels) return DSM_E_CAPACITY;
    if (n == 0) return DSM_OK;
    CK(cudaMemcpyAsync(ctx->d.pool + cur, surfels, (size_t)n * sizeof(dsm_surfel_t), cudaMemcpyHostToDevice, ctx->stream));
    return set_pool_size(ctx, cur + n);
}

extern "C" int dsm_pool_transform(dsm_ctx *ctx, const float Wm[16])
{
    if (!ctx || !Wm) return DSM_E_INVALID;
    if (!ctx->res_active) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(ctx->wmat, Wm, 16 * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    dsm_launch_pool_transform(resident_view(ctx, 0), 0, ctx->res_upper, ctx->wmat, ctx->stream);
    CK(cudaGetLastError());
    return DSM_OK;
}

// ---- inactive store (DESIGN.md section 8.2) ----
static DsmDev inactive_view(dsm_ctx *ctx)
{
    DsmDev d = ctx->d;
    d.frame0 = 0;
    d.pool = ctx->inact->surfels;
    d.poolofs = ctx->inact->range;
    return d;
}

// dsm_publish_*: the store's part of a publishing context, the shadow of the inactive cloud and its pinned host mirror
// (what an earlier, failed attempt allocated is kept and used)
static cudaError_t store_publish_alloc(InactStore &s)
{
    if (!s.shadow) s.own.device(&s.shadow, (size_t)s.cap);
    if (!s.mirror) s.own.mapped(&s.mirror, &s.mirror_dev, (size_t)s.cap);
    return s.own.take();
}
// k_cloud_mirror's state for a shadow that holds nothing: the next snapshot forwards the whole cloud.  Ordered on the
// context's stream, like the kernels that read it, and waited for (the source is on the stack).
static cudaError_t publish_state_reset(dsm_ctx *ctx)
{
    const int32_t fresh[4] = {0, INT32_MAX, 0, 0};
    const cudaError_t e = cudaMemcpyAsync(ctx->pub_state, fresh, sizeof(fresh), cudaMemcpyHostToDevice, ctx->stream);
    return e != cudaSuccess ? e : cudaStreamSynchronize(ctx->stream);
}

static cudaError_t checkpoint_images(dsm_ctx *ctx);

extern "C" int dsm_inactive_reserve(dsm_ctx *ctx, int max_inactive_surfels)
{
    if (!ctx || max_inactive_surfels < 1) return DSM_E_INVALID;
    if (ctx->pub_in_flight) return DSM_E_STATE; // the snapshot's inactive buffer goes with the old store
    if (ctx->field && ctx->field->in_flight) return DSM_E_STATE; // as does the store a field request reads
    if (ctx->ckpt && ctx->ckpt->pending) return DSM_E_STATE; // and the checkpoint's images are sized by it
    int rs = res_sync(ctx);
    if (rs != DSM_OK) return rs;
    if (ctx->inact && ctx->inact->size > 0) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->inact.reset(); // before the new store is allocated: the two need not fit at once
    auto s = std::make_unique<InactStore>();
    const int cap = max_inactive_surfels, npool = std::max(ctx->p.max_local_surfels, 1);
    s->cap = cap;
    s->blk_stride = npool / 256 + 1;
    cudaError_t e = s->own.device(&s->surfels, cap, true);
    if (e == cudaSuccess) e = s->own.device(&s->seg, cap, true);
    if (e == cudaSuccess) e = s->own.device(&s->blk, (size_t)DSM_WINDOW_MAX_KEYS * s->blk_stride, true);
    if (e == cudaSuccess) e = s->own.device(&s->sync, dsm_win_sync_len(cap), true);
    if (e == cudaSuccess) e = s->own.device(&s->range, 2, true);
    if (e == cudaSuccess) e = cudaMemset(ctx->win_hdr, 0, 4 * sizeof(int32_t));
    if (e == cudaSuccess && ctx->pub_on) e = store_publish_alloc(*s);
    if (e == cudaSuccess && ctx->pub_on) e = publish_state_reset(ctx);
    if (e != cudaSuccess)
    {
        cudaGetLastError();
        return DSM_E_NOMEM;
    }
    ctx->inact = std::move(s);
    if (ctx->ckpt && checkpoint_images(ctx) != cudaSuccess)
    {
        cudaGetLastError();
        return DSM_E_NOMEM;
    }
    return DSM_OK;
}

extern "C" int dsm_inactive_size(dsm_ctx *ctx, int *n_surfels, int *n_segments)
{
    if (!ctx) return DSM_E_INVALID;
    int rs = res_sync(ctx);
    if (rs != DSM_OK) return rs;
    const InactStore *s = ctx->inact.get();
    if (n_surfels) *n_surfels = s ? s->size : 0;
    if (n_segments) *n_segments = s ? (int)s->segs.size() : 0;
    return DSM_OK;
}

// dsm_inactive_retire / _reactivate: the window step of one frame whose retire (or reactivation) list is {kf}, staged in
// half 0.  The caller has synchronised the stream, into which both phases of stream_run are joined, so the half is free.
// It has also checked capacity with exact sizes, so the step's own check cannot fail; S = 0, as no fuse follows.  No
// window tag is drawn: the step leaves the error gate of the resident kernels as it is.  Waits for the step and
// refreshes the mirror in the same round trip.
static int inactive_step(dsm_ctx *ctx, int kf, bool react)
{
    const int32_t ofs[2] = {0, 1};
    const WinLists w = react ? WinLists{nullptr, nullptr, &kf, ofs} : WinLists{&kf, ofs, nullptr, nullptr};
    const int rc = stage_window(ctx, 0, 1, w, 0, ctx->stream);
    if (rc != DSM_OK) return rc;
    const int nseg = (int)ctx->inact->segs.size();
    dsm_launch_window_step(resident_view(ctx, 0), window_view(ctx, 0, 0, 0), ctx->res_upper, react ? 0 : 1, react ? 1 : 0, ctx->stream);
    CK(cudaGetLastError());
    ctx->win_pending = true;
    return res_sync(ctx, react ? nseg : nseg + 1);
}

// move_add_surfels, removal loop: local surfels last updated by keyframe kf -> a new segment of the store
extern "C" int dsm_inactive_retire(dsm_ctx *ctx, int kf, int *n_moved)
{
    if (!ctx) return DSM_E_INVALID;
    int rc = res_enter(ctx, NEED_POOL | NEED_STORE);
    if (rc != DSM_OK) return rc;
    int cur = 0;
    rc = dsm_pool_size(ctx, &cur); // exact pool size: bounds the segment
    if (rc != DSM_OK) return rc;
    const InactStore &s = *ctx->inact;
    if (s.size + cur > s.cap) return DSM_E_CAPACITY;
    const int before = s.size;
    rc = inactive_step(ctx, kf, false);
    if (rc != DSM_OK) return rc;
    if (n_moved) *n_moved = s.size - before;
    return DSM_OK;
}

// move_add_surfels, insertion: the pose re-enters the drift-free window, its surfels go back to the end of the pool
extern "C" int dsm_inactive_reactivate(dsm_ctx *ctx, int kf, int *n_moved)
{
    if (!ctx) return DSM_E_INVALID;
    int rc = res_enter(ctx, NEED_POOL | NEED_STORE);
    if (rc != DSM_OK) return rc;
    int total = 0;
    for (const auto &sg : ctx->inact->segs)
        if (sg.kf == kf) total += sg.cnt;
    if (n_moved) *n_moved = total;
    if (total == 0) return DSM_OK;
    int cur = 0;
    rc = dsm_pool_size(ctx, &cur);
    if (rc != DSM_OK) return rc;
    if (cur + total > ctx->p.max_local_surfels) return DSM_E_CAPACITY;
    return inactive_step(ctx, kf, true);
}

// warp_inactive_surfels_cpu_kernel for ONE pose (surfel_map.cpp:704-733): p <- W p, n <- R_W n over its segment(s),
// W = (T_loop * T_cam^-1) computed by the caller in fp64 and cast to float, column-major.  Asynchronous: the keyframe's
// segments are found in the device table, in stream order.
extern "C" int dsm_inactive_transform(dsm_ctx *ctx, int kf, const float Wm[16])
{
    if (!ctx || !Wm) return DSM_E_INVALID;
    if (!ctx->inact) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(ctx->wmat, Wm, 16 * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    dsm_launch_inactive_transform(window_view(ctx, 0, 0, 0), kf, ctx->wmat, ctx->stream);
    CK(cudaGetLastError());
    return DSM_OK;
}

// attached_surfels of one pose (kf >= 0) or of every pose in store order (kf < 0), e.g. for save_mesh
extern "C" int dsm_inactive_download(dsm_ctx *ctx, int kf, dsm_surfel_t *out, int cap, int *n_out)
{
    if (!ctx || !n_out || cap < 0 || (cap > 0 && !out)) return DSM_E_INVALID;
    const int rc = res_enter(ctx, NEED_STORE);
    if (rc != DSM_OK) return rc;
    int n = 0;
    for (const auto &sg : ctx->inact->segs)
    {
        if (kf >= 0 && sg.kf != kf) continue;
        const int c = (n + sg.cnt <= cap) ? sg.cnt : (cap > n ? cap - n : 0);
        if (c > 0) CK(cudaMemcpyAsync(out + n, ctx->inact->surfels + sg.ofs, (size_t)c * sizeof(dsm_surfel_t), cudaMemcpyDeviceToHost, ctx->stream));
        n += sg.cnt;
    }
    CK(cudaStreamSynchronize(ctx->stream));
    *n_out = n;
    return DSM_OK;
}

// The store ranges [ofs, ofs + cnt) as one PointXYZI per stored surfel, concatenated in list order: *n_out = their total,
// the first min(cap, total) points are written
static int inactive_export_ranges(dsm_ctx *ctx, const std::vector<InactStore::Seg> &ranges, dsm_point_t *out, int cap, int *n_out)
{
    int total = 0;
    for (const auto &r : ranges) total += r.cnt;
    *n_out = total;
    const int npool = std::max(ctx->p.max_local_surfels, 1);
    const DsmDev d = inactive_view(ctx);
    int n = 0;
    for (const auto &r : ranges)
        for (int c0 = 0; c0 < r.cnt && n < cap;)
        { // chunks sized for the block tables and the second pool buffer (16-byte points into 44-byte slots)
            const int len = std::min({r.cnt - c0, npool, cap - n});
            dsm_launch_set2(ctx->inact->range, r.ofs + c0, r.ofs + c0 + len, ctx->stream);
            // every stored surfel passes update_times >= INT32_MIN: all len points are selected
            const int rc = select_out(ctx, d, len, 2, INT32_MIN, DSM_REC_POINT, out + n, len, nullptr);
            if (rc != DSM_OK) return rc;
            c0 += len;
            n += len;
        }
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    return DSM_OK;
}

// inactive_pointcloud (publish_inactive_pointcloud surfel_map.cpp:1385-1396, the tail of publish_all_pointcloud and
// save_cloud): one PointXYZI per stored surfel, store order
extern "C" int dsm_inactive_export_cloud(dsm_ctx *ctx, dsm_point_t *out, int cap, int *n_out)
{
    if (!ctx || !n_out || cap < 0 || (cap > 0 && !out)) return DSM_E_INVALID;
    const int rc = res_enter(ctx, NEED_STORE);
    return rc != DSM_OK ? rc : inactive_export_ranges(ctx, {InactStore::Seg{-1, 0, ctx->inact->size}}, out, cap, n_out);
}

// the inactive half of publish_neighbor_pointcloud (surfel_map.cpp:1306-1321): the stored points of each listed
// keyframe, list order, store order within a keyframe.  A keyframe without stored points (a local pose, or one with
// empty attached_surfels) contributes nothing, which is the reference's skip of both (:1311-1316).
extern "C" int dsm_inactive_export_poses(dsm_ctx *ctx, const int32_t *keyframes, int n_keyframes, dsm_point_t *out, int cap, int *n_out)
{
    if (!ctx || !n_out || n_keyframes < 0 || (n_keyframes > 0 && !keyframes) || cap < 0 || (cap > 0 && !out)) return DSM_E_INVALID;
    const int rc = res_enter(ctx, NEED_STORE);
    if (rc != DSM_OK) return rc;
    std::vector<InactStore::Seg> ranges;
    for (int k = 0; k < n_keyframes; k++)
        for (const auto &sg : ctx->inact->segs)
            if (sg.kf == keyframes[k]) ranges.push_back(sg);
    return inactive_export_ranges(ctx, ranges, out, cap, n_out);
}

// the segment table in store order, (keyframe, offset, count) per segment, from the mirror res_sync refreshes
extern "C" int dsm_inactive_segments(dsm_ctx *ctx, int32_t *kf_ofs_cnt, int cap, int *n_out)
{
    if (!ctx || !n_out || cap < 0 || (cap > 0 && !kf_ofs_cnt)) return DSM_E_INVALID;
    const int rc = res_enter(ctx, NEED_STORE);
    if (rc != DSM_OK) return rc;
    const std::vector<InactStore::Seg> &segs = ctx->inact->segs;
    for (int i = 0; i < (int)segs.size() && i < cap; i++)
    {
        kf_ofs_cnt[3 * i] = segs[i].kf;
        kf_ofs_cnt[3 * i + 1] = segs[i].ofs;
        kf_ofs_cnt[3 * i + 2] = segs[i].cnt;
    }
    *n_out = (int)segs.size();
    return DSM_OK;
}

int dsm_inactive_load_check(const dsm_ctx *ctx, const dsm_surfel_t *surfels, int n, const int32_t *kf_ofs_cnt, int n_segments)
{
    if (!ctx || n < 0 || n_segments < 0 || (n > 0 && !surfels) || (n_segments > 0 && !kf_ofs_cnt)) return DSM_E_INVALID;
    if (!ctx->inact || ctx->pub_in_flight || (ctx->field && ctx->field->in_flight)) return DSM_E_STATE;
    if (n > ctx->inact->cap) return DSM_E_CAPACITY;
    // the table: contiguous from 0, every segment at least one surfel, n in all, no negative keyframe
    int64_t ofs = 0;
    for (int i = 0; i < n_segments; i++)
    {
        const int32_t *g = kf_ofs_cnt + 3 * i;
        if (g[0] < 0 || g[1] != ofs || g[2] < 1) return DSM_E_INVALID;
        ofs += g[2];
        if (ofs > n) return DSM_E_INVALID;
    }
    if (ofs != n) return DSM_E_INVALID;
    // every stored surfel is live and was last updated by its segment's keyframe: retire selects by last_update and
    // the transforms leave it alone, so every store the library builds satisfies this
    for (int i = 0; i < n_segments; i++)
    {
        const int32_t *g = kf_ofs_cnt + 3 * i;
        for (int j = g[1]; j < g[1] + g[2]; j++)
            if (surfels[j].update_times == 0 || surfels[j].last_update != g[0]) return DSM_E_INVALID;
    }
    return DSM_OK;
}

// Replaces the store's contents and table.  Everything is checked before the device is touched.
extern "C" int dsm_inactive_load(dsm_ctx *ctx, const dsm_surfel_t *surfels, int n, const int32_t *kf_ofs_cnt, int n_segments)
{
    int rc = dsm_inactive_load_check(ctx, surfels, n, kf_ofs_cnt, n_segments);
    if (rc != DSM_OK) return rc;
    rc = res_enter(ctx, NEED_STORE);
    if (rc != DSM_OK) return rc;
    InactStore &s = *ctx->inact;
    dsm_checkpoint_map_replaced(ctx);
    std::vector<int4> table((size_t)n_segments);
    for (int i = 0; i < n_segments; i++) table[i] = make_int4(kf_ofs_cnt[3 * i], kf_ofs_cnt[3 * i + 1], kf_ofs_cnt[3 * i + 2], 0);
    const int32_t hdr[4] = {n, n_segments, 0, 0};
    CK(cudaStreamSynchronize(ctx->stream)); // nothing enqueued earlier may still read or write the store
    if (n > 0) CK(cudaMemcpyAsync(s.surfels, surfels, (size_t)n * sizeof(dsm_surfel_t), cudaMemcpyHostToDevice, ctx->stream));
    if (n_segments > 0) CK(cudaMemcpyAsync(s.seg, table.data(), table.size() * sizeof(int4), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->win_hdr, hdr, sizeof(hdr), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream)); // the sources are the caller's and the stack's
    s.segs.clear();
    for (int i = 0; i < n_segments; i++) s.segs.push_back(InactStore::Seg{table[i].x, table[i].y, table[i].z});
    s.size = s.upper = n;
    if (ctx->pub_on) CK(publish_state_reset(ctx));
    return DSM_OK;
}

int dsm_map_info(const dsm_ctx *ctx, DsmMapInfo *info)
{
    if (!ctx || !info) return DSM_E_INVALID;
    info->params = ctx->p;
    info->constants = dsm_constants{ctx->d.huber, ctx->d.baseline, ctx->d.disparity_error, ctx->d.min_tolerate_diff};
    info->store_cap = ctx->inact ? ctx->inact->cap : 0;
    info->publish_in_flight = ctx->pub_in_flight;
    info->field_in_flight = ctx->field && ctx->field->in_flight;
    info->view_rays = ctx->views && ctx->views->checkpointed ? ctx->d.S : 0;
    return DSM_OK;
}

// ---- publishing from inside the stream (include/dsm.h) ----
extern "C" int dsm_publish_enable(dsm_ctx *ctx)
{
    if (!ctx) return DSM_E_INVALID;
    if (!ctx->res_active || ctx->pub_on) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    // a call that failed half-way keeps what it allocated; the next one allocates only what is missing
    if (!ctx->pub_active) ctx->own.mapped(&ctx->pub_active, &ctx->pub_active_dev, (size_t)std::max(ctx->p.max_local_surfels, 1));
    if (!ctx->pub_hdr) ctx->own.mapped(&ctx->pub_hdr, &ctx->pub_hdr_dev, DSM_PUB_WORDS);
    if (!ctx->pub_state) ctx->own.device(&ctx->pub_state, 4);
    if (!ctx->pub_ev) ctx->own.event(&ctx->pub_ev);
    cudaError_t e = ctx->own.take();
    if (e == cudaSuccess) e = publish_state_reset(ctx);
    if (e == cudaSuccess && ctx->inact) e = store_publish_alloc(*ctx->inact);
    if (e != cudaSuccess)
    {
        cudaGetLastError();
        return DSM_E_NOMEM;
    }
    memset(ctx->pub_hdr, 0, DSM_PUB_WORDS * sizeof(int32_t));
    ctx->pub_on = true;
    return DSM_OK;
}

// Enqueue only: the selection writes the active points and their count, k_cloud_mirror the changed chunks of the
// inactive cloud and the rest of the header, all through device aliases of pinned host memory.  The view has no gate:
// after a rejected frame the pool is the one of the last applied frame, which is what the snapshot reports.
extern "C" int dsm_publish_enqueue(dsm_ctx *ctx, int min_update_times)
{
    if (!ctx) return DSM_E_INVALID;
    if (!ctx->pub_on || ctx->pub_in_flight) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    DsmDev d = resident_view(ctx, 0);
    d.gate = nullptr;
    // A publisher may never synchronise, so the host bound of the pool only grows: the grids are sized from the view's
    // bound, which is clamped to the capacity (the block tables hold no more), as the schedule's own launches are.
    dsm_launch_pool_select(d, 0, d.max_pool_per_frame, 2, min_update_times, DSM_REC_POINT, ctx->pub_active_dev, ctx->blkcnt, ctx->blkofs,
                           ctx->pub_hdr_dev + DSM_PUB_N_ACTIVE, ctx->stream);
    const InactStore *s = ctx->inact.get();
    dsm_launch_cloud_mirror(s ? s->surfels : nullptr, ctx->win_hdr, ctx->res_ofs, s ? s->upper : 0, s ? s->shadow : nullptr,
                            s ? s->mirror_dev : nullptr, ctx->pub_state, ctx->pub_hdr_dev, ctx->stream);
    CK(cudaGetLastError());
    CK(cudaEventRecord(ctx->pub_ev, ctx->stream));
    ctx->pub_in_flight = true;
    return DSM_OK;
}

extern "C" int dsm_publish_wait(dsm_ctx *ctx, const dsm_point_t **active, int *n_active, const dsm_point_t **inactive, int *n_inactive,
                                int *inactive_changed_from)
{
    if (!ctx) return DSM_E_INVALID;
    if (!ctx->pub_in_flight) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    CK(cudaEventSynchronize(ctx->pub_ev));
    ctx->pub_in_flight = false;
    const int32_t *h = ctx->pub_hdr;
    if (active) *active = ctx->pub_active;
    if (n_active) *n_active = h[DSM_PUB_N_ACTIVE];
    if (inactive) *inactive = ctx->inact ? ctx->inact->mirror : nullptr;
    if (n_inactive) *n_inactive = h[DSM_PUB_N_INACTIVE];
    if (inactive_changed_from) *inactive_changed_from = h[DSM_PUB_CHANGED_FROM];
    return capacity(ctx, h, DSM_PUB_ERR_TAG, "dsm_publish_wait", "the snapshot");
}

extern "C" int dsm_debug_publish_chunks(dsm_ctx *ctx, int *count)
{
    if (!ctx || !count) return DSM_E_INVALID;
    if (!ctx->pub_on || ctx->pub_in_flight) return DSM_E_STATE;
    *count = ctx->pub_hdr[DSM_PUB_CHUNKS];
    return DSM_OK;
}

// ---- the map as a distance field (include/dsm.h, DESIGN.md §8.7) ----
extern "C" int dsm_field_enable(dsm_ctx *ctx, const dsm_field_params *params)
{
    if (!ctx || !params) return DSM_E_INVALID;
    const dsm_field_params &p = *params;
    if (!std::isfinite(p.voxel) || !(p.voxel > 0.f)) return DSM_E_INVALID;
    for (int n : {p.nx, p.ny, p.nz})
        if (n < 1 || n > 1024) return DSM_E_INVALID;
    if (!ctx->res_active || ctx->field) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    auto f = std::make_unique<DsmField>();
    f->g.voxel = p.voxel;
    f->g.n[0] = p.nx, f->g.n[1] = p.ny, f->g.n[2] = p.nz;
    f->voxels = (size_t)p.nx * p.ny * p.nz;
    f->bytes = (dsm_field_header(f->voxels) + DSM_FIELD_WORDS) * sizeof(int32_t);
    f->own.device(&f->occ, f->voxels);
    f->own.device(&f->dist, f->bytes / sizeof(int32_t));
    f->own.host(&f->host, f->bytes / sizeof(int32_t));
    f->own.event(&f->ev);
    return keep(ctx->field, f, dsm_field_setup() == 0);
}

// ---- the signed distance field (include/dsm.h, DESIGN.md §8.16) ----
extern "C" int dsm_field_signed_enable(dsm_ctx *ctx)
{
    if (!ctx) return DSM_E_INVALID;
    DsmField *f = ctx->field.get();
    if (!f || f->sgn || f->in_flight) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    auto s = std::make_unique<DsmSignedField>();
    s->own.device(&s->grid, dsm_field_header(f->voxels) + DSM_SIGNED_WORDS);
    s->own.host(&s->host, f->voxels);
    return keep(f->sgn, s);
}

extern "C" int dsm_field_signed(dsm_ctx *ctx, const float **sdist)
{
    if (!ctx) return DSM_E_INVALID;
    const DsmField *f = ctx->field.get();
    if (!f || !f->signed_waited) return DSM_E_STATE;
    if (sdist) *sdist = f->resident ? nullptr : f->sgn->host;
    return capacity(ctx, f->host + dsm_field_header(f->voxels), DSM_FIELD_ERR_TAG, "dsm_field_signed", "the field");
}

// The views of a known request (dsm_field_enqueue_known), checked by the caller
struct KnownViews
{
    const int32_t *slots;
    const double *poses;
    int n;
};

// Enqueue only, like dsm_publish_enqueue: clear, mark, the three EDT passes and one copy of the grid with its header into
// the pinned buffer (host_copy), or of the header alone, then the event.  The launches have no gate: after a rejected
// frame the map is the one of the last applied frame, which is what the field reports.  With `known` the pose list is
// staged and copied first, the carve runs between the mark and the EDT, and host_copy copies the state grid as well.
static int field_enqueue(dsm_ctx *ctx, const double center[3], int min_update_times, bool host_copy, const KnownViews *known = nullptr)
{
    if (!ctx || !center || min_update_times < 1) return DSM_E_INVALID;
    DsmField *f = ctx->field.get();
    if (!f || f->in_flight) return DSM_E_STATE;
    DsmFieldGrid g = f->g;
    const int64_t lim = int64_t(1) << 24;
    for (int k = 0; k < 3; k++)
    {
        if (!std::isfinite(center[k])) return DSM_E_INVALID;
        const double q = std::floor(center[k] / (double)g.voxel);
        if (!(std::fabs(q) <= 4.0 * (double)lim)) return DSM_E_INVALID;
        const int64_t o = (int64_t)q - g.n[k] / 2;
        if (o < -lim || o > lim || o + g.n[k] < -lim || o + g.n[k] > lim) return DSM_E_INVALID;
        g.o[k] = (int)o;
        g.lo[k] = (float)o;
        g.hi[k] = (float)(o + g.n[k]);
    }
    CK(cudaSetDevice(ctx->device));
    const DsmDev d = resident_view(ctx, 0);
    const InactStore *s = ctx->inact.get();
    int32_t *header = f->dist + dsm_field_header(f->voxels);
    DsmViews *vw = ctx->views.get();
    if (known && known->n > 0)
    { // the previous known request's copy out of this staging ended before its wait, which no field in flight implies
        double *hp = reinterpret_cast<double *>(vw->stage_host);
        std::memcpy(hp, known->poses, 12 * sizeof(double) * (size_t)known->n);
        std::memcpy(hp + 12 * (size_t)known->n, known->slots, sizeof(int32_t) * (size_t)known->n);
        CK(cudaMemcpyAsync(vw->stage_dev, vw->stage_host, DsmViews::stage_bytes(known->n), cudaMemcpyHostToDevice, ctx->stream));
    }
    CK(cudaMemsetAsync(f->occ, 0, f->voxels, ctx->stream));
    CK(cudaMemsetAsync(header, 0, (known ? DSM_FIELD_VIEW + 1 : 1) * sizeof(int32_t), ctx->stream));
    int32_t *sgrid = f->sgn ? f->sgn->grid : nullptr; // every request after dsm_field_signed_enable builds the signed grid
    if (sgrid) CK(cudaMemsetAsync(sgrid + dsm_field_header(f->voxels) + DSM_SIGNED_N_F, 0, sizeof(int32_t), ctx->stream));
    dsm_launch_field_mark(ctx->d.pool, ctx->res_ofs, d.max_pool_per_frame, min_update_times, s ? s->surfels : nullptr, ctx->win_hdr,
                          s ? std::min(s->upper, s->cap) : 0, g, f->occ, header, ctx->stream);
    if (known)
    {
        const double *poses = reinterpret_cast<const double *>(vw->stage_dev);
        dsm_launch_field_carve(g, vw->rays, ctx->d.S, poses, reinterpret_cast<const int32_t *>(poses + 12 * (size_t)known->n), known->n,
                               vw->max_range, f->occ, ctx->stream);
    }
    dsm_launch_field_edt(g, f->occ, known != nullptr, f->dist, header, sgrid, ctx->stream);
    CK(cudaGetLastError());
    if (host_copy)
    {
        CK(cudaMemcpyAsync(f->host, f->dist, f->bytes, cudaMemcpyDeviceToHost, ctx->stream));
        if (known) CK(cudaMemcpyAsync(vw->state, f->occ, f->voxels, cudaMemcpyDeviceToHost, ctx->stream));
        if (sgrid) CK(cudaMemcpyAsync(f->sgn->host, sgrid, f->voxels * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    }
    else
        CK(cudaMemcpyAsync(f->host + dsm_field_header(f->voxels), header, DSM_FIELD_WORDS * sizeof(int32_t), cudaMemcpyDeviceToHost,
                           ctx->stream));
    CK(cudaEventRecord(f->ev, ctx->stream));
    f->g = g;
    f->in_flight = f->requested = true;
    f->resident = !host_copy;
    f->known = known != nullptr;
    f->known_waited = false;
    f->signed_latest = sgrid != nullptr;
    f->signed_waited = false;
    f->requests++;
    return DSM_OK;
}

extern "C" int dsm_field_enqueue(dsm_ctx *ctx, const double center[3], int min_update_times)
{
    return field_enqueue(ctx, center, min_update_times, true);
}

extern "C" int dsm_field_enqueue_resident(dsm_ctx *ctx, const double center[3], int min_update_times)
{
    return field_enqueue(ctx, center, min_update_times, false);
}

extern "C" int dsm_field_wait(dsm_ctx *ctx, const float **dist, int32_t origin[3], int *n_occupied)
{
    if (!ctx) return DSM_E_INVALID;
    DsmField *f = ctx->field.get();
    const int rc = wait_head(ctx, f);
    if (rc != DSM_OK) return rc;
    f->known_waited = f->known;
    f->signed_waited = f->signed_latest;
    const int32_t *h = f->host + dsm_field_header(f->voxels);
    if (dist) *dist = f->resident ? nullptr : reinterpret_cast<const float *>(f->host);
    if (origin) origin[0] = f->g.o[0], origin[1] = f->g.o[1], origin[2] = f->g.o[2];
    if (n_occupied) *n_occupied = h[DSM_FIELD_N_OCCUPIED];
    return capacity(ctx, h, DSM_FIELD_ERR_TAG, "dsm_field_wait", "the field");
}

// ---- free versus unknown space: captured views and the known-space field (include/dsm.h, DESIGN.md §8.9) ----
extern "C" int dsm_views_enable(dsm_ctx *ctx, int max_views, float max_range)
{
    if (!ctx || max_views < 1 || max_views > DSM_VIEWS_MAX || !std::isfinite(max_range) || !(max_range > 0.f)) return DSM_E_INVALID;
    const DsmField *f = ctx->field.get();
    if (!f || ctx->views) return DSM_E_STATE;
    // a ray visits at most about 3 * 1024 voxels
    if (!((double)max_range <= 1024.0 * (double)f->g.voxel)) return DSM_E_INVALID;
    // k_field_carve's one-dimensional grid over max_views views (only frames of billions of pixels come near it)
    if ((int64_t)max_views * dsm_carve_ctas_per_view(ctx->d.S) > INT32_MAX) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    auto v = std::make_unique<DsmViews>();
    v->max_views = max_views, v->max_range = max_range;
    v->filled.assign((size_t)max_views, 0);
    v->gen.assign((size_t)max_views, 0);
    v->own.device(&v->rays, (size_t)max_views * ctx->d.S);
    v->own.host(&v->state, f->voxels);
    v->own.host(&v->stage_host, DsmViews::stage_bytes(max_views));
    v->own.device(&v->stage_dev, DsmViews::stage_bytes(max_views));
    return keep(ctx->views, v);
}

// Enqueue only.  The frame's slot is safe to read on the main stream: the call that filled it left its schedule ordered
// before later work there, and the next call that rewrites the slot is the next-but-one resident run, whose phase 1
// waits for half_free of this half (recorded on the main stream at the entry of the run in between, so after this
// capture), or any other call that takes images, which synchronises with the main stream before it stages them.
extern "C" int dsm_views_capture(dsm_ctx *ctx, int frame, int slot)
{
    if (!ctx) return DSM_E_INVALID;
    DsmViews *v = ctx->views.get();
    if (!v) return DSM_E_STATE;
    if (slot < 0 || slot >= v->max_views) return DSM_E_INVALID;
    if (ctx->img_n == 0) return DSM_E_STATE;
    if (frame < 0 || frame >= ctx->img_n) return DSM_E_INVALID;
    if (!ctx->img_fit) return DSM_E_STATE; // uploaded but not run, or run with the plane fit cut off
    CK(cudaSetDevice(ctx->device));
    const int S = ctx->d.S;
    dsm_launch_views_capture(ctx->d.plane + (size_t)(ctx->img_slot0 + frame) * S * 3, S, v->rays + (size_t)slot * S, ctx->stream);
    CK(cudaGetLastError());
    v->filled[(size_t)slot] = 1;
    v->gen[(size_t)slot] = ++v->gens;
    return DSM_OK;
}

// ---- views in the checkpoint (include/dsm.h, DESIGN.md §8.18) ----
// Calls f(first, count) for each run of consecutive slots in an ascending list
template <typename F>
static cudaError_t slot_runs(const int32_t *slots, int n, F f)
{
    for (int i = 0; i < n;)
    {
        int j = i + 1;
        while (j < n && slots[j] == slots[j - 1] + 1) j++;
        const cudaError_t e = f(i, j - i);
        if (e != cudaSuccess) return e;
        i = j;
    }
    return cudaSuccess;
}

int dsm_views_load_check(const dsm_ctx *ctx, const int32_t *slots, int n, const void *rays)
{
    const DsmViews *v = ctx->views.get();
    for (int i = 0; i < n; i++)
        if (slots[i] >= v->max_views) return DSM_E_CAPACITY;
    // what k_views_capture writes: finite coordinates with w = 1, or all 16 bytes zero
    const uint8_t *b = static_cast<const uint8_t *>(rays);
    static const uint8_t zero[16] = {};
    for (size_t r = 0; r < (size_t)n * ctx->d.S; r++)
    {
        float4 q;
        std::memcpy(&q, b + 16 * r, 16);
        const bool ray = q.w == 1.f && std::isfinite(q.x) && std::isfinite(q.y) && std::isfinite(q.z);
        if (!ray && std::memcmp(&q, zero, 16) != 0) return DSM_E_INVALID;
    }
    return DSM_OK;
}

int dsm_views_load(dsm_ctx *ctx, const int32_t *slots, int n, const void *rays)
{
    DsmViews &v = *ctx->views;
    const size_t S = (size_t)ctx->d.S;
    const uint8_t *b = static_cast<const uint8_t *>(rays);
    CK(cudaSetDevice(ctx->device));
    CK(slot_runs(slots, n, [&](int i, int c) {
        return cudaMemcpyAsync(v.rays + (size_t)slots[i] * S, b + 16 * S * i, 16 * S * c, cudaMemcpyHostToDevice, ctx->stream);
    }));
    CK(cudaStreamSynchronize(ctx->stream)); // the source is the file's buffer
    std::fill(v.filled.begin(), v.filled.end(), 0);
    for (int i = 0; i < n; i++) v.filled[(size_t)slots[i]] = 1;
    for (uint64_t &g : v.gen) g = ++v.gens; // every slot differs from the checkpoint image
    return DSM_OK;
}

int dsm_views_download(dsm_ctx *ctx, std::vector<int32_t> &slots, std::vector<uint8_t> &rays)
{
    const DsmViews &v = *ctx->views;
    const size_t S = (size_t)ctx->d.S;
    slots.clear();
    for (int s = 0; s < v.max_views; s++)
        if (v.filled[(size_t)s]) slots.push_back(s);
    rays.resize(16 * S * slots.size());
    CK(cudaSetDevice(ctx->device));
    CK(slot_runs(slots.data(), (int)slots.size(), [&](int i, int c) {
        return cudaMemcpyAsync(rays.data() + 16 * S * i, v.rays + (size_t)slots[i] * S, 16 * S * c, cudaMemcpyDeviceToHost, ctx->stream);
    }));
    CK(cudaStreamSynchronize(ctx->stream));
    return DSM_OK;
}

static cudaError_t checkpoint_view_image(dsm_ctx *ctx);

extern "C" int dsm_checkpoint_views_enable(dsm_ctx *ctx)
{
    if (!ctx) return DSM_E_INVALID;
    DsmViews *v = ctx->views.get();
    if (!v || v->checkpointed) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    v->checkpointed = true;
    if (ctx->ckpt && checkpoint_view_image(ctx) != cudaSuccess)
    {
        cudaGetLastError();
        v->checkpointed = false;
        return DSM_E_NOMEM;
    }
    return DSM_OK;
}

extern "C" int dsm_field_enqueue_known(dsm_ctx *ctx, const double center[3], int min_update_times, const int32_t *slots,
                                       const double *poses, int n_views, int host_copy)
{
    if (!ctx) return DSM_E_INVALID;
    const DsmViews *v = ctx->views.get();
    if (!v) return DSM_E_STATE;
    if (n_views < 0 || n_views > v->max_views || (n_views > 0 && (!slots || !poses))) return DSM_E_INVALID;
    for (int j = 0; j < n_views; j++)
    {
        if (slots[j] < 0 || slots[j] >= v->max_views || !v->filled[(size_t)slots[j]]) return DSM_E_INVALID;
        for (int k = 0; k < 12; k++)
            if (!std::isfinite(poses[12 * (size_t)j + k])) return DSM_E_INVALID;
    }
    const KnownViews known{slots, poses, n_views};
    return field_enqueue(ctx, center, min_update_times, host_copy != 0, &known);
}

extern "C" int dsm_field_state(dsm_ctx *ctx, const uint8_t **state, int *n_free)
{
    if (!ctx) return DSM_E_INVALID;
    const DsmField *f = ctx->field.get();
    if (!f || !f->known_waited) return DSM_E_STATE;
    if (state) *state = f->resident ? nullptr : ctx->views->state;
    if (n_free) *n_free = f->host[dsm_field_header(f->voxels) + DSM_FIELD_N_FREE];
    return DSM_OK;
}

// A known request without views: the caller's states, the known distance transform and the host copy of dist with its
// header (the states are already in the pinned state buffer).  The error words stay 0.
extern "C" int dsm_debug_field_load_state(dsm_ctx *ctx, const uint8_t *state, const int32_t origin[3])
{
    if (!ctx || !state || !origin) return DSM_E_INVALID;
    DsmField *f = ctx->field.get();
    DsmViews *vw = ctx->views.get();
    if (!f || !vw || f->in_flight) return DSM_E_STATE;
    DsmFieldGrid g = f->g;
    const int64_t lim = int64_t(1) << 24;
    for (int k = 0; k < 3; k++)
    {
        const int64_t o = origin[k];
        if (o < -lim || o > lim || o + g.n[k] < -lim || o + g.n[k] > lim) return DSM_E_INVALID;
        g.o[k] = (int)o;
        g.lo[k] = (float)o;
        g.hi[k] = (float)(o + g.n[k]);
    }
    for (size_t i = 0; i < f->voxels; i++)
        if (state[i] > DSM_STATE_FREE) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    std::memcpy(vw->state, state, f->voxels); // no copy out of it is pending: no field is in flight
    int32_t *header = f->dist + dsm_field_header(f->voxels);
    CK(cudaMemcpyAsync(f->occ, vw->state, f->voxels, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemsetAsync(header, 0, (DSM_FIELD_VIEW + 1) * sizeof(int32_t), ctx->stream));
    int32_t *sgrid = f->sgn ? f->sgn->grid : nullptr; // every request after dsm_field_signed_enable builds the signed grid
    if (sgrid) CK(cudaMemsetAsync(sgrid + dsm_field_header(f->voxels) + DSM_SIGNED_N_F, 0, sizeof(int32_t), ctx->stream));
    dsm_launch_field_edt(g, f->occ, true, f->dist, header, sgrid, ctx->stream);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(f->host, f->dist, f->bytes, cudaMemcpyDeviceToHost, ctx->stream));
    if (sgrid) CK(cudaMemcpyAsync(f->sgn->host, sgrid, f->voxels * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaEventRecord(f->ev, ctx->stream));
    f->g = g;
    f->in_flight = f->requested = f->known = true;
    f->resident = f->known_waited = f->signed_waited = false;
    f->signed_latest = sgrid != nullptr;
    f->requests++;
    return DSM_OK;
}

// ---- checkpoints that do not stop the stream (include/dsm.h, DESIGN.md §8.5) ----
// The two images at the context's current capacities; whatever was there before is released first (the old and the new
// need not fit at once).  On failure the checkpoint has no images and its calls return DSM_E_STATE.
static cudaError_t checkpoint_images(dsm_ctx *ctx)
{
    DsmCheckpoint &k = *ctx->ckpt;
    k.img.reset();
    k.dev = k.host = k.host_dev = nullptr;
    k.stale = true;
    auto own = std::make_unique<CudaOwner>();
    const int store_cap = ctx->inact ? ctx->inact->cap : 0;
    const DsmSnapLayout lay = dsm_snap_layout(ctx->p.max_local_surfels, store_cap);
    const int pool_chunks = std::max(dsm_snap_chunks(ctx->p.max_local_surfels), 1), store_chunks = dsm_snap_chunks(store_cap);
    const size_t bytes = lay.bytes + dsm_line_up((size_t)pool_chunks + store_chunks); // k_map_delta's flags follow the image
    uint8_t *dev = nullptr, *host = nullptr, *host_dev = nullptr;
    // not zeroed but for the header line (k_map_delta's count of finished CTAs): the drain also copies the unused tail of
    // each section's last line, which the writer never reads
    cudaError_t e = own->device(&dev, bytes);
    if (e == cudaSuccess) e = cudaMemsetAsync(dev, 0, 128, ctx->stream); // ordered before the first snapshot
    if (e == cudaSuccess) e = own->mapped(&host, &host_dev, bytes);
    if (e != cudaSuccess) return e;
    k.img = std::move(own);
    k.lay = lay;
    k.pool_chunks = pool_chunks, k.store_chunks = store_chunks;
    k.dev = dev, k.host = host, k.host_dev = host_dev;
    return cudaSuccess;
}

// The views section of the image (DESIGN.md §8.18), once both dsm_checkpoint_enable and dsm_checkpoint_views_enable have
// run: it holds no slot yet, so the next snapshot copies every filled one, and the next incremental checkpoint is a base.
// On failure nothing is kept.
static cudaError_t checkpoint_view_image(dsm_ctx *ctx)
{
    DsmCheckpoint &k = *ctx->ckpt;
    const DsmViews &v = *ctx->views;
    const size_t rays = (size_t)v.max_views * ctx->d.S;
    auto own = std::make_unique<CudaOwner>();
    float4 *dev = nullptr, *host = nullptr;
    cudaError_t e = own->device(&dev, rays);
    if (e == cudaSuccess) e = own->host(&host, rays);
    if (e != cudaSuccess) return e;
    k.vimg = std::move(own);
    k.vdev = dev, k.vhost = host;
    k.vgen.assign((size_t)v.max_views, 0);
    k.stale = true;
    return cudaSuccess;
}

void dsm_checkpoint_map_replaced(dsm_ctx *ctx)
{
    if (ctx && ctx->ckpt) ctx->ckpt->stale = true;
}

// An incremental checkpoint on the checkpoint's thread (DESIGN.md §8.6): a base writes the file and a fresh journal
// header, a record lists the chunks k_map_delta flagged and appends them with the table and extra.  The chain ends on any
// failure, so that the next incremental checkpoint writes a base.
static int checkpoint_write_incremental(DsmCheckpoint &k, const DsmMapSections &s)
{
    if (k.kind == DsmCheckpoint::BASE)
    {
        uint64_t sum = 0, bytes = 0, jbytes = 0;
        int rc = dsm_map_write(k.path.c_str(), k.info, s, &sum, &bytes);
        if (rc == DSM_OK) rc = dsm_journal_start(k.path.c_str(), sum, s.rays_per_view, &jbytes);
        if (rc != DSM_OK) return rc;
        k.chain_path = k.path;
        k.chain_sum = sum, k.sequence = 1, k.base_bytes = bytes, k.journal_bytes = jbytes;
        return DSM_OK;
    }
    const uint8_t *flags = k.host + k.lay.bytes;
    k.chunks.clear();
    const int cp = dsm_snap_chunks(s.n_pool), cs = dsm_snap_chunks(s.n_store);
    for (int c = 0; c < cp; c++)
        if (flags[c]) k.chunks.push_back(c);
    const int k_pool = (int)k.chunks.size();
    for (int c = 0; c < cs; c++)
        if (flags[k.pool_chunks + c]) k.chunks.push_back(c);
    const DsmJournalRecord r{k.sequence, k.chain_sum, s.n_pool, s.n_store, s.n_segments, k.chunks.data(), k_pool,
                             k.chunks.data() + k_pool, (int)k.chunks.size() - k_pool, k.host + k.lay.pool, k.host + k.lay.store,
                             s.table, s.extra, s.extra_bytes, s.view_slots, s.n_views, s.view_rays, s.rays_per_view};
    uint64_t sum = 0, bytes = 0;
    const int rc = dsm_journal_append(k.path.c_str(), k.journal_bytes, r, &sum, &bytes);
    if (rc != DSM_OK) return rc;
    k.chain_path = k.path;
    k.chain_sum = sum, k.sequence++, k.journal_bytes += bytes;
    return DSM_OK;
}

// The write of one enqueued checkpoint, on the checkpoint's thread: waits for the drain, then writes the host image's
// sections through the file's one writer.  A snapshot that recorded a rejected frame writes nothing.
static int checkpoint_write(DsmCheckpoint &k)
{
    if (k.kind != DsmCheckpoint::FULL) k.chain_path.clear(); // set again once the base or the record is on the disk
    if (cudaEventSynchronize(k.ev_drain) != cudaSuccess) return DSM_E_CUDA;
    const volatile int32_t *h = reinterpret_cast<const volatile int32_t *>(k.host);
    if (h[DSM_SNAP_ERR_TAG] != 0)
    {
        k.err_frame = h[DSM_SNAP_ERR_FRAME];
        return DSM_E_CAPACITY;
    }
    // the views the drain brought over, by slot: every filled one for a file or a base, the snapshot's for a record
    const int S = k.info.view_rays;
    std::vector<const void *> views(k.view_slots.size());
    for (size_t i = 0; i < views.size(); i++) views[i] = k.vhost + (size_t)k.view_slots[i] * S;
    const DsmMapSections s{reinterpret_cast<const dsm_surfel_t *>(k.host + k.lay.pool), h[DSM_SNAP_N_POOL],
                           reinterpret_cast<const dsm_surfel_t *>(k.host + k.lay.store), h[DSM_SNAP_N_STORE],
                           reinterpret_cast<const int32_t *>(k.host + k.lay.table), h[DSM_SNAP_N_SEGMENTS],
                           k.extra.data(), k.extra.size(), k.view_slots.data(), (int)k.view_slots.size(), views.data(), S};
    if (k.kind == DsmCheckpoint::FULL) return dsm_map_write(k.path.c_str(), k.info, s);
    return checkpoint_write_incremental(k, s);
}

static void checkpoint_thread(DsmCheckpoint *k, int device)
{
    cudaSetDevice(device);
    std::unique_lock<std::mutex> lk(k->m);
    for (;;)
    {
        k->cv.wait(lk, [k] { return k->queued || k->quit; });
        if (!k->queued) return;
        lk.unlock();
        const int rc = checkpoint_write(*k);
        lk.lock();
        k->result = rc;
        k->queued = false;
        k->cv.notify_all();
    }
}

extern "C" int dsm_checkpoint_enable(dsm_ctx *ctx)
{
    if (!ctx) return DSM_E_INVALID;
    if (!ctx->res_active || ctx->ckpt) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    auto k = std::make_unique<DsmCheckpoint>();
    int lo = 0, hi = 0;
    cudaError_t e = cudaDeviceGetStreamPriorityRange(&lo, &hi);
    if (e == cudaSuccess) e = k->own.stream(&k->s_drain, lo); // the least priority: the stream's kernels come first
    if (e == cudaSuccess) e = k->own.event(&k->ev_snap);
    // the thread waits on this event for the whole stream queued before the snapshot: it sleeps instead of spinning a core
    if (e == cudaSuccess) e = k->own.event(&k->ev_drain, cudaEventDisableTiming | cudaEventBlockingSync);
    ctx->ckpt = std::move(k);
    if (e == cudaSuccess) e = checkpoint_images(ctx);
    if (e == cudaSuccess && ctx->views && ctx->views->checkpointed) e = checkpoint_view_image(ctx);
    if (e != cudaSuccess)
    {
        cudaGetLastError();
        ctx->ckpt.reset();
        return DSM_E_NOMEM;
    }
    try
    {
        ctx->ckpt->worker = std::thread(checkpoint_thread, ctx->ckpt.get(), ctx->device);
    }
    catch (...)
    {
        ctx->ckpt.reset();
        return DSM_E_NOMEM;
    }
    return DSM_OK;
}

// Enqueue only, like dsm_publish_enqueue: the snapshot on the context's stream, the drain on the checkpoint's stream
// after it, the write on the checkpoint's thread.  The view of the map has no gate: the snapshot records the error word.
static int checkpoint_enqueue(dsm_ctx *ctx, const char *path, const void *extra, size_t extra_bytes, bool incremental)
{
    if (!ctx || !path || (extra_bytes > 0 && !extra)) return DSM_E_INVALID;
    DsmCheckpoint *k = ctx->ckpt.get();
    if (!k || k->pending || !k->img) return DSM_E_STATE;
    // as dsm_map_save (through dsm_pool_size): a batch call since the last dsm_pool_upload left the batch's slices in the
    // pool buffer and no resident pool to save; an asynchronous batch still in flight runs on streams the snapshot is not
    // ordered against
    if (!ctx->res_active || ctx->in_flight) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    DsmMapInfo info;
    dsm_map_info(ctx, &info);
    const InactStore *s = ctx->inact.get();
    // a record needs the image to hold the chain's last checkpoint, under this path, and a journal no larger than its
    // base; the thread has retired the previous checkpoint, so its chain state is final here
    DsmCheckpoint::Kind kind = DsmCheckpoint::FULL;
    if (incremental)
        kind = k->stale || k->chain_path != path || k->journal_bytes > k->base_bytes ? DsmCheckpoint::BASE : DsmCheckpoint::RECORD;
    // grids from the host bounds, clamped to the capacities: a caller that never synchronises keeps bounds that only grow
    const int pool_upper = std::min(ctx->res_upper, ctx->p.max_local_surfels), store_upper = s ? std::min(s->upper, s->cap) : 0;
    if (kind == DsmCheckpoint::RECORD)
        dsm_launch_map_delta(ctx->d.pool, ctx->res_ofs, pool_upper, s ? s->surfels : nullptr, s ? s->seg : nullptr, ctx->win_hdr,
                             store_upper, k->dev, k->lay, k->pool_chunks, ctx->stream);
    else
        dsm_launch_map_snapshot(ctx->d.pool, ctx->res_ofs, pool_upper, s ? s->surfels : nullptr, s ? s->seg : nullptr, ctx->win_hdr,
                                store_upper, k->dev, k->lay, ctx->stream);
    CK(cudaGetLastError());
    // views (DESIGN.md §8.18): the slots captured or loaded since the previous snapshot into the image, at the same
    // stream position; then, after the snapshot, every filled slot of the image to the host, or for a record the copied ones
    const DsmViews *v = info.view_rays > 0 ? ctx->views.get() : nullptr;
    const size_t S = (size_t)ctx->d.S;
    std::vector<int32_t> &snap = k->snap_slots, filled;
    snap.clear();
    if (v)
    {
        for (int i = 0; i < v->max_views; i++)
            if (v->filled[(size_t)i])
            {
                filled.push_back(i);
                if (v->gen[(size_t)i] != k->vgen[(size_t)i]) snap.push_back(i);
            }
        CK(slot_runs(snap.data(), (int)snap.size(), [&](int i, int c) {
            return cudaMemcpyAsync(k->vdev + snap[i] * S, v->rays + snap[i] * S, 16 * S * c, cudaMemcpyDeviceToDevice, ctx->stream);
        }));
    }
    CK(cudaEventRecord(k->ev_snap, ctx->stream));
    CK(cudaStreamWaitEvent(k->s_drain, k->ev_snap, 0));
    if (kind == DsmCheckpoint::RECORD)
        dsm_launch_map_drain_delta(k->dev, k->host_dev, k->lay, k->pool_chunks, k->store_chunks, k->drain_ctas, k->s_drain);
    else
        dsm_launch_map_drain(k->dev, k->host_dev, k->lay, k->drain_ctas, k->s_drain);
    CK(cudaGetLastError());
    const std::vector<int32_t> &drained = kind == DsmCheckpoint::RECORD ? snap : filled;
    if (v)
        CK(slot_runs(drained.data(), (int)drained.size(), [&](int i, int c) {
            return cudaMemcpyAsync(k->vhost + drained[i] * S, k->vdev + drained[i] * S, 16 * S * c, cudaMemcpyDeviceToHost, k->s_drain);
        }));
    CK(cudaEventRecord(k->ev_drain, k->s_drain));
    // the image now holds these slots, whether or not the write succeeds: a failed write ends the chain, and the base
    // that follows drains every filled slot of the image
    for (int32_t i : snap) k->vgen[(size_t)i] = v->gen[(size_t)i];
    {
        std::lock_guard<std::mutex> lk(k->m);
        k->view_slots = drained;
        k->path = path;
        k->extra.assign(static_cast<const uint8_t *>(extra), static_cast<const uint8_t *>(extra) + extra_bytes);
        k->info = info;
        k->kind = kind;
        k->queued = true;
    }
    k->cv.notify_all();
    k->pending = true;
    k->stale = kind == DsmCheckpoint::FULL; // k_map_snapshot wrote the image for a file outside the chain
    return DSM_OK;
}

extern "C" int dsm_checkpoint_enqueue(dsm_ctx *ctx, const char *path, const void *extra, size_t extra_bytes)
{
    return checkpoint_enqueue(ctx, path, extra, extra_bytes, false);
}

// One chunk pass and a drain of the changed lines for a record; the map of k_map_snapshot for a base (DESIGN.md §8.6)
extern "C" int dsm_checkpoint_enqueue_incremental(dsm_ctx *ctx, const char *path, const void *extra, size_t extra_bytes)
{
    return checkpoint_enqueue(ctx, path, extra, extra_bytes, true);
}

extern "C" int dsm_checkpoint_wait(dsm_ctx *ctx, int block, int *finished)
{
    if (finished) *finished = 0;
    if (!ctx) return DSM_E_INVALID;
    DsmCheckpoint *k = ctx->ckpt.get();
    if (!k || !k->pending) return DSM_E_STATE;
    std::unique_lock<std::mutex> lk(k->m);
    if (k->queued && !block) return DSM_OK;
    k->cv.wait(lk, [k] { return !k->queued; });
    k->pending = false;
    if (finished) *finished = 1;
    if (k->result == DSM_E_CAPACITY)
        snprintf(ctx->err, sizeof(ctx->err), "dsm_checkpoint_wait: frame %d of a dsm_fuse_stream_window call did not fit the pool or "
                 "the store before the checkpoint; no file was written", k->err_frame);
    else if (k->result == DSM_E_IO)
        snprintf(ctx->err, sizeof(ctx->err), "dsm_checkpoint_wait: %s could not be written", k->path.c_str());
    else if (k->result == DSM_E_CUDA)
        snprintf(ctx->err, sizeof(ctx->err), "dsm_checkpoint_wait: the drain of the snapshot failed");
    return k->result;
}

extern "C" int dsm_debug_checkpoint_drain_ctas(dsm_ctx *ctx, int ctas)
{
    if (!ctx || ctas < 1) return DSM_E_INVALID;
    if (!ctx->ckpt || ctx->ckpt->pending) return DSM_E_STATE;
    ctx->ckpt->drain_ctas = ctas;
    return DSM_OK;
}

// A run of n consecutive frames of ONE sequential stream on the resident pool.  Results are identical to n runs of one
// frame each (dsm_fuse_frame_resident): superpixels, normals and plane fits do not depend on the pose or the pool, so they run
// for all n frames as one batch (full-width launches instead of n latency-bound single-frame ones); only the fuse /
// initialise / post-step, which carry the pool from frame t to frame t+1, run frame by frame.
static int list_len(const int32_t *o, int t) { return o ? o[t + 1] - o[t] : 0; }

// Host-side validation of the lists (include/dsm.h); *any: some frame has a non-empty list
static int window_validate(const dsm_ctx *ctx, int n, const WinLists &w, bool *any)
{
    *any = false;
    const int32_t *k[2] = {w.rk, w.ak}, *o[2] = {w.ro, w.ao};
    for (int l = 0; l < 2; l++)
    {
        if (!o[l]) continue;
        if (o[l][0] < 0) return DSM_E_INVALID;
        for (int t = 0; t < n; t++)
            if (o[l][t + 1] < o[l][t] || o[l][t + 1] - o[l][t] > DSM_WINDOW_MAX_KEYS) return DSM_E_INVALID;
        if (o[l][n] > o[l][0])
        {
            if (!k[l]) return DSM_E_INVALID;
            *any = true;
        }
    }
    std::vector<int32_t> f;
    for (int t = 0; t < n; t++)
    { // no keyframe twice in one frame's lists, nor in both
        f.clear();
        for (int l = 0; l < 2; l++)
            for (int i = o[l] ? o[l][t] : 0; o[l] && i < o[l][t + 1]; i++)
            {
                if (k[l][i] < 0) return DSM_E_INVALID;
                f.push_back(k[l][i]);
            }
        std::sort(f.begin(), f.end());
        if (std::adjacent_find(f.begin(), f.end()) != f.end()) return DSM_E_INVALID;
    }
    if (*any && !ctx->inact) return DSM_E_STATE;
    return DSM_OK;
}

// dsm_fuse_stream_resident and dsm_fuse_frame_resident, and with `win` dsm_fuse_stream_window: each frame's window step
// runs right before its fuse.  Rows of the n images lie gray_pitch / depth_pitch bytes apart.
static int stream_run(dsm_ctx *ctx, int n, const int32_t *ref_idx, const uint8_t *gray, size_t gray_pitch, const float *depth,
                      size_t depth_pitch, const float *poses, int32_t *n_new, const WinLists *win)
{
    if (!ctx || !ref_idx || !gray || !depth || !poses) return DSM_E_INVALID;
    if (n < 1 || n > ctx->p.max_batch) return DSM_E_INVALID;
    bool any = false;
    if (win)
    {
        const int rv = window_validate(ctx, n, *win, &any);
        if (rv != DSM_OK) return rv;
    }
    if (!ctx->res_active) return DSM_E_STATE;
    if (ctx->in_flight) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    // (the windowed call checks every frame on the device, with the counts only the device has)
    if (!win && ctx->res_upper + n * ctx->d.S > ctx->p.max_local_surfels)
    { // the bound may be loose: fetch the exact size before giving up
        int cur = 0;
        int rc = dsm_pool_size(ctx, &cur);
        if (rc != DSM_OK) return rc;
        if (cur + n * ctx->d.S > ctx->p.max_local_surfels) return DSM_E_CAPACITY;
    }
    const size_t fpx = (size_t)ctx->p.height * ctx->p.width;
    // two staging halves when they fit: the H2D copy of this run overlaps the kernels of the previous one
    const bool dbl = 2 * n <= ctx->p.max_batch;
    const int par = dbl ? (ctx->res_frame & 1) : 0;
    ctx->res_frame++;
    cudaStream_t st = ctx->stream;
    // The ordering rule of include/dsm.h (dsm_fuse_stream_resident).  Each call records half_free of the OTHER half on the
    // main stream at its entry: the next run uses that half, and everything enqueued before this call (that half's
    // previous run and any later reads of its slots included) comes before that point, but this run does not, so the
    // next run's phase 1 overlaps this run's phase 2.  The host waits for the same point before it rewrites the half's
    // pinned tables and staging buffers.  A run over both halves (!dbl) is ordered on the main stream and frees both
    // halves at its end.
    CK(cudaEventRecord(ctx->half_free[1 - par], st));
    CK(cudaEventSynchronize(ctx->half_free[par]));
    if (!dbl) CK(cudaEventSynchronize(ctx->half_free[1 - par]));
    const size_t so = (size_t)par * (size_t)(ctx->p.max_batch / 2); // fixed halves: runs of different length never overlap
    const int slot0 = (int)so;
    int rc = stage_images(ctx, slot0, n, gray, gray_pitch, depth, depth_pitch, ctx->s_h2d);
    if (rc != DSM_OK) return rc;
    CK(cudaEventRecord(ctx->half_h2d[par], ctx->s_h2d));
    // Phase 1 (superpixels, normals, plane fits of all n frames; never touches the pool) runs on a side stream and in this
    // half's own frame slots [so, so + n): it overlaps the frame-by-frame phase 2 of the PREVIOUS run, which owns the
    // other half's slots and the main stream.  (With a single half, so == 0 and everything is ordered on the main stream.)
    // Phase 2 is a chain of small launches per frame: next to phase 1's full-width grids its CTAs would queue behind a
    // wave of theirs at every launch, so it runs on the context's highest-priority stream (forked from / joined into the
    // main stream, which keeps the order with every other call on the context).
    cudaStream_t s1 = dbl ? ctx->s_comp[par] : st;
    cudaStream_t s2 = dbl ? ctx->s_hi : st;
    if (dbl)
    { // this half's slots and device tables were last read by the phase 2 of the run before the previous one
        CK(cudaEventRecord(ctx->ev_fork, st));
        CK(cudaStreamWaitEvent(s2, ctx->ev_fork, 0));
        CK(cudaStreamWaitEvent(s1, ctx->half_free[par], 0));
    }
    // pinned tables of this mode live in the second half of h_pose / h_ref (the first half belongs to the batch calls,
    // which only wait for their own copies before rewriting it); this half's previous table copy ran before
    // half_free[par], which has been waited for above
    rc = stage_tables(ctx, (size_t)ctx->p.max_batch + so, slot0, n, poses, ref_idx, s1);
    if (rc != DSM_OK) return rc;
    const int tag = win ? (ctx->win_tag = ctx->win_tag % 0x3fffffff + 1) : 0;
    if (win)
    {
        rc = stage_window(ctx, par, n, *win, tag, s1);
        if (rc != DSM_OK) return rc;
    }
    CK(cudaStreamWaitEvent(s1, ctx->half_h2d[par], 0));
    // phase 1: all n frames at once, in the batch view (never touches the pool)
    DsmDev v = ctx->d;
    v.frame0 = slot0;
    v.max_pool_per_frame = 0;
    {
        ProfScope p(ctx, DSM_K_REPACK, s1);
        dsm_launch_repack(v, n, ctx->gray_packed + so * fpx, ctx->depth_packed + so * fpx, s1);
    }
    rc = enqueue_schedule(ctx, v, n, s1, 1);
    if (rc != DSM_OK) return rc;
    if (dbl)
    {
        CK(cudaEventRecord(ctx->ev_join[par], s1));
        CK(cudaStreamWaitEvent(s2, ctx->ev_join[par], 0));
    }
    // phase 2: frame by frame on the resident pool, each frame ending with the in-place post-step
    const int cap = ctx->p.max_local_surfels;
    for (int t = 0; t < n; t++)
    {
        if (win)
        { // host bounds without readback: a retire can move at most the pool, a reactivation at most the store
            const int nr = list_len(win->ro, t), na = list_len(win->ao, t);
            InactStore *s = ctx->inact.get(); // present whenever a list is not empty (window_validate)
            if (nr > 0) s->upper = (int)std::min<long long>((long long)s->upper + ctx->res_upper, s->cap);
            if (na > 0) ctx->res_upper = (int)std::min<long long>((long long)ctx->res_upper + s->upper, cap);
            // with empty lists the step is only the capacity check, needed once the bound no longer proves the frame fits
            if (nr > 0 || na > 0 || ctx->res_upper + ctx->d.S > cap)
            {
                const DsmDev dv = resident_view(ctx, slot0 + t);
                dsm_launch_window_step(dv, window_view(ctx, par, t, ctx->d.S), dv.max_pool_per_frame, nr, na, s2);
            }
        }
        rc = enqueue_schedule(ctx, resident_view(ctx, slot0 + t), 1, s2, 2);
        if (rc != DSM_OK) return rc;
        // the device applies no frame that would pass the capacity, so the capacity bounds the pool as well: a caller
        // that never synchronises (a publishing node) keeps a bound that stays finite
        ctx->res_upper = std::min(ctx->res_upper + ctx->d.S, cap);
    }
    if (win) ctx->win_pending = true;
    hold_frames(ctx, slot0, n, true); // the slots are ordered before the main stream through phase 2 (ev_join / ev_p2)
    if (dbl)
    {
        CK(cudaEventRecord(ctx->ev_p2, s2));
        CK(cudaStreamWaitEvent(st, ctx->ev_p2, 0));
    }
    else
    {
        for (cudaEvent_t ev : ctx->half_free) CK(cudaEventRecord(ev, st));
    }
    CK(cudaGetLastError());
    // the caller may reuse its image buffers as soon as we return
    CK(cudaEventSynchronize(ctx->half_h2d[par]));
    if (n_new)
    {
        int32_t h[4] = {0, 0, 0, 0};
        CK(cudaMemcpyAsync(n_new, ctx->d.nnew + slot0, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        if (ctx->win_pending) CK(cudaMemcpyAsync(h, ctx->res_ofs, sizeof(h), cudaMemcpyDeviceToHost, st)); // (only set by a windowed call)
        CK(cudaStreamSynchronize(st));
        if (h[2] != 0)
        { // frames from the rejected one on (all of them when an earlier call's frame was rejected) were not applied
            for (int t = h[2] == tag ? h[3] : 0; t < n; t++) n_new[t] = -1;
        }
        return res_sync(ctx);
    }
    return DSM_OK;
}

extern "C" int dsm_fuse_frame_resident(dsm_ctx *ctx, int ref_idx, const uint8_t *gray, size_t gray_pitch,
                                       const float *depth, size_t depth_pitch, const float pose[16], int *n_new)
{
    if (!ctx || !gray || !depth || !pose) return DSM_E_INVALID;
    if (!ctx->res_active) return DSM_E_STATE;
    if (gray_pitch < (size_t)ctx->p.width || depth_pitch < (size_t)ctx->p.width * 4) return DSM_E_INVALID;
    const int32_t ref = ref_idx;
    return stream_run(ctx, 1, &ref, gray, gray_pitch, depth, depth_pitch, pose, n_new, nullptr);
}

extern "C" int dsm_fuse_stream_resident(dsm_ctx *ctx, int n, const int32_t *ref_idx, const uint8_t *gray, const float *depth,
                                        const float *poses, int32_t *n_new)
{
    if (!ctx) return DSM_E_INVALID;
    return stream_run(ctx, n, ref_idx, gray, (size_t)ctx->p.width, depth, (size_t)ctx->p.width * 4, poses, n_new, nullptr);
}

extern "C" int dsm_fuse_stream_window(dsm_ctx *ctx, int n, const int32_t *ref_idx, const uint8_t *gray, const float *depth,
                                      const float *poses, const int32_t *retire_kf, const int32_t *retire_ofs,
                                      const int32_t *reactivate_kf, const int32_t *reactivate_ofs, int32_t *n_new)
{
    if (!ctx) return DSM_E_INVALID;
    const WinLists w{retire_kf, retire_ofs, reactivate_kf, reactivate_ofs};
    return stream_run(ctx, n, ref_idx, gray, (size_t)ctx->p.width, depth, (size_t)ctx->p.width * 4, poses, n_new, &w);
}

// ---- raw cloud of a frame (publish_raw_pointcloud, surfel_map.cpp:1115-1151) ----
// R = Quaternionf(qw, qx, qy, qz).toRotationMatrix() (not normalised) and T = position, in float like the reference
static DsmRawPose raw_pose(const double p7[7])
{
    const float qx = (float)p7[3], qy = (float)p7[4], qz = (float)p7[5], qw = (float)p7[6];
    const float tx = 2.f * qx, ty = 2.f * qy, tz = 2.f * qz;
    const float twx = tx * qw, twy = ty * qw, twz = tz * qw;
    const float txx = tx * qx, txy = ty * qx, txz = tz * qx;
    const float tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
    return DsmRawPose{{1.f - (tyy + tzz), txy - twz, txz + twy,
                       txy + twz, 1.f - (txx + tzz), tyz - twx,
                       txz - twy, tyz + twx, 1.f - (txx + tyy)},
                      {(float)p7[0], (float)p7[1], (float)p7[2]}};
}

extern "C" int dsm_frame_raw_cloud(dsm_ctx *ctx, int frame, const double pose7[7], dsm_point_t *out, int cap, int *n_out)
{
    if (!ctx || !pose7 || !n_out || cap < 0 || (cap > 0 && !out)) return DSM_E_INVALID;
    if (ctx->img_n == 0) return DSM_E_STATE;
    if (frame < 0 || frame >= ctx->img_n) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    const int rc = finish_batch(ctx);
    if (rc != DSM_OK) return rc;
    const int W = ctx->p.width, H = ctx->p.height;
    const size_t npx = (size_t)W * H;
    if (!ctx->raw_out && ctx->own.device(&ctx->raw_out, npx) != cudaSuccess)
    {
        cudaGetLastError();
        ctx->own.take();
        ctx->raw_out = nullptr;
        return DSM_E_NOMEM;
    }
    // every entry point leaves the frame's copy and repack ordered before later work on the main stream
    dsm_launch_raw_cloud(ctx->d, ctx->img_slot0 + frame, raw_pose(pose7), ctx->raw_out, ctx->stream);
    CK(cudaGetLastError());
    *n_out = (int)npx;
    const size_t c = npx < (size_t)cap ? npx : (size_t)cap;
    if (c > 0) CK(cudaMemcpyAsync(out, ctx->raw_out, c * sizeof(dsm_point_t), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return DSM_OK;
}

// ---- superpixel normal image of a frame (FusionFunctions::debug_show, fusion_functions.cpp:977-1006) ----
extern "C" int dsm_frame_superpixel_image(dsm_ctx *ctx, int frame, uint8_t *bgr, size_t pitch)
{
    if (!ctx || !bgr || pitch < (size_t)3 * ctx->p.width) return DSM_E_INVALID;
    if (ctx->img_n == 0) return DSM_E_STATE;
    if (frame < 0 || frame >= ctx->img_n) return DSM_E_INVALID;
    if (!ctx->img_fit) return DSM_E_STATE; // uploaded but not run, or run with the plane fit cut off
    CK(cudaSetDevice(ctx->device));
    const int rc = finish_batch(ctx);
    if (rc != DSM_OK) return rc;
    const int W = ctx->p.width, H = ctx->p.height;
    const size_t row = (size_t)3 * ctx->d.Wp; // staging row pitch: a multiple of 48 bytes, so every row is word-aligned
    if (!ctx->spimg_out && ctx->own.device(&ctx->spimg_out, row * H) != cudaSuccess)
    {
        cudaGetLastError();
        ctx->own.take();
        ctx->spimg_out = nullptr;
        return DSM_E_NOMEM;
    }
    // every entry point leaves the frame's schedule ordered before later work on the main stream
    dsm_launch_superpixel_image(ctx->d, ctx->img_slot0 + frame, ctx->spimg_out, ctx->stream);
    CK(cudaGetLastError());
    CK(cudaMemcpy2DAsync(bgr, pitch, ctx->spimg_out, row, (size_t)3 * W, H, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return DSM_OK;
}

// ---- parity / debug readback ----
extern "C" int dsm_get_labels(dsm_ctx *ctx, int frame, int32_t *labels_hw)
{
    if (!ctx || !labels_hw || frame < 0 || frame >= ctx->p.max_batch) return DSM_E_INVALID;
    if (!ctx->ran) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    const int W = ctx->p.width, H = ctx->p.height;
    dsm_launch_labels_export(ctx->d, frame, ctx->stream); // the schedule keeps the labels as the u8 code plane only
    CK(cudaGetLastError());
    CK(cudaMemcpy2DAsync(labels_hw, (size_t)W * 4, ctx->d.labels + (size_t)frame * ctx->d.px_stride, (size_t)ctx->d.Wp * 4,
                         (size_t)W * 4, H, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return DSM_OK;
}

extern "C" int dsm_get_seeds(dsm_ctx *ctx, int frame, dsm_seed_t *seeds)
{
    if (!ctx || !seeds || frame < 0 || frame >= ctx->p.max_batch) return DSM_E_INVALID;
    if (!ctx->ran) return DSM_E_STATE;
    CK(cudaSetDevice(ctx->device));
    dsm_launch_seeds_export(ctx->d, frame, ctx->seed_export, (ctx->stop_after > 0 && ctx->stop_after < kPlaneFitSteps) ? 1 : 0, ctx->stream);
    CK(cudaMemcpyAsync(seeds, ctx->seed_export, (size_t)ctx->d.S * sizeof(dsm_seed_t), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    return DSM_OK;
}

extern "C" int dsm_device_buffer(dsm_ctx *ctx, int which, void **dev_ptr, size_t *bytes)
{
    if (!ctx || !dev_ptr || !bytes) return DSM_E_INVALID;
    switch (which)
    {
    case DSM_BUF_NEW_SURFELS:
        *dev_ptr = ctx->d.newsurf;
        *bytes = (size_t)ctx->p.max_batch * ctx->d.S * sizeof(dsm_surfel_t);
        return DSM_OK;
    case DSM_BUF_NEW_COUNTS:
        *dev_ptr = ctx->d.nnew;
        *bytes = (size_t)ctx->p.max_batch * sizeof(int32_t);
        return DSM_OK;
    case DSM_BUF_LOCAL:
        *dev_ptr = ctx->d.pool;
        *bytes = (size_t)(ctx->p.max_local_surfels > 0 ? ctx->p.max_local_surfels : 1) * sizeof(dsm_surfel_t);
        return DSM_OK;
    default:
        return DSM_E_INVALID;
    }
}
