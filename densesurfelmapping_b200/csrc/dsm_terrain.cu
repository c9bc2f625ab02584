// The terrain of the latest known field (dsm_terrain_*, DESIGN.md §8.20): per column of the field grid along the up
// axis, the uppermost occupied voxel with observed free headroom above it, the step to its neighbours, a status in the
// field's state codes and the distance to the nearest cell that is not traversable, in stream order.
//
//   k_terrain_support  one thread per column, walking from the top of the column down in the up sense with a run of
//                      consecutive free voxels; the first occupied voxel with a run of at least `headroom` is the
//                      support.  Consecutive threads take consecutive cells of the terrain grid: with up along y or z
//                      those are consecutive x, so every load of a warp is one coalesced row segment.  With up along x
//                      a column is a contiguous row of the grid and consecutive threads walk rows nx bytes apart: each
//                      warp load touches 32 lines, which the next loads of the walk find in L1.  CTA 0 copies the
//                      field's error words into the terrain header.
//   k_terrain_step     one thread per cell: the 3x3 neighbourhood of `level` in the two horizontal axes gives step and
//                      status.
//   the clearance      the known field's three EDT passes (dsm_launch_field_edt, unchanged) on the terrain grid, over
//                      the status plane, into the result's distance plane and header: the row pass's counts of states
//                      1 and 2 are the blocked and the traversable cells.
// The kernels carry no error gate and are launched without PDL, as the other field kernels.  The job's C ABI calls
// (dsm_terrain_enable, _enqueue and _wait) follow them.
//
// One packed result (D2H), its layout in DsmTerrain (dsm_ctx.hpp); the terrain reach job (dsm_reach.cu) reads its status
// and clearance planes and its header on the device.
#include "dsm_ctx.hpp"

#define TERRAIN_BLOCK 256
#define TERRAIN_HEADER_WORDS DsmTerrain::HEADER_WORDS

static_assert(sizeof(dsm_terrain_info_t) == 64 && offsetof(dsm_terrain_info_t, n_support) == 36, "dsm_terrain_info_t layout");
static_assert(DSM_FIELD_WORDS <= TERRAIN_HEADER_WORDS, "the terrain header holds a field header");

// the column of cell c starts at voxel base and steps by stride along the up axis
__global__ void __launch_bounds__(TERRAIN_BLOCK) k_terrain_support(const uint8_t *__restrict__ st, const int32_t *__restrict__ fhdr, int cells,
                                                                   int m0, int m1, int n0, int n1, int len, int stride, int up,
                                                                   int headroom, int16_t *__restrict__ level, int32_t *hdr)
{
    if (blockIdx.x == 0 && threadIdx.x == 0)
    { // the field's error words at its request travel with the result
        hdr[DSM_FIELD_ERR_TAG] = fhdr[DSM_FIELD_ERR_TAG];
        hdr[DSM_FIELD_ERR_FRAME] = fhdr[DSM_FIELD_ERR_FRAME];
    }
    const int c = blockIdx.x * TERRAIN_BLOCK + threadIdx.x;
    if (c >= cells) return;
    const int x = c % m0, y = c / m0 % m1, z = c / (m0 * m1);
    const uint8_t *col = st + ((size_t)z * n1 + y) * n0 + x;
    int run = 0, found = -1;
    for (int j = 0; j < len; j++)
    {
        const int k = up > 0 ? len - 1 - j : j;
        const uint8_t s = col[(size_t)k * stride];
        if (s == DSM_STATE_OCCUPIED && run >= headroom)
        {
            found = k;
            break;
        }
        run = s == DSM_STATE_FREE ? run + 1 : 0;
    }
    level[c] = (int16_t)found;
}

// h0 < h1 the two horizontal axes of the terrain grid, s0 and s1 their cell strides
__global__ void __launch_bounds__(TERRAIN_BLOCK) k_terrain_step(const int16_t *__restrict__ level, int cells, int m0, int m1, int h0, int h1,
                                                                int s0, int s1, int len0, int len1, int max_step,
                                                                uint8_t *__restrict__ status, uint8_t *__restrict__ step)
{
    const int c = blockIdx.x * TERRAIN_BLOCK + threadIdx.x;
    if (c >= cells) return;
    const int l = level[c];
    int worst = 0;
    if (l >= 0)
    {
        const int x = c % m0, y = c / m0 % m1, z = c / (m0 * m1);
        const int u = h0 == 0 ? x : y, w = h1 == 1 ? y : z; // h0 is 0 or 1, h1 is 1 or 2
        for (int du = -1; du <= 1; du++)
            for (int dw = -1; dw <= 1; dw++)
            {
                if ((du == 0 && dw == 0) || (unsigned)(u + du) >= (unsigned)len0 || (unsigned)(w + dw) >= (unsigned)len1) continue;
                const int ln = level[c + du * s0 + dw * s1];
                if (ln >= 0) worst = max(worst, abs(l - ln));
            }
    }
    status[c] = l < 0 ? DSM_STATE_UNKNOWN : (worst > max_step ? DSM_STATE_OCCUPIED : DSM_STATE_FREE);
    step[c] = (uint8_t)min(worst, 255);
}

static unsigned tr_blocks(int n) { return (unsigned)((n + TERRAIN_BLOCK - 1) / TERRAIN_BLOCK); }

extern "C" int dsm_terrain_enable(dsm_ctx *ctx, int up)
{
    if (!ctx) return DSM_E_INVALID;
    const DsmField *f = ctx->field.get();
    if (!f || !ctx->views || ctx->terrain) return DSM_E_STATE;
    if (up == 0 || up < -3 || up > 3) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    auto tr = std::make_unique<DsmTerrain>();
    tr->up = up;
    for (int k = 0; k < 3; k++) tr->m[k] = k == std::abs(up) - 1 ? 1 : f->g.n[k];
    tr->cells = tr->m[0] * tr->m[1] * tr->m[2];
    const size_t res = DsmTerrain::res_bytes(tr->cells);
    tr->own.device(&tr->res, res);
    tr->own.host(&tr->res_host, res);
    tr->own.event(&tr->ev);
    return keep(ctx->terrain, tr);
}

// Enqueue only: the job on the state grid of the latest (known) field request with that request's origin, one D2H copy
// of the result and the event.  A later field request clears that grid only behind the job, in stream order.
extern "C" int dsm_terrain_enqueue(dsm_ctx *ctx, int headroom, int max_step)
{
    if (!ctx) return DSM_E_INVALID;
    DsmTerrain *tr = ctx->terrain.get();
    const DsmField *f = known_field(ctx);
    if (!tr || !f || tr->in_flight) return DSM_E_STATE;
    const int a = std::abs(tr->up) - 1, len = f->g.n[a];
    if (headroom < 1 || headroom > len - 1 || max_step < 0 || max_step > DSM_TERRAIN_MAX_STEP) return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    const cudaStream_t s = ctx->stream;
    const int C = tr->cells, *n = f->g.n, *m = tr->m;
    int32_t *dist = reinterpret_cast<int32_t *>(tr->res);
    int32_t *hdr = reinterpret_cast<int32_t *>(tr->res + DsmTerrain::header_at(C));
    int16_t *level = reinterpret_cast<int16_t *>(tr->res + DsmTerrain::level_at(C));
    uint8_t *status = tr->res + DsmTerrain::status_at(C), *step = tr->res + DsmTerrain::step_at(C);
    const int strides[3] = {1, n[0], n[0] * n[1]}, cstrides[3] = {1, m[0], m[0] * m[1]};
    const int h0 = a == 0 ? 1 : 0, h1 = a == 2 ? 1 : 2;
    CK(cudaMemsetAsync(hdr, 0, 4 * TERRAIN_HEADER_WORDS, s));
    k_terrain_support<<<tr_blocks(C), TERRAIN_BLOCK, 0, s>>>(f->occ, f->dist + dsm_field_header(f->voxels), C, m[0], m[1], n[0], n[1], len,
                                                              strides[a], tr->up, headroom, level, hdr);
    k_terrain_step<<<tr_blocks(C), TERRAIN_BLOCK, 0, s>>>(level, C, m[0], m[1], h0, h1, cstrides[h0], cstrides[h1], m[h0], m[h1], max_step,
                                                           status, step);
    DsmFieldGrid g = f->g; // the terrain grid: the request's grid collapsed along the up axis, at its origin
    g.n[a] = 1;
    dsm_launch_field_edt(g, status, true, dist, hdr, nullptr, s);
    CK(cudaGetLastError());
    for (int k = 0; k < 3; k++) tr->origin[k] = f->g.o[k];
    tr->headroom = headroom, tr->max_step = max_step;
    tr->enqueues++;
    return submit(ctx, *tr, tr->res, DsmTerrain::res_bytes(C), f->requests);
}

extern "C" int dsm_terrain_wait(dsm_ctx *ctx, dsm_terrain_info_t *info, const int16_t **level, const uint8_t **status, const uint8_t **step,
                                const float **clearance)
{
    if (!ctx) return DSM_E_INVALID;
    DsmTerrain *tr = ctx->terrain.get();
    const int rc = wait_head(ctx, tr);
    if (rc != DSM_OK) return rc;
    const int C = tr->cells;
    const int32_t *h = reinterpret_cast<const int32_t *>(tr->res_host + DsmTerrain::header_at(C));
    if (info)
    {
        *info = dsm_terrain_info_t();
        for (int k = 0; k < 3; k++) info->origin[k] = tr->origin[k], info->m[k] = tr->m[k];
        info->up = tr->up, info->headroom = tr->headroom, info->max_step = tr->max_step;
        info->n_blocked = h[DSM_FIELD_N_OCCUPIED];
        info->n_traversable = h[DSM_FIELD_N_FREE];
        info->n_support = info->n_blocked + info->n_traversable;
    }
    if (level) *level = reinterpret_cast<const int16_t *>(tr->res_host + DsmTerrain::level_at(C));
    if (status) *status = tr->res_host + DsmTerrain::status_at(C);
    if (step) *step = tr->res_host + DsmTerrain::step_at(C);
    if (clearance) *clearance = reinterpret_cast<const float *>(tr->res_host);
    return capacity(ctx, h, DSM_FIELD_ERR_TAG, "dsm_terrain_wait", "the field the job read");
}
