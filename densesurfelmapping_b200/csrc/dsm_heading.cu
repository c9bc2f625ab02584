// Headings along trajectories (dsm_heading_*, DESIGN.md §8.19): per sample of a trajectory and per rotation of a list,
// the unknown and frontier voxels a camera there would see through the latest known field, then per trajectory the
// best rate-limited rotation sequence.
//
//   k_heading_views  one 8x8x4 brick of a sample's box per CTA of 256 threads, one voxel per thread, bricks laid out
//                    sample-major in a one-dimensional grid (the layout of k_gain_views); thread 0 finds the CTA's sample
//                    by a binary search over the samples' first bricks.  Each thread builds the mask of rotations whose
//                    frustum holds its voxel (dsm_gain_frustum, rotations in shared memory), walks once for a non-empty
//                    mask (dsm_gain_walk: a walk depends on the camera position and the voxel, never on the rotation),
//                    and ballots and popcounts add its unknown or frontier voxel to per-rotation counts in shared
//                    memory, as k_vp_score does; one atomicAdd per non-zero counter per CTA.
//   k_heading_plan   one warp per trajectory: the backward pass over the samples with the rotations spread across the
//                    lanes (r = lane, lane + 32), the values of the next sample in double-buffered shared memory and the
//                    first best step per (sample, rotation) stored as int8 in the successor table; then lane 0 traces
//                    forward from start and writes the rotations, turns and the record.  Block 0 writes the header.
// The counts are integers and the plan exact in int64, so the result does not depend on the schedule.  The kernels
// carry no error gate and are launched without PDL, as the other field kernels.  The job's C ABI calls
// (dsm_heading_enable, _enqueue and _wait) follow them.
//
// One staged request (H2D, head_stage_bytes(n, S)):
//   double rotations[64][9] | DsmHeadingTraj trajectories[n] | DsmHeadingSample samples[S]
// and one packed result (D2H, head_res_bytes(n, S, n_rot)):
//   int32 header[DSM_HEAD_WORDS] | dsm_heading_t records[n] | dsm_heading_sample_t samples[S] | dsm_heading_count_t counts[S][n_rot]
// The header's first eleven words are those of dsm_heading_info_t; its last two carry the field's error words, cleared
// by dsm_heading_wait.
#include "dsm_ctx.hpp"
#include <climits>

enum
{
    DSM_HEAD_ORIGIN = 0, // 3 words
    DSM_HEAD_N = 3,
    DSM_HEAD_N_SAMPLES,
    DSM_HEAD_N_ROT,
    DSM_HEAD_UNKNOWN_BLOCKS,
    DSM_HEAD_N_STATUS,     // 2 words: trajectories per status (k_heading_plan adds)
    DSM_HEAD_ERR_TAG = 14, // the field header's DSM_FIELD_ERR_TAG / _ERR_FRAME, copied by k_heading_plan
    DSM_HEAD_ERR_FRAME,
    DSM_HEAD_WORDS = 16 // 64 B
};
// one trajectory as the host stages it: its first sample and samples, the request, and its samples outside the grid
struct DsmHeadingTraj
{
    int32_t sample0, n_samples, start, end, max_step, n_outside;
}; // 24 B
// one sample as the host stages it: the camera position, the hull of its gain boxes over the rotations (lo, size; size
// 0 on an axis: empty, as for a camera outside the grid) and its first brick in the launch
struct DsmHeadingSample
{
    double p[3];
    int32_t lo[3], size[3], brick0, pad;
}; // 56 B

#define HEAD_BLOCK (DSM_GAIN_BX * DSM_GAIN_BY * DSM_GAIN_BZ) // 256
#define HEAD_PLAN_WARPS 4
#define HEAD_NONE LLONG_MIN // the value of a (sample, rotation) from which the end cannot be reached

static_assert(sizeof(dsm_heading_request_t) == 16 && sizeof(dsm_heading_t) == 32 && sizeof(dsm_heading_sample_t) == 32 &&
                  sizeof(dsm_heading_count_t) == 8 && sizeof(dsm_heading_info_t) == 64, "dsm_heading layouts");
static_assert(DSM_HEAD_WORDS * 4 == sizeof(dsm_heading_info_t) && DSM_HEAD_N_STATUS == 7, "the header starts with the info");
static_assert(sizeof(DsmHeadingTraj) == 24 && sizeof(DsmHeadingSample) == 56, "staged layouts");
static_assert(DSM_HEADING_MAX_ROTATIONS == 64, "one 64-bit rotation mask, two rotations per lane, int8 steps");

// §8.10's frontier voxel: free, with a face neighbour of state unknown inside the grid (the test of k_gain_views)
__device__ __forceinline__ bool head_frontier(const uint8_t *__restrict__ state, size_t i, int x, int y, int z, int nx, int ny, int nz)
{
    return (x > 0 && __ldg(state + i - 1) == DSM_STATE_UNKNOWN) || (x + 1 < nx && __ldg(state + i + 1) == DSM_STATE_UNKNOWN) ||
           (y > 0 && __ldg(state + i - nx) == DSM_STATE_UNKNOWN) || (y + 1 < ny && __ldg(state + i + nx) == DSM_STATE_UNKNOWN) ||
           (z > 0 && __ldg(state + i - (size_t)nx * ny) == DSM_STATE_UNKNOWN) ||
           (z + 1 < nz && __ldg(state + i + (size_t)nx * ny) == DSM_STATE_UNKNOWN);
}

__global__ void __launch_bounds__(HEAD_BLOCK) k_heading_views(const DsmFieldGrid g, const uint8_t *__restrict__ state,
                                                              const DsmHeadingSample *__restrict__ smp, int n_samples,
                                                              const double *__restrict__ rotations, int n_rot, double fx, double fy,
                                                              double cx, double cy, double width, double height, double range2,
                                                              int unknown_blocks, dsm_heading_count_t *__restrict__ counts)
{
    __shared__ double s_rot[9 * DSM_HEADING_MAX_ROTATIONS];
    __shared__ DsmHeadingSample sv;
    __shared__ int s_smp;
    __shared__ unsigned s_cnt[2][DSM_HEADING_MAX_ROTATIONS]; // unknown, frontier
    const int tid = threadIdx.x, lane = tid & 31;
    for (int k = tid; k < 9 * n_rot; k += HEAD_BLOCK) s_rot[k] = rotations[k];
    if (tid == 0)
    {
        int lo = 0, hi = n_samples; // the last sample whose first brick is <= this one
        while (hi - lo > 1)
        {
            const int m = (lo + hi) / 2;
            if (smp[m].brick0 <= (int)blockIdx.x)
                lo = m;
            else
                hi = m;
        }
        s_smp = lo;
    }
    if (tid < 2 * DSM_HEADING_MAX_ROTATIONS) s_cnt[tid / DSM_HEADING_MAX_ROTATIONS][tid % DSM_HEADING_MAX_ROTATIONS] = 0;
    __syncthreads();
    const int j = s_smp;
    if (tid < (int)(sizeof(DsmHeadingSample) / 4))
        reinterpret_cast<int32_t *>(&sv)[tid] = reinterpret_cast<const int32_t *>(smp + j)[tid];
    __syncthreads();
    const int nbx = (sv.size[0] + DSM_GAIN_BX - 1) / DSM_GAIN_BX, nby = (sv.size[1] + DSM_GAIN_BY - 1) / DSM_GAIN_BY;
    const int b = (int)blockIdx.x - sv.brick0;
    const int dx = b % nbx * DSM_GAIN_BX + tid % DSM_GAIN_BX, dy = b / nbx % nby * DSM_GAIN_BY + tid / DSM_GAIN_BX % DSM_GAIN_BY,
              dz = b / (nbx * nby) * DSM_GAIN_BZ + tid / (DSM_GAIN_BX * DSM_GAIN_BY);
    const int x = sv.lo[0] + dx, y = sv.lo[1] + dy, z = sv.lo[2] + dz;
    const int nx = g.n[0], ny = g.n[1], nz = g.n[2];
    const double v = (double)g.voxel;
    const double tx = sv.p[0], ty = sv.p[1], tz = sv.p[2];
    unsigned long long mask = 0;
    bool unknown = false, front = false;
    if (dx < sv.size[0] && dy < sv.size[1] && dz < sv.size[2])
    {
        const double c0 = __dmul_rn(__dadd_rn((double)(g.o[0] + x), 0.5), v), c1 = __dmul_rn(__dadd_rn((double)(g.o[1] + y), 0.5), v),
                     c2 = __dmul_rn(__dadd_rn((double)(g.o[2] + z), 0.5), v);
        const double d0 = __dsub_rn(c0, tx), d1 = __dsub_rn(c1, ty), d2 = __dsub_rn(c2, tz);
        for (int r = 0; r < n_rot; r++)
            if (dsm_gain_frustum<3>(s_rot + 9 * r, d0, d1, d2, fx, fy, cx, cy, width, height, range2)) mask |= 1ull << r;
        if (mask && dsm_gain_walk(g, state, unknown_blocks, tx, ty, tz, c0, c1, c2))
        {
            const size_t i = ((size_t)z * ny + y) * nx + x;
            const uint8_t st = __ldg(state + i);
            unknown = st == DSM_STATE_UNKNOWN;
            front = st == DSM_STATE_FREE && head_frontier(state, i, x, y, z, nx, ny, nz);
        }
    }
    if (__any_sync(0xffffffffu, unknown || front))
        for (int r = 0; r < n_rot; r++)
        {
            const bool in = mask >> r & 1;
            const unsigned bu = __ballot_sync(0xffffffffu, unknown && in), bf = __ballot_sync(0xffffffffu, front && in);
            if (lane == 0)
            {
                if (bu) atomicAdd(&s_cnt[0][r], __popc(bu));
                if (bf) atomicAdd(&s_cnt[1][r], __popc(bf));
            }
        }
    __syncthreads();
    if (tid < 2 * DSM_HEADING_MAX_ROTATIONS)
    {
        const int kind = tid / DSM_HEADING_MAX_ROTATIONS, r = tid % DSM_HEADING_MAX_ROTATIONS;
        if (r < n_rot && s_cnt[kind][r]) atomicAdd(&counts[(size_t)j * n_rot + r].n_unknown + kind, (int)s_cnt[kind][r]);
    }
}

__global__ void __launch_bounds__(HEAD_PLAN_WARPS * 32) k_heading_plan(const DsmFieldGrid g, const int32_t *__restrict__ fhdr,
                                                                       const DsmHeadingTraj *__restrict__ traj, int n,
                                                                       const DsmHeadingSample *__restrict__ smp, int n_samples, int n_rot,
                                                                       int unknown_blocks, long long w_unknown, long long w_frontier,
                                                                       const dsm_heading_count_t *__restrict__ counts,
                                                                       int8_t *__restrict__ succ, int32_t *__restrict__ hdr,
                                                                       dsm_heading_t *__restrict__ rec, dsm_heading_sample_t *__restrict__ out)
{
    __shared__ long long s_val[HEAD_PLAN_WARPS][2][DSM_HEADING_MAX_ROTATIONS];
    __shared__ int s_steps[HEAD_PLAN_WARPS][2][DSM_HEADING_MAX_ROTATIONS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (blockIdx.x == 0 && threadIdx.x == 0)
    {
        for (int k = 0; k < 3; k++) hdr[DSM_HEAD_ORIGIN + k] = g.o[k];
        hdr[DSM_HEAD_N] = n;
        hdr[DSM_HEAD_N_SAMPLES] = n_samples;
        hdr[DSM_HEAD_N_ROT] = n_rot;
        hdr[DSM_HEAD_UNKNOWN_BLOCKS] = unknown_blocks;
        hdr[DSM_HEAD_ERR_TAG] = fhdr[DSM_FIELD_ERR_TAG];
        hdr[DSM_HEAD_ERR_FRAME] = fhdr[DSM_FIELD_ERR_FRAME];
    }
    const int j = blockIdx.x * HEAD_PLAN_WARPS + warp;
    if (j >= n) return;
    const DsmHeadingTraj T = traj[j];
    const int S = T.n_samples, base = T.sample0, m = T.max_step;
    long long(*val)[DSM_HEADING_MAX_ROTATIONS] = s_val[warp];
    int(*steps)[DSM_HEADING_MAX_ROTATIONS] = s_steps[warp];
    for (int s = lane; s < S; s += 32)
        for (int k = 0; k < 3; k++) out[base + s].p[k] = smp[base + s].p[k];
    auto score = [&](int s, int r) {
        const dsm_heading_count_t c = counts[(size_t)(base + s) * n_rot + r];
        return w_unknown * c.n_unknown + w_frontier * c.n_frontier;
    };
    // the last sample: its own score where the sequence may end
    for (int r = lane; r < n_rot; r += 32)
    {
        val[(S - 1) & 1][r] = T.end < 0 || r == T.end ? score(S - 1, r) : HEAD_NONE;
        steps[(S - 1) & 1][r] = 0;
    }
    __syncwarp();
    for (int s = S - 2; s >= 0; s--)
    {
        const long long *vn = val[(s + 1) & 1];
        const int *sn = steps[(s + 1) & 1];
        for (int r = lane; r < n_rot; r += 32)
        {
            long long bv = HEAD_NONE;
            int bs = 0, bd = 0;
            for (int i = 0; i <= 2 * m; i++)
            {
                const int d = i & 1 ? -((i + 1) >> 1) : i >> 1; // 0, -1, +1, -2, +2, ...
                int q = (r + d) % n_rot;
                q += q < 0 ? n_rot : 0;
                const long long cv = vn[q];
                if (cv == HEAD_NONE) continue;
                const int cs = sn[q] + abs(d);
                if (bv == HEAD_NONE || cv > bv || (cv == bv && cs < bs)) bv = cv, bs = cs, bd = d;
            }
            succ[(size_t)(base + s) * DSM_HEADING_MAX_ROTATIONS + r] = (int8_t)bd;
            val[s & 1][r] = bv == HEAD_NONE ? HEAD_NONE : score(s, r) + bv;
            steps[s & 1][r] = bs;
        }
        __syncwarp();
    }
    if (lane != 0) return;
    dsm_heading_t R;
    R.n_samples = S, R.sample_offset = base, R.n_outside = T.n_outside, R.reserved = 0;
    const long long v0 = val[0][T.start];
    R.status = v0 == HEAD_NONE ? 1 : 0;
    R.score = R.status ? 0 : v0;
    R.steps = R.status ? 0 : steps[0][T.start];
    int cur = T.start, turn = 0;
    for (int s = 0; s < S; s++)
    {
        out[base + s].rotation = R.status ? -1 : cur;
        out[base + s].turn = R.status ? 0 : turn;
        if (R.status || s + 1 == S) continue;
        const int d = succ[(size_t)(base + s) * DSM_HEADING_MAX_ROTATIONS + cur];
        turn += d;
        cur = (cur + d) % n_rot;
        cur += cur < 0 ? n_rot : 0;
    }
    rec[j] = R;
    atomicAdd(&hdr[DSM_HEAD_N_STATUS + R.status], 1);
}

// The sections of a staged request at `base` (the pinned staging or its device twin) and of a result at `base` (the
// device result or its pinned copy), for n trajectories and S samples
struct HeadStage
{
    double *rot;
    DsmHeadingTraj *traj;
    DsmHeadingSample *smp;
};
static HeadStage head_stage(uint8_t *base, int n)
{
    HeadStage h;
    h.rot = reinterpret_cast<double *>(base);
    h.traj = reinterpret_cast<DsmHeadingTraj *>(base + 72 * (size_t)DSM_HEADING_MAX_ROTATIONS);
    h.smp = reinterpret_cast<DsmHeadingSample *>(h.traj + n);
    return h;
}
struct HeadResult
{
    int32_t *hdr;
    dsm_heading_t *rec;
    dsm_heading_sample_t *out;
    dsm_heading_count_t *counts;
};
static HeadResult head_result(uint8_t *base, int n, int S)
{
    HeadResult r;
    r.hdr = reinterpret_cast<int32_t *>(base);
    r.rec = reinterpret_cast<dsm_heading_t *>(base + 4 * DSM_HEAD_WORDS);
    r.out = reinterpret_cast<dsm_heading_sample_t *>(r.rec + n);
    r.counts = reinterpret_cast<dsm_heading_count_t *>(r.out + S);
    return r;
}
static size_t head_stage_bytes(int n, int S)
{
    return 72 * (size_t)DSM_HEADING_MAX_ROTATIONS + sizeof(DsmHeadingTraj) * (size_t)n + sizeof(DsmHeadingSample) * (size_t)S;
}
static size_t head_res_bytes(int n, int S, int n_rot)
{
    return 4 * (size_t)DSM_HEAD_WORDS + sizeof(dsm_heading_t) * (size_t)n + (sizeof(dsm_heading_sample_t) + sizeof(dsm_heading_count_t) * (size_t)n_rot) * S;
}

extern "C" int dsm_heading_enable(dsm_ctx *ctx, int max_trajectories, int max_samples)
{
    if (!ctx) return DSM_E_INVALID;
    const DsmField *f = ctx->field.get();
    if (!f || !ctx->views || ctx->heading) return DSM_E_STATE;
    if (max_trajectories < 1 || max_trajectories > DSM_HEADING_MAX_CAPACITY || max_samples < 1 || max_samples > DSM_HEADING_MAX_CAPACITY)
        return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    auto hd = std::make_unique<DsmHeading>();
    hd->max_traj = max_trajectories, hd->max_samples = max_samples;
    const size_t stage = head_stage_bytes(max_trajectories, max_samples), res = head_res_bytes(max_trajectories, max_samples, DSM_HEADING_MAX_ROTATIONS);
    CudaOwner &o = hd->own;
    o.host(&hd->stage_host, stage);
    o.device(&hd->stage_dev, stage);
    o.device(&hd->succ, (size_t)DSM_HEADING_MAX_ROTATIONS * max_samples);
    o.device(&hd->res, res);
    o.host(&hd->res_host, res);
    o.event(&hd->ev);
    return keep(ctx->heading, hd);
}

// Sample s of the uniform cubic B-spline Q[N][3] at K samples per segment (include/dsm.h: the final-check samples of a
// trajectory job), each operation rounded once (the host code is built without contraction)
static void spline_sample(const double *Q, int N, int K, int s, double p[3])
{
    const int m = std::min(s / K, N - 4);
    const double u = (double)(s - m * K) / (double)K, u2 = u * u, u3 = u2 * u, w = 1.0 - u;
    const double b0 = ((w * w) * w) / 6.0, b1 = ((3.0 * u3 - 6.0 * u2) + 4.0) / 6.0, b2 = (((3.0 * u2 - 3.0 * u3) + 3.0 * u) + 1.0) / 6.0,
                 b3 = u3 / 6.0;
    const double *q = Q + 3 * (size_t)m;
    for (int k = 0; k < 3; k++) p[k] = ((b0 * q[k] + b1 * q[3 + k]) + b2 * q[6 + k]) + b3 * q[9 + k];
}

// Stages the request on the calling thread (checking it on the way): per sample its position and the hull of gain's
// boxes over the rotations, then enqueues one H2D copy, the kernels on the state grid of the latest (known) field
// request, one D2H copy of the used result and the event.  Later field requests overwrite that grid only behind the job.
extern "C" int dsm_heading_enqueue(dsm_ctx *ctx, const double *points, const int32_t *offsets, int n_trajectories, const dsm_gain_camera_t *camera,
                                   const double *rotations, int n_rot, int samples, const dsm_heading_request_t *requests, int32_t w_unknown,
                                   int32_t w_frontier)
{
    if (!ctx) return DSM_E_INVALID;
    DsmHeading *hd = ctx->heading.get();
    const DsmField *f = known_field(ctx);
    if (!hd || !f || hd->in_flight) return DSM_E_STATE;
    if (!points || !offsets || !camera || !rotations || !requests || n_trajectories < 1 || n_trajectories > hd->max_traj) return DSM_E_INVALID;
    const dsm_gain_camera_t &c = *camera;
    const double v = (double)f->g.voxel;
    if (!gain_camera_ok(c, v) || n_rot < 1 || n_rot > DSM_HEADING_MAX_ROTATIONS || samples < 1 || samples > DSM_HEADING_MAX_SAMPLES_PER_SEGMENT ||
        w_unknown < 0 || w_unknown > DSM_HEADING_MAX_WEIGHT || w_frontier < 0 || w_frontier > DSM_HEADING_MAX_WEIGHT)
        return DSM_E_INVALID;
    for (size_t i = 0; i < 9 * (size_t)n_rot; i++)
        if (!std::isfinite(rotations[i])) return DSM_E_INVALID;
    if (!spline_points_ok(points, offsets, n_trajectories, INT32_MAX)) return DSM_E_INVALID;
    long long n_samples = 0;
    for (int j = 0; j < n_trajectories; j++)
    {
        const dsm_heading_request_t &q = requests[j];
        if (q.start < 0 || q.start >= n_rot || q.end < -1 || q.end >= n_rot || q.max_step < 0 || q.max_step > n_rot) return DSM_E_INVALID;
        n_samples += (long long)samples * (offsets[j + 1] - offsets[j] - 3) + 1;
    }
    const long long m = 2 * (long long)std::ceil((double)c.max_range / v) + 3;
    if (n_samples > hd->max_samples || n_samples * m * m * m > DSM_HEADING_MAX_WORK) return DSM_E_INVALID;
    // the packed request; the previous job's copy out of this staging ended before its wait, which no job in flight
    // implies
    const HeadStage h = head_stage(hd->stage_host, n_trajectories);
    std::memcpy(h.rot, rotations, 72 * (size_t)n_rot);
    long long bricks = 0;
    int s0 = 0;
    for (int j = 0; j < n_trajectories; j++)
    {
        const int N = offsets[j + 1] - offsets[j], S = samples * (N - 3) + 1;
        DsmHeadingTraj &T = h.traj[j];
        T.sample0 = s0, T.n_samples = S, T.start = requests[j].start, T.end = requests[j].end, T.max_step = requests[j].max_step;
        T.n_outside = 0;
        for (int s = 0; s < S; s++)
        {
            DsmHeadingSample &Z = h.smp[s0 + s];
            spline_sample(points + 3 * (size_t)offsets[j], N, samples, s, Z.p);
            Z.pad = 0;
            bool inside = true;
            for (int k = 0; k < 3; k++)
            {
                const double q = std::floor(Z.p[k] / v) - (double)f->g.o[k];
                inside = inside && q >= 0.0 && q < (double)f->g.n[k];
            }
            int lo[3] = {INT32_MAX, INT32_MAX, INT32_MAX}, hi[3] = {-1, -1, -1}; // the hull, exclusive of hi
            for (int r = 0; inside && r < n_rot; r++)
            {
                DsmGainView V;
                for (int a = 0; a < 3; a++)
                {
                    for (int b = 0; b < 3; b++) V.P[4 * a + b] = rotations[9 * r + 3 * a + b];
                    V.P[4 * a + 3] = Z.p[a];
                }
                gain_box(V.P, c, f->g, V);
                if (V.size[0] == 0 || V.size[1] == 0 || V.size[2] == 0) continue;
                for (int k = 0; k < 3; k++) lo[k] = std::min(lo[k], V.lo[k]), hi[k] = std::max(hi[k], V.lo[k] + V.size[k]);
            }
            T.n_outside += !inside;
            for (int k = 0; k < 3; k++)
            {
                Z.lo[k] = hi[k] < 0 ? 0 : lo[k];
                Z.size[k] = hi[k] < 0 ? 0 : hi[k] - lo[k];
            }
            Z.brick0 = (int)bricks; // below 2^31: the work bound caps the bricks far lower
            bricks += dsm_gain_bricks(Z.size);
        }
        s0 += S;
    }
    CK(cudaSetDevice(ctx->device));
    const cudaStream_t st = ctx->stream;
    const int n = n_trajectories;
    CK(cudaMemcpyAsync(hd->stage_dev, hd->stage_host, head_stage_bytes(n, s0), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(hd->res, 0, head_res_bytes(n, s0, n_rot), st));
    const HeadStage d = head_stage(hd->stage_dev, n);
    const HeadResult r = head_result(hd->res, n, s0);
    const double R = (double)c.max_range;
    if (bricks > 0)
        k_heading_views<<<(unsigned)bricks, HEAD_BLOCK, 0, st>>>(f->g, f->occ, d.smp, s0, d.rot, n_rot, c.fx, c.fy, c.cx, c.cy, (double)c.width,
                                                                 (double)c.height, R * R, c.unknown_blocks, r.counts);
    k_heading_plan<<<(unsigned)((n + HEAD_PLAN_WARPS - 1) / HEAD_PLAN_WARPS), HEAD_PLAN_WARPS * 32, 0, st>>>(
        f->g, f->dist + dsm_field_header(f->voxels), d.traj, n, d.smp, s0, n_rot, c.unknown_blocks, w_unknown, w_frontier, r.counts, hd->succ,
        r.hdr, r.rec, r.out);
    CK(cudaGetLastError());
    hd->n = n, hd->n_samples = s0, hd->n_rot = n_rot;
    return submit(ctx, *hd, hd->res, head_res_bytes(n, s0, n_rot), f->requests);
}

extern "C" int dsm_heading_wait(dsm_ctx *ctx, dsm_heading_info_t *info, const dsm_heading_t **records, const dsm_heading_sample_t **samples,
                                const dsm_heading_count_t **counts)
{
    if (!ctx) return DSM_E_INVALID;
    DsmHeading *hd = ctx->heading.get();
    const int rc = wait_head(ctx, hd);
    if (rc != DSM_OK) return rc;
    copy_info(info, hd->words());
    const HeadResult r = head_result(hd->res_host, hd->n, hd->n_samples);
    if (records) *records = r.rec;
    if (samples) *samples = r.out;
    if (counts) *counts = r.counts;
    return capacity(ctx, hd->words(), DSM_HEAD_ERR_TAG, "dsm_heading_wait", "the field the job read");
}
