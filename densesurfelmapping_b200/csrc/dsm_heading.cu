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
// carry no error gate and are launched without PDL, as the other field kernels.
#include "dsm_device.cuh"
#include <algorithm>
#include <climits>

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

cudaError_t dsm_launch_heading(const DsmFieldGrid &g, const uint8_t *state, const int32_t *dist, const dsm_gain_camera_t &cam,
                               const uint8_t *stage, int n, int n_samples, int n_rot, long long bricks, int w_unknown, int w_frontier,
                               int8_t *succ, uint8_t *res, cudaStream_t st)
{
    const size_t voxels = (size_t)g.n[0] * g.n[1] * g.n[2];
    const cudaError_t e = cudaMemsetAsync(res, 0, dsm_heading_res_bytes(n, n_samples, n_rot), st);
    if (e != cudaSuccess) return e;
    int32_t *hdr = reinterpret_cast<int32_t *>(res);
    auto *rec = reinterpret_cast<dsm_heading_t *>(res + 4 * DSM_HEAD_WORDS);
    auto *out = reinterpret_cast<dsm_heading_sample_t *>(rec + n);
    auto *counts = reinterpret_cast<dsm_heading_count_t *>(out + n_samples);
    const double *rot = reinterpret_cast<const double *>(stage);
    const auto *traj = reinterpret_cast<const DsmHeadingTraj *>(stage + 72 * (size_t)DSM_HEADING_MAX_ROTATIONS);
    const auto *smp = reinterpret_cast<const DsmHeadingSample *>(traj + n);
    const double R = (double)cam.max_range;
    if (bricks > 0)
        k_heading_views<<<(unsigned)bricks, HEAD_BLOCK, 0, st>>>(g, state, smp, n_samples, rot, n_rot, cam.fx, cam.fy, cam.cx, cam.cy,
                                                                 (double)cam.width, (double)cam.height, R * R, cam.unknown_blocks, counts);
    k_heading_plan<<<(unsigned)((n + HEAD_PLAN_WARPS - 1) / HEAD_PLAN_WARPS), HEAD_PLAN_WARPS * 32, 0, st>>>(
        g, dist + dsm_field_header(voxels), traj, n, smp, n_samples, n_rot, cam.unknown_blocks, w_unknown, w_frontier, counts, succ, hdr,
        rec, out);
    return cudaGetLastError();
}
