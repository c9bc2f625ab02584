// The trajectory job of dsm_trajectory_enqueue (DESIGN.md §8.17): L-BFGS with Armijo backtracking over the free control
// points of uniform cubic B-splines against the signed grid of the latest field request, then a dense clearance check
// of each optimised curve.
//
//   k_trajectory  one warp (one CTA) per trajectory.  Free point i (3 <= i < N - 3) belongs to lane (i - 3) mod 32, at
//                 most 8 per lane.  The control points x, the trial points xt, the gradients g and gt and the direction d
//                 live in shared memory (x and xt whole, since every cost term reads neighbouring points; the other
//                 three per free point); the (s, y) history lives in the enable-time scratch, each lane touching only
//                 its own points, and the scalars every lane needs (sᵀy, yᵀy, the two-loop alphas) in shared memory.
//                 Every sum over points is a lane-strided ordered sum followed by a __shfl_xor_sync butterfly, which
//                 leaves every lane with the same bits, so all control flow is warp-uniform and the result does not
//                 depend on the schedule.  Trajectories finish independently.
// Every fp64 step is an explicit _rn intrinsic (the library is built with -fmad=false), so the numpy restatement
// (oracle/pyoracle_trajectory.py) is bit-exact; the field samples are the fp32 signed point query of k_field_query<true>.
// The job's C ABI calls (dsm_trajectory_enable, _enqueue and _wait) follow the kernel.
//
// One staged request (H2D):
//   double points[n_points][3] | double dt[n] | int32 offsets[n + 1]
// and one packed result (D2H, 64 + 96 n + 24 n_points B):
//   int32 header[DSM_TRAJ_WORDS] | dsm_trajectory_t records[n] | double points[n_points][3]
// The header's first nine words are those of dsm_trajectory_info_t; its last two carry the signed grid's error words,
// cleared by dsm_trajectory_wait.
#include "dsm_ctx.hpp"
#include <climits>

enum
{
    DSM_TRAJ_ORIGIN = 0, // 3 words
    DSM_TRAJ_N = 3,
    DSM_TRAJ_N_POINTS,
    DSM_TRAJ_N_STATUS,   // 4 words: trajectories per status (zeroed before the launch; k_trajectory adds)
    DSM_TRAJ_ERR_TAG = 14, // the signed grid header's DSM_SIGNED_ERR_TAG / _ERR_FRAME, copied by k_trajectory
    DSM_TRAJ_ERR_FRAME,
    DSM_TRAJ_WORDS = 16 // 64 B
};

#define TRAJ_C1 1e-4
// Every per-free-point array (g, gt, d and the history) is touched only by the lane that owns the free point: lane
// f mod 32 owns free point f and its three words c = 3 f .. 3 f + 2, in traj_eval, traj_dot and the vector loops alike.
// So only x and xt, which every cost term reads at neighbouring points, are shared between lanes, and each write to them
// is followed by a __syncwarp before another lane reads it.
#define TRAJ_OWNED(c) \
    for (int f_ = lane; f_ < M; f_ += 32) \
        for (int c = 3 * f_; c < 3 * f_ + 3; c++)

static_assert(sizeof(dsm_trajectory_params_t) == 88 && sizeof(dsm_trajectory_t) == 96 && sizeof(dsm_trajectory_info_t) == 64,
              "dsm_trajectory layouts");

__device__ __forceinline__ double traj_sum(double a)
{
    for (int k = 16; k > 0; k >>= 1) a = __dadd_rn(a, __shfl_xor_sync(0xffffffffu, a, k));
    return a;
}
__device__ __forceinline__ double traj_max(double a)
{
    for (int k = 16; k > 0; k >>= 1) a = fmax(a, __shfl_xor_sync(0xffffffffu, a, k));
    return a;
}
__device__ __forceinline__ int traj_count(int a)
{
    for (int k = 16; k > 0; k >>= 1) a += __shfl_xor_sync(0xffffffffu, a, k);
    return a;
}
// ((a_x b_x + a_y b_y) + a_z b_z) of one point
__device__ __forceinline__ double traj_dot3(const double *a, const double *b)
{
    return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}
// the reduction of traj_dot3 over the M free points of two per-free-point arrays
__device__ __forceinline__ double traj_dot(const double *a, const double *b, int M, int lane)
{
    double s = 0.0;
    for (int f = lane; f < M; f += 32) s = __dadd_rn(s, traj_dot3(a + 3 * f, b + 3 * f));
    return traj_sum(s);
}
// axis k of the jerk term m: (x[m+3] - x[m]) + 3 (x[m+1] - x[m+2])
__device__ __forceinline__ double traj_jerk(const double *x, int m, int k)
{
    return __dadd_rn(__dsub_rn(x[3 * (m + 3) + k], x[3 * m + k]), __dmul_rn(3.0, __dsub_rn(x[3 * (m + 1) + k], x[3 * (m + 2) + k])));
}
__device__ __forceinline__ double traj_vel(const double *x, int m, int k, double dt)
{
    return __ddiv_rn(__dsub_rn(x[3 * (m + 1) + k], x[3 * m + k]), dt);
}
__device__ __forceinline__ double traj_acc(const double *x, int m, int k, double dt2)
{
    const double a = x[3 * m + k], b = x[3 * (m + 1) + k], c = x[3 * (m + 2) + k];
    return __ddiv_rn(__dsub_rn(__dsub_rn(c, b), __dsub_rn(b, a)), dt2);
}
// the penalty max(0, q^2 - lim2)^2 of one axis, and its derivative 4 t q (0 without a penalty)
__device__ __forceinline__ double traj_pen(double q, double lim2, double &dq)
{
    const double t = __dsub_rn(__dmul_rn(q, q), lim2);
    dq = t > 0.0 ? __dmul_rn(__dmul_rn(4.0, t), q) : 0.0;
    return t > 0.0 ? __dmul_rn(t, t) : 0.0;
}

struct TrajEval
{
    double J, Js, Jc, Jf;
    int n_out; // free points outside the grid
};

// The cost at x ([N][3]) and its gradient g ([M][3], one row per free point) per include/dsm.h
__device__ __forceinline__ TrajEval traj_eval(const double *x, double *g, int N, double dt, double dt2, const dsm_trajectory_params_t &p,
                                              double v2, double a2, const float *__restrict__ sdist, const DsmFieldGrid &fg, bool empty,
                                              float fill, int lane)
{
    double as = 0.0, av = 0.0, aa = 0.0, ac = 0.0, dq;
    int n_out = 0;
    for (int m = lane; m < N - 3; m += 32)
    {
        const double jx = traj_jerk(x, m, 0), jy = traj_jerk(x, m, 1), jz = traj_jerk(x, m, 2);
        as = __dadd_rn(as, __dadd_rn(__dadd_rn(__dmul_rn(jx, jx), __dmul_rn(jy, jy)), __dmul_rn(jz, jz)));
    }
    for (int m = lane; m < N - 1; m += 32)
        av = __dadd_rn(av, __dadd_rn(__dadd_rn(traj_pen(traj_vel(x, m, 0, dt), v2, dq), traj_pen(traj_vel(x, m, 1, dt), v2, dq)),
                                     traj_pen(traj_vel(x, m, 2, dt), v2, dq)));
    for (int m = lane; m < N - 2; m += 32)
        aa = __dadd_rn(aa, __dadd_rn(__dadd_rn(traj_pen(traj_acc(x, m, 0, dt2), a2, dq), traj_pen(traj_acc(x, m, 1, dt2), a2, dq)),
                                     traj_pen(traj_acc(x, m, 2, dt2), a2, dq)));
    for (int i = 3 + lane; i < N - 3; i += 32)
    {
        bool inside;
        const float4 s = q_sample<true>(sdist, fg, empty, fill, x[3 * i], x[3 * i + 1], x[3 * i + 2], inside);
        n_out += !inside;
        const double e = __dsub_rn(p.margin, (double)s.x);
        const bool hit = inside && e > 0.0; // +inf (no site) gives e = -inf
        if (hit) ac = __dadd_rn(ac, __dmul_rn(e, e));
        const double ce = __dmul_rn(-2.0, e);
        const double sg[3] = {(double)s.y, (double)s.z, (double)s.w};
#pragma unroll
        for (int k = 0; k < 3; k++)
        {
            // smoothness: the terms i-3 .. i holding x_i at coefficients 1, -3, 3, -1
            const double gs = __dmul_rn(2.0, __dsub_rn(__dadd_rn(__dsub_rn(traj_jerk(x, i - 3, k), __dmul_rn(3.0, traj_jerk(x, i - 2, k))),
                                                                 __dmul_rn(3.0, traj_jerk(x, i - 1, k))),
                                                       traj_jerk(x, i, k)));
            const double gc = hit ? __dmul_rn(ce, sg[k]) : 0.0;
            double v0, v1, a0, a1, a2d;
            traj_pen(traj_vel(x, i - 1, k, dt), v2, v0);
            traj_pen(traj_vel(x, i, k, dt), v2, v1);
            traj_pen(traj_acc(x, i - 2, k, dt2), a2, a0);
            traj_pen(traj_acc(x, i - 1, k, dt2), a2, a1);
            traj_pen(traj_acc(x, i, k, dt2), a2, a2d);
            const double gf = __dadd_rn(__ddiv_rn(__dsub_rn(v0, v1), dt), __ddiv_rn(__dadd_rn(__dsub_rn(a0, __dmul_rn(2.0, a1)), a2d), dt2));
            g[3 * (i - 3) + k] = __dadd_rn(__dadd_rn(__dmul_rn(p.w_smooth, gs), __dmul_rn(p.w_clear, gc)), __dmul_rn(p.w_feas, gf));
        }
    }
    TrajEval r;
    r.Js = traj_sum(as);
    r.Jc = traj_sum(ac);
    r.Jf = __dadd_rn(traj_sum(av), traj_sum(aa));
    r.J = __dadd_rn(__dadd_rn(__dmul_rn(p.w_smooth, r.Js), __dmul_rn(p.w_clear, r.Jc)), __dmul_rn(p.w_feas, r.Jf));
    r.n_out = traj_count(n_out);
    return r;
}

__global__ void __launch_bounds__(32, 1) k_trajectory(const double *__restrict__ pts, const double *__restrict__ dts, const int32_t *__restrict__ ofs,
                                                   int n_traj, int nmax, const float *__restrict__ sdist, const int32_t *__restrict__ fhdr,
                                                   const DsmFieldGrid fg, const dsm_trajectory_params_t p, double *__restrict__ hist,
                                                   uint8_t *__restrict__ res)
{
    extern __shared__ double s_traj[];
    __shared__ double s_alpha[DSM_TRAJECTORY_MAX_MEMORY], s_sy[DSM_TRAJECTORY_MAX_MEMORY], s_yy[DSM_TRAJECTORY_MAX_MEMORY];
    const int t = blockIdx.x, lane = threadIdx.x;
    int32_t *hdr = reinterpret_cast<int32_t *>(res);
    if (t == 0 && lane == 0)
    { // the field's origin and error words at its request travel with the job's results
        for (int k = 0; k < 3; k++) hdr[DSM_TRAJ_ORIGIN + k] = fg.o[k];
        hdr[DSM_TRAJ_N] = n_traj;
        hdr[DSM_TRAJ_N_POINTS] = ofs[n_traj];
        hdr[DSM_TRAJ_ERR_TAG] = fhdr[DSM_SIGNED_ERR_TAG];
        hdr[DSM_TRAJ_ERR_FRAME] = fhdr[DSM_SIGNED_ERR_FRAME];
    }
    const int o = ofs[t], N = ofs[t + 1] - o, M = N - 6, mem = p.memory;
    double *x = s_traj, *xt = x + 3 * nmax, *g = xt + 3 * nmax, *gt = g + 3 * nmax, *d = gt + 3 * nmax;
    for (int c = lane; c < 3 * N; c += 32) x[c] = xt[c] = pts[3 * (size_t)o + c];
    __syncwarp();
    float fill;
    const bool empty = q_empty<true>(fhdr, fill);
    const double dt = dts[t], dt2 = __dmul_rn(dt, dt);
    const double v2 = __dmul_rn(p.v_max, p.v_max), a2 = __dmul_rn(p.a_max, p.a_max);
    dsm_trajectory_t rec = {};
    if (empty && fill < 0.f)
        rec.status = 3; // no voxel of F: not optimised
    else
    {
        TrajEval cur = traj_eval(x, g, N, dt, dt2, p, v2, a2, sdist, fg, empty, fill, lane);
        rec.evaluations = 1;
        rec.cost_start = cur.J;
        double *hs = hist + (size_t)o * 6 * mem; // slot k: s at [2k][N][3], y at [2k + 1][N][3], by free point
        int h = 0, head = mem - 1;
        const double v = (double)fg.voxel;
        while (true)
        {
            double gmax = 0.0;
            TRAJ_OWNED(c) gmax = fmax(gmax, fabs(g[c]));
            if (traj_max(gmax) <= p.g_tol)
            {
                rec.status = 0;
                break;
            }
            if (rec.iterations == p.max_iter)
            {
                rec.status = 1;
                break;
            }
            bool steep = h == 0;
            double gd = 0.0;
            if (!steep)
            { // two-loop recursion: q (in d) from g, newest to oldest, then r = gamma q, oldest to newest, d = -r
                TRAJ_OWNED(c) d[c] = g[c];
                for (int tt = 0; tt < h; tt++)
                {
                    const int k = (head - tt + mem) % mem;
                    const double *S = hs + (size_t)(2 * k) * 3 * N, *Y = S + 3 * (size_t)N;
                    const double a = __dmul_rn(__ddiv_rn(1.0, s_sy[k]), traj_dot(S, d, M, lane));
                    if (lane == 0) s_alpha[k] = a;
                    TRAJ_OWNED(c) d[c] = __dsub_rn(d[c], __dmul_rn(a, Y[c]));
                }
                __syncwarp();
                const double gamma = __ddiv_rn(s_sy[head], s_yy[head]);
                TRAJ_OWNED(c) d[c] = __dmul_rn(gamma, d[c]);
                for (int tt = h - 1; tt >= 0; tt--)
                {
                    const int k = (head - tt + mem) % mem;
                    const double *S = hs + (size_t)(2 * k) * 3 * N, *Y = S + 3 * (size_t)N;
                    const double b = __dmul_rn(__ddiv_rn(1.0, s_sy[k]), traj_dot(Y, d, M, lane));
                    const double ab = __dsub_rn(s_alpha[k], b);
                    TRAJ_OWNED(c) d[c] = __dadd_rn(d[c], __dmul_rn(S[c], ab));
                }
                TRAJ_OWNED(c) d[c] = -d[c];
                gd = traj_dot(g, d, M, lane);
                if (!(gd < 0.0))
                {
                    h = 0; // not a descent direction: the history is dropped
                    steep = true;
                }
            }
            double step = 1.0;
            if (steep)
            {
                TRAJ_OWNED(c) d[c] = -g[c];
                gd = traj_dot(g, d, M, lane);
                step = __ddiv_rn(v, __dsqrt_rn(traj_dot(g, g, M, lane)));
            }
            bool accepted = false;
            TrajEval trial;
            for (int ls = 0; ls < p.max_ls; ls++)
            {
                TRAJ_OWNED(c) xt[9 + c] = __dadd_rn(x[9 + c], __dmul_rn(step, d[c]));
                __syncwarp();
                trial = traj_eval(xt, gt, N, dt, dt2, p, v2, a2, sdist, fg, empty, fill, lane);
                rec.evaluations++;
                if (trial.J <= __dadd_rn(cur.J, __dmul_rn(__dmul_rn(TRAJ_C1, step), gd)))
                {
                    accepted = true;
                    break;
                }
                step = __dmul_rn(step, 0.5);
                __syncwarp(); // every lane has read xt before it changes
            }
            if (!accepted)
            {
                rec.status = 2; // the last accepted point stays
                break;
            }
            // the pair (s, y) = (xt - x, gt - g), kept when sᵀy > 0 (in the slot after the newest, over the oldest)
            double sy = 0.0, yy = 0.0;
            for (int f = lane; f < M; f += 32)
            {
                double s3[3], y3[3];
#pragma unroll
                for (int k = 0; k < 3; k++)
                {
                    s3[k] = __dsub_rn(xt[3 * (f + 3) + k], x[3 * (f + 3) + k]);
                    y3[k] = __dsub_rn(gt[3 * f + k], g[3 * f + k]);
                }
                sy = __dadd_rn(sy, traj_dot3(s3, y3));
                yy = __dadd_rn(yy, traj_dot3(y3, y3));
            }
            sy = traj_sum(sy);
            yy = traj_sum(yy);
            if (sy > 0.0)
            {
                head = (head + 1) % mem;
                double *S = hs + (size_t)(2 * head) * 3 * N, *Y = S + 3 * (size_t)N;
                TRAJ_OWNED(c)
                {
                    S[c] = __dsub_rn(xt[9 + c], x[9 + c]);
                    Y[c] = __dsub_rn(gt[c], g[c]);
                }
                if (lane == 0) s_sy[head] = sy, s_yy[head] = yy;
                h = min(h + 1, mem);
            }
            double *sw = x;
            x = xt, xt = sw;
            sw = g;
            g = gt, gt = sw;
            cur = trial;
            rec.iterations++;
            __syncwarp();
        }
        rec.cost = cur.J;
        rec.smoothness = cur.Js;
        rec.clearance = cur.Jc;
        rec.feasibility = cur.Jf;
        rec.n_free_outside = cur.n_out;
    }
    // the returned points, their largest per-axis |V| and |A|, and the curve's samples
    double *out = reinterpret_cast<double *>(res + 4 * DSM_TRAJ_WORDS + sizeof(dsm_trajectory_t) * (size_t)n_traj) + 3 * (size_t)o;
    for (int c = lane; c < 3 * N; c += 32) out[c] = x[c];
    double mv = 0.0, ma = 0.0;
    for (int m = lane; m < N - 1; m += 32)
#pragma unroll
        for (int k = 0; k < 3; k++) mv = fmax(mv, fabs(traj_vel(x, m, k, dt)));
    for (int m = lane; m < N - 2; m += 32)
#pragma unroll
        for (int k = 0; k < 3; k++) ma = fmax(ma, fabs(traj_acc(x, m, k, dt2)));
    rec.max_v = traj_max(mv);
    rec.max_a = traj_max(ma);
    const int K = p.samples, total = (N - 3) * K + 1;
    const double dK = (double)K;
    float best = INFINITY;
    int arg = INT_MAX, hit = INT_MAX, outside = 0; // INT_MAX: none yet
    for (int s = lane; s < total; s += 32)
    {
        const int m = min(s / K, N - 4);
        const double u = __ddiv_rn((double)(s - m * K), dK);
        const double u2 = __dmul_rn(u, u), u3 = __dmul_rn(u2, u), w = __dsub_rn(1.0, u);
        const double b0 = __ddiv_rn(__dmul_rn(__dmul_rn(w, w), w), 6.0);
        const double b1 = __ddiv_rn(__dadd_rn(__dsub_rn(__dmul_rn(3.0, u3), __dmul_rn(6.0, u2)), 4.0), 6.0);
        const double b2 = __ddiv_rn(__dadd_rn(__dadd_rn(__dsub_rn(__dmul_rn(3.0, u2), __dmul_rn(3.0, u3)), __dmul_rn(3.0, u)), 1.0), 6.0);
        const double b3 = __ddiv_rn(u3, 6.0);
        double q[3];
#pragma unroll
        for (int k = 0; k < 3; k++)
        {
            const double *c = x + 3 * m + k;
            q[k] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(b0, c[0]), __dmul_rn(b1, c[3])), __dmul_rn(b2, c[6])), __dmul_rn(b3, c[9]));
        }
        bool inside;
        const float dd = q_sample<false>(sdist, fg, empty, fill, q[0], q[1], q[2], inside).x;
        if (!inside)
        {
            outside++;
            continue;
        }
        if (arg == INT_MAX || dd < best) best = dd, arg = s; // this lane's samples rise: the first minimum stays
        if (hit == INT_MAX && dd < p.radius) hit = s;
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
        rec.min_dist = best;
        rec.argmin = arg == INT_MAX ? -1 : arg;
        rec.first_hit = hit == INT_MAX ? -1 : hit;
        rec.n_outside = outside;
        reinterpret_cast<dsm_trajectory_t *>(res + 4 * DSM_TRAJ_WORDS)[t] = rec;
        atomicAdd(&hdr[DSM_TRAJ_N_STATUS + rec.status], 1);
    }
}

// byte offsets of the staged request's dt and offsets and its end, and of the result's points and its end
static size_t traj_stage_dt(int n_points) { return 24 * (size_t)n_points; }
static size_t traj_stage_offsets(int n_points, int n) { return traj_stage_dt(n_points) + 8 * (size_t)n; }
static size_t traj_stage_bytes(int n_points, int n) { return traj_stage_offsets(n_points, n) + 4 * ((size_t)n + 1); }
static size_t traj_points_at(int n) { return 4 * (size_t)DSM_TRAJ_WORDS + sizeof(dsm_trajectory_t) * (size_t)n; }
static size_t traj_res_bytes(int n_points, int n) { return traj_points_at(n) + 24 * (size_t)n_points; }

extern "C" int dsm_trajectory_enable(dsm_ctx *ctx, int max_trajectories, int max_points, int max_memory)
{
    if (!ctx) return DSM_E_INVALID;
    const DsmField *f = ctx->field.get();
    if (!f || !f->sgn || ctx->trajectory) return DSM_E_STATE;
    if (max_trajectories < 1 || max_trajectories > DSM_TRAJECTORY_MAX_CAPACITY || max_points < 1 || max_points > DSM_TRAJECTORY_MAX_CAPACITY ||
        max_memory < 1 || max_memory > DSM_TRAJECTORY_MAX_MEMORY)
        return DSM_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    auto tr = std::make_unique<DsmTrajectory>();
    tr->max_traj = max_trajectories, tr->max_points = max_points, tr->max_memory = max_memory;
    const size_t stage = traj_stage_bytes(max_points, max_trajectories), res = traj_res_bytes(max_points, max_trajectories);
    CudaOwner &o = tr->own;
    o.host(&tr->stage_host, stage);
    o.device(&tr->stage_dev, stage);
    o.device(&tr->hist, 6 * (size_t)max_memory * max_points);
    o.device(&tr->res, res);
    o.host(&tr->res_host, res);
    o.event(&tr->ev);
    return keep(ctx->trajectory, tr);
}

static bool traj_params_ok(const dsm_trajectory_params_t &p, int max_memory)
{
    for (double w : {p.w_smooth, p.w_clear, p.w_feas, p.margin, p.v_max, p.a_max, p.g_tol})
        if (!std::isfinite(w) || !(w >= 0.0)) return false;
    return p.max_iter >= 0 && p.max_iter <= DSM_TRAJECTORY_MAX_ITER && p.memory >= 1 && p.memory <= max_memory && p.max_ls >= 1 &&
           p.max_ls <= DSM_TRAJECTORY_MAX_LS && p.samples >= 1 && p.samples <= DSM_TRAJECTORY_MAX_SAMPLES_PER_SEGMENT &&
           std::isfinite(p.radius) && p.radius >= 0.f;
}

// Stages the request on the calling thread (checking it on the way), then enqueues one H2D copy, the kernel on the
// signed grid of the latest field request, one D2H copy of the used result and the event.
extern "C" int dsm_trajectory_enqueue(dsm_ctx *ctx, const double *points, const int32_t *offsets, const double *dt, int n_trajectories,
                                      const dsm_trajectory_params_t *params)
{
    if (!ctx) return DSM_E_INVALID;
    DsmTrajectory *tr = ctx->trajectory.get();
    const DsmField *f = ctx->field.get();
    if (!tr || !f || !f->requested || !f->signed_latest || tr->in_flight) return DSM_E_STATE;
    if (!points || !offsets || !dt || !params || n_trajectories < 1 || n_trajectories > tr->max_traj) return DSM_E_INVALID;
    const dsm_trajectory_params_t p = *params;
    if (!traj_params_ok(p, tr->max_memory) || !spline_points_ok(points, offsets, n_trajectories, tr->max_points)) return DSM_E_INVALID;
    int nmax = 0;
    unsigned long long samples = 0;
    for (int j = 0; j < n_trajectories; j++)
    {
        const int n = offsets[j + 1] - offsets[j];
        if (!std::isfinite(dt[j]) || !(dt[j] > 0.0)) return DSM_E_INVALID;
        nmax = std::max(nmax, n);
        samples += (unsigned long long)(n - 3) * (unsigned long long)p.samples + 1;
    }
    const int n_points = offsets[n_trajectories];
    if ((unsigned long long)n_points * (unsigned long long)p.max_iter * (unsigned long long)(p.max_ls + 1) > DSM_TRAJECTORY_MAX_WORK ||
        samples > DSM_TRAJECTORY_MAX_SAMPLES)
        return DSM_E_INVALID;
    // the packed request; the previous job's copy out of this staging ended before its wait, which no job in flight
    // implies
    uint8_t *h = tr->stage_host;
    std::memcpy(h, points, 24 * (size_t)n_points);
    std::memcpy(h + traj_stage_dt(n_points), dt, 8 * (size_t)n_trajectories);
    std::memcpy(h + traj_stage_offsets(n_points, n_trajectories), offsets, 4 * ((size_t)n_trajectories + 1));
    CK(cudaSetDevice(ctx->device));
    const cudaStream_t st = ctx->stream;
    CK(cudaMemcpyAsync(tr->stage_dev, h, traj_stage_bytes(n_points, n_trajectories), cudaMemcpyHostToDevice, st));
    const int32_t *grid = f->sgn->grid;
    CK(cudaMemsetAsync(tr->res, 0, 4 * DSM_TRAJ_WORDS, st));
    // k_trajectory's shared memory: x, xt, g, gt and d, nmax x 3 doubles each
    k_trajectory<<<n_trajectories, 32, 5 * 3 * sizeof(double) * (size_t)nmax, st>>>(
        reinterpret_cast<const double *>(tr->stage_dev), reinterpret_cast<const double *>(tr->stage_dev + traj_stage_dt(n_points)),
        reinterpret_cast<const int32_t *>(tr->stage_dev + traj_stage_offsets(n_points, n_trajectories)), n_trajectories, nmax,
        reinterpret_cast<const float *>(grid), grid + dsm_field_header(f->voxels), f->g, p, tr->hist, tr->res);
    CK(cudaGetLastError());
    tr->n = n_trajectories, tr->n_points = n_points;
    return submit(ctx, *tr, tr->res, traj_res_bytes(n_points, n_trajectories), f->requests);
}

extern "C" int dsm_trajectory_wait(dsm_ctx *ctx, dsm_trajectory_info_t *info, const dsm_trajectory_t **records, const double **points)
{
    if (!ctx) return DSM_E_INVALID;
    DsmTrajectory *tr = ctx->trajectory.get();
    const int rc = wait_head(ctx, tr);
    if (rc != DSM_OK) return rc;
    copy_info(info, tr->words());
    if (records) *records = reinterpret_cast<const dsm_trajectory_t *>(tr->res_host + 4 * DSM_TRAJ_WORDS);
    if (points) *points = reinterpret_cast<const double *>(tr->res_host + traj_points_at(tr->n));
    return capacity(ctx, tr->words(), DSM_TRAJ_ERR_TAG, "dsm_trajectory_wait", "the field the job read");
}
