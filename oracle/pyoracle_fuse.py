"""TEST INFRASTRUCTURE ONLY -- a host model of the last two stages of fuse_initialize_map: the surfel fuse
(fuse_surfels_kernel, fusion_functions.cpp:190-313; k_fuse in csrc/dsm_kernels.cu) and the surfel initialise
(initialize_surfels, :315-361; k_init_surfels), on a given seed table and label image.

Every operation is written out in np.float32 / np.float64 with the reference's promotions, vectorised over the pool
(elementwise numpy arithmetic rounds each operation once, as the scalar code does).  Matrix-vector products follow the
Eigen stand-in's column-by-column accumulation (oracle/shim/Eigen/Eigen; mat4_mul / mat3_mul of the kernel) and the
inverse pose is its adjugate-over-determinant inverse (inverse4f of csrc/dsm_capi.cu).  Besides the outputs the model
reports which branch each surfel and each seed took, so that tests can state which branches their inputs reach.

`mutation` names one deliberate mistake (see MUTATIONS); tests/test_fuse_model.py proves that each of them changes the
output on the committed inputs, which is what makes bit-for-bit agreement of the kernels with the model meaningful.
"""
import numpy as np

F32 = np.float32
F64 = np.float64
MAX_ANGLE_COS = 0.1  # fusion_functions.h:11
INT_MIN = -(2 ** 31)

# surfel outcomes, in the order fuse_surfels_kernel tests them
(UNSTABLE, DEAD, NEAR, FAR, BORDER, OCCLUDING, ZERO_NORMAL, LOW_VIEW_COS, TOO_NEAR, TOO_FAR, NORMAL_MISMATCH,
 FUSED_SHRUNK, FUSED_KEPT) = range(13)
OUTCOMES = ("unstable", "dead", "near", "far", "border", "occluding", "zero normal", "low view_cos", "too near",
            "too far", "normal mismatch", "fused, size shrunk", "fused, size kept")
# seed outcomes of initialize_surfels
S_MD_ZERO, S_FUSED, S_LOW_VIEW_COS, S_ZERO_NORMAL, S_EMITTED = range(5)
SEED_OUTCOMES = ("mean_depth == 0", "fused", "low view_cos", "zero normal", "emitted")

MUTATIONS = (
    "unstable_age<=", "unstable_times<=", "near<=", "far>=", "border_lo<=", "border_hi>=", "occlusion<=",
    "too_near<=", "too_far>=", "tol_float", "weight_float", "mat3_row_order", "mat4_row_order",
    "size_quotient_double", "normal_len_double", "init_ignores_fused", "ipose_transposed",
)


def inverse4f(m):
    """Eigen stand-in's Matrix4f::inverse() (oracle/shim/Eigen/Eigen:145-171; inverse4f of csrc/dsm_capi.cu):
    adjugate over determinant in float32, products and sums left to right.  m: column-major float32[16]."""
    m = [F32(v) for v in np.asarray(m, F32).reshape(16)]
    inv = [F32(0)] * 16
    inv[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10]
    inv[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10]
    inv[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9]
    inv[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9]
    inv[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10]
    inv[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10]
    inv[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9]
    inv[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9]
    inv[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6]
    inv[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6]
    inv[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5]
    inv[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5]
    inv[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6]
    inv[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6]
    inv[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5]
    inv[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5]
    det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12]
    inv_det = F32(1) / det
    return np.array([v * inv_det for v in inv], F32)


def _mat4_mul(m, x, y, z, w, row_order=False):
    """Matrix4f * Vector4f: r_i = ((m_i0 x + m_i1 y) + m_i2 z) + m_i3 w, column-major m (shim :50-61)."""
    if row_order:
        m = m.reshape(4, 4).T.reshape(16)
    return [((m[i] * x + m[4 + i] * y) + m[8 + i] * z) + m[12 + i] * w for i in range(4)]


def _mat3_mul(m, x, y, z, row_order=False):
    """pose.block<3,3>(0,0) * Vector3f: r_i = (m_i0 x + m_i1 y) + m_i2 z."""
    if row_order:
        m = m.reshape(4, 4).T.reshape(16)
    return [(m[i] * x + m[4 + i] * y) + m[8 + i] * z for i in range(3)]


def camera_f(cam):
    """float camera_f = (fabs(fx) + fabs(fy)) / 2.0 (:250, :350): ::fabs(double), sum and halving in double."""
    return F32((abs(F64(F32(cam.fx))) + abs(F64(F32(cam.fy)))) / 2.0)


def get_weight(md, in_float=False):
    """get_weight (:99-102): std::min(1.0 / depth / depth, 1.0) in double, returned as float; std::min(a, b) is
    (b < a) ? b : a, so a NaN weight stays NaN."""
    with np.errstate(all="ignore"):
        if in_float:
            w = F32(1) / md / md
            return np.where(F32(1) < w, F32(1), w).astype(F32)
        w = 1.0 / md.astype(F64) / md.astype(F64)
        return np.where(1.0 < w, 1.0, w).astype(F32)


def new_size(size, md, vc, cf, quotient_double=False):
    """size * fabs(mean_depth / (camera_f * view_cos)) (:305, :351): the quotient in float, ::fabs(double) and the
    product in double, rounded to float on assignment."""
    with np.errstate(all="ignore"):
        if quotient_double:  # a mutation of the model
            q = md.astype(F64) / (F64(cf) * vc.astype(F64))
            return (size.astype(F64) * np.abs(q)).astype(F32)
        q = md / (cf * vc)
        return (size.astype(F64) * np.abs(q.astype(F64))).astype(F32)


def _trunc_int(v):
    """int conversion of a double as the reference's x86-64 build does it (cvttsd2si): toward zero, and INT_MIN for
    NaN and anything outside the int range.  The kernel's saturating conversion differs only outside the range, where
    both results fail the border test."""
    ok = np.isfinite(v) & (v > -2147483649.0) & (v < 2147483648.0)
    out = np.full(v.shape, INT_MIN, np.int64)
    out[ok] = np.trunc(v[ok]).astype(np.int64)
    return out


def fuse(seeds, labels, depth, pose, ipose, cam, constants, ref, pool, mutation=None):
    """fuse_surfels_kernel then initialize_surfels on one frame.

    seeds: SEED_DTYPE[S] (their `fused` flags are taken as given; clear them for a fresh frame); labels: int32[H, W];
    depth: float32[H, W]; pose / ipose: column-major float32[16] (ipose = inverse4f(pose) for the reference's call);
    constants: (huber_range, baseline, disparity_error, min_tolerate_diff); ref: reference frame index; pool:
    SURFEL_DTYPE[n].  Returns a dict: pool (updated copy), fused (uint8[S]), new (SURFEL_DTYPE, seed order),
    outcome (int8[n], OUTCOMES), seed_outcome (int8[S], SEED_OUTCOMES), emit_seed (seed index of every new surfel)."""
    mut = mutation
    assert mut is None or mut in MUTATIONS, mut
    _, baseline, disparity_error, min_tol = (float(c) for c in constants)
    H, W = labels.shape
    fx, fy, cx, cy = F32(cam.fx), F32(cam.fy), F32(cam.cx), F32(cam.cy)
    fnear, ffar = F32(cam.near), F32(cam.far)
    cf = camera_f(cam)
    pose = np.asarray(pose, F32).reshape(16)
    ipose = np.asarray(ipose, F32).reshape(16)
    if mut == "ipose_transposed":
        ipose = ipose.reshape(4, 4).T.reshape(16)
    out = np.array(pool, copy=True)
    n = len(out)
    fused = np.array(seeds["fused"], np.uint8, copy=True)
    outcome = np.full(n, -1, np.int8)
    ref = int(ref)
    ut = out["update_times"].astype(np.int64)
    lu = out["last_update"].astype(np.int64)
    todo = np.ones(n, bool)

    def settle(mask, code, kill=False):
        nonlocal todo
        m = todo & mask
        outcome[m] = code
        if kill:
            out["update_times"][m] = 0
        todo = todo & ~m

    with np.errstate(all="ignore"):
        # remove unstable (:207-211)
        age, few = ref - lu, ut
        settle((age >= 5 if mut == "unstable_age<=" else age > 5) & (few <= 5 if mut == "unstable_times<=" else few < 5), UNSTABLE, True)
        settle(ut == 0, DEAD)                                                                            # :213-214
        pc = _mat4_mul(ipose, out["px"], out["py"], out["pz"], F32(1), mut == "mat4_row_order")         # :215-220
        z = pc[2]
        settle((z <= fnear) if mut == "near<=" else (z < fnear), NEAR)                                  # :221-222
        settle((z >= ffar) if mut == "far>=" else (z > ffar), FAR)
        nc = _mat3_mul(ipose, out["nx"], out["ny"], out["nz"], mut == "mat3_row_order")                 # :223-228
        pu = pc[0] * fx / z + cx                                                                         # :85-89, :234
        pv = pc[1] * fy / z + cy
        ui = _trunc_int(pu.astype(F64) + 0.5)                                                            # :235-236
        vi = _trunc_int(pv.astype(F64) + 0.5)
        lo_bad = (ui <= 1) | (vi <= 1) if mut == "border_lo<=" else (ui < 1) | (vi < 1)
        hi_bad = (ui >= W - 2) | (vi >= H - 2) if mut == "border_hi>=" else (ui > W - 2) | (vi > H - 2)
        settle(lo_bad | hi_bad, BORDER)                                                                  # :237-238
        uc, vc_ = np.clip(ui, 0, W - 1), np.clip(vi, 0, H - 1)
        dthr = depth[vc_, uc].astype(F64) - 1.0
        settle((z.astype(F64) <= dthr) if mut == "occlusion<=" else (z.astype(F64) < dthr), OCCLUDING, True)  # :239-243
        sp = labels[vc_, uc]                                                                             # :244
        s = seeds[sp]
        snx, sny, snz = s["norm_x"], s["norm_y"], s["norm_z"]
        settle((snx == 0) & (sny == 0) & (snz == 0), ZERO_NORMAL)                                        # :245-246
        svc = s["view_cos"]
        settle(svc.astype(F64) < MAX_ANGLE_COS, LOW_VIEW_COS)                                            # :247-248
        zz = z * z                                                                                       # :250-253
        if mut == "tol_float":
            tol = (zz / F32(baseline * F64(cf)) * F32(disparity_error)).astype(F32)
        else:
            tol = (zz.astype(F64) / (baseline * F64(cf)) * disparity_error).astype(F32)
        tol = np.where(tol.astype(F64) < min_tol, F32(min_tol), tol).astype(F32)
        md = s["mean_depth"]
        settle((z <= md - tol) if mut == "too_near<=" else (z < md - tol), TOO_NEAR)                     # :254-258
        settle((z >= md + tol) if mut == "too_far>=" else (z > md + tol), TOO_FAR)                       # :259-263
        ndc = (nc[0] * snx + nc[1] * sny) + nc[2] * snz                                                  # :265-267
        settle(ndc.astype(F64) < MAX_ANGLE_COS, NORMAL_MISMATCH, True)                                   # :268-272
        f = todo
        ow = out["weight"][f]                                                                            # :273-275
        nw = get_weight(md[f], mut == "weight_float")
        sw = ow + nw
        pw = _mat4_mul(pose, s["posi_x"][f], s["posi_y"][f], s["posi_z"][f], F32(1), mut == "mat4_row_order")  # :276-281
        fp = [(out[k][f] * ow + nw * pw[i]) / sw for i, k in enumerate(("px", "py", "pz"))]             # :282-284
        fn = [nc[0][f] * ow + nw * snx[f], nc[1][f] * ow + nw * sny[f], nc[2][f] * ow + nw * snz[f]]     # :285-287
        l2 = (fn[0] * fn[0] + fn[1] * fn[1]) + fn[2] * fn[2]
        nl = np.sqrt(l2.astype(F64)) if mut == "normal_len_double" else np.sqrt(l2).astype(F64)          # :288
        fn = [(v.astype(F64) / nl).astype(F32) for v in fn]                                              # :289-291
        nwd = _mat3_mul(pose, fn[0], fn[1], fn[2], mut == "mat3_row_order")                              # :292-296
        for i, k in enumerate(("px", "py", "pz")):                                                      # :297-304
            out[k][f] = fp[i]
        for i, k in enumerate(("nx", "ny", "nz")):
            out[k][f] = nwd[i]
        out["weight"][f] = sw
        out["color"][f] = s["mean_intensity"][f]
        ns = new_size(s["size"][f], md[f], svc[f], cf, mut == "size_quotient_double")                             # :305
        old = out["size"][f]
        shrink = ns < old                                                                                # :306-307
        out["size"][f] = np.where(shrink, ns, old)
        outcome[np.nonzero(f)[0]] = np.where(shrink, FUSED_SHRUNK, FUSED_KEPT)
        out["last_update"][f] = ref                                                                      # :308-310
        out["update_times"][f] = out["update_times"][f] + 1
        fused[sp[f]] = 1                                                                                 # :311
    assert (outcome >= 0).all()

    # initialize_surfels (:315-361), seeds in index order
    seed_outcome = np.full(len(seeds), -1, np.int8)
    left = np.ones(len(seeds), bool)
    for mask, code in ((seeds["mean_depth"] == 0, S_MD_ZERO),
                       (np.zeros(len(seeds), bool) if mut == "init_ignores_fused" else fused != 0, S_FUSED),
                       (seeds["view_cos"].astype(F64) < MAX_ANGLE_COS, S_LOW_VIEW_COS),
                       ((seeds["norm_x"] == 0) & (seeds["norm_y"] == 0) & (seeds["norm_z"] == 0), S_ZERO_NORMAL)):
        seed_outcome[left & mask] = code
        left &= ~mask
    seed_outcome[left] = S_EMITTED
    e = np.nonzero(left)[0]
    s = seeds[e]
    new = np.zeros(len(e), pool.dtype)
    with np.errstate(all="ignore"):
        pw = _mat4_mul(pose, s["posi_x"], s["posi_y"], s["posi_z"], F32(1), mut == "mat4_row_order")     # :331-340
        nw = _mat3_mul(pose, s["norm_x"], s["norm_y"], s["norm_z"], mut == "mat3_row_order")             # :335-341
        for i, k in enumerate(("px", "py", "pz")):
            new[k] = pw[i]
        for i, k in enumerate(("nx", "ny", "nz")):
            new[k] = nw[i]
        new["size"] = new_size(s["size"], s["mean_depth"], s["view_cos"], cf, mut == "size_quotient_double")      # :350-354
        new["color"] = s["mean_intensity"]                                                               # :355
        new["weight"] = get_weight(s["mean_depth"], mut == "weight_float")                               # :356
    new["update_times"] = 1                                                                              # :357-358
    new["last_update"] = ref
    return dict(pool=out, fused=fused, new=new, outcome=outcome, seed_outcome=seed_outcome, emit_seed=e,
                ui=ui, vi=vi, z=z, tol=tol, md=md, ndc=ndc, sp=sp)
