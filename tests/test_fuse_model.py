"""The host model of the surfel fuse and initialise (oracle/pyoracle_fuse.py) against the reference's own
fuse_initialize_map, bit for bit, on pools built to reach every branch (tests/fuse_inputs.py); the census of the
branches those pools reach; and the mutations of the model that the pools catch.  tests/test_gpu_fuse.py then holds
k_fuse and k_init_surfels bit for bit to the unmutated model on the same kind of pools."""
import functools

import numpy as np
import pytest

import fuse_inputs as fi
import pyoracle
import pyoracle_fuse as pf
from util import bits_equal_nan, canon

REF_FRAME = 9  # reference frame index of every crafted call


def _oracle(cam, cname):
    if pyoracle.have_reference():
        return (pyoracle.RefSerial if cname == "drive" else pyoracle.RefSerialRGBD)(cam)
    return pyoracle.Restatement(cam, fi.CONSTANTS[cname])


@functools.lru_cache(maxsize=None)
def _seeded(fname, cname):
    cam, gray, depth = fi.frame(fname)
    orc = _oracle(cam, cname)
    labels, seeds = orc.superpixels(gray, depth)
    return cam, gray, depth, labels, seeds


@functools.lru_cache(maxsize=None)
def _case(fname, cname, pname):
    cam, gray, depth, labels, seeds = _seeded(fname, cname)
    fr = fi.Frame(cam, seeds, labels, depth, fi.POSES[pname], fi.CONSTANTS[cname], REF_FRAME)
    pool, probes = fi.build(fr)
    return fr, pool, probes


@functools.lru_cache(maxsize=None)
def _init_case(cname, pattern):
    cam, gray, depth, labels, seeds = _seeded("hd", cname)
    fr = fi.Frame(cam, seeds, labels, depth, fi.POSES["general"], fi.CONSTANTS[cname], REF_FRAME)
    return fr, fi.init_pool(fr, pattern)


CASES = [(f, c, p) for f in fi.FRAMES for c in fi.CONSTANTS for p in fi.POSES]


def _against_reference(fname, cname, fr, pool):
    cam, gray, depth, _, _ = _seeded(fname, cname)
    orc = _oracle(cam, cname)
    want_pool, want_new = orc.fuse(REF_FRAME, gray, depth, fr.pose, pool)
    want_fused = orc.seeds()["fused"]
    got = fr.run(pool)
    assert canon(got["pool"]) == canon(want_pool), f"pool differs at {np.nonzero(~_rows_equal(got['pool'], want_pool))[0][:8]}"
    assert len(got["new"]) == len(want_new), f"{len(got['new'])} new surfels, the reference {len(want_new)}"
    assert canon(got["new"]) == canon(want_new), f"new surfels differ at {np.nonzero(~_rows_equal(got['new'], want_new))[0][:8]}"
    assert (got["fused"] == want_fused).all(), f"fused flags differ at {np.nonzero(got['fused'] != want_fused)[0][:8]}"


def _rows_equal(a, b):
    ok = np.ones(len(a), bool)
    for f in a.dtype.names:
        ok &= bits_equal_nan(a[f], b[f]) if a[f].dtype.kind == "f" else (a[f] == b[f])
    return ok


@pytest.mark.parametrize("fname,cname,pname", CASES)
def test_model_equals_reference(fname, cname, pname):
    """Updated pool, new surfels in seed order and fused flags equal the reference's bit for bit (NaN == NaN)."""
    fr, pool, _ = _case(fname, cname, pname)
    _against_reference(fname, cname, fr, pool)


@pytest.mark.parametrize("cname", list(fi.CONSTANTS))
@pytest.mark.parametrize("pattern", fi.INIT_PATTERNS)
def test_init_patterns(cname, pattern):
    """On the 1280 x 720 frame (15 CTAs of k_init_surfels) the chosen seeds are fused so the emitters follow the
    pattern around the CTA boundaries, and the model equals the reference."""
    fr, pool = _init_case(cname, pattern)
    r = fr.run(pool)
    e = r["emit_seed"]
    cap = np.zeros(len(fr.seeds), bool)
    cap[fr.usable()] = True
    if pattern == "none_before":
        assert (e >= fi.CTA).all() and (e < 2 * fi.CTA).any()
    elif pattern == "boundary_pair":
        pair = fi.boundary_pair(fr)
        assert e.tolist() == list(pair), e[:8]
    elif pattern == "alternating":
        assert (e[cap[e]] % 2 == 0).all() and (e % 2 == 0).sum() > 100
    else:
        assert not ((e >= 5 * fi.CTA) & (e < 6 * fi.CTA) & cap[e]).any()
        assert ((e >= 5 * fi.CTA) & (e < 6 * fi.CTA)).sum() <= 8
    _against_reference("hd", cname, fr, pool)


# Outcomes a frame cannot reach, with the reason.
UNREACHABLE = {
    # every depth is under 1 m, so depth - 1.0 < 0 < fuse_near: no surfel past the near cut can occlude a measurement
    "near": {pf.OCCLUDING},
}


def test_census_every_outcome_on_every_frame():
    """Every surfel outcome and every seed outcome is reached on each frame (both constant sets and poses together),
    but for the stated exceptions; at every threshold both neighbouring floats are in the pool and take different
    branches."""
    report = []
    for fname in fi.FRAMES:
        seen, seen_seed, thr = set(), set(), set()
        for cname in fi.CONSTANTS:
            for pname in fi.POSES:
                fr, pool, probes = _case(fname, cname, pname)
                r = fr.run(pool)
                seen |= set(r["outcome"].tolist())
                seen_seed |= set(r["seed_outcome"].tolist())
                for name, pairs in probes.items():
                    for i, j in pairs:
                        assert r["outcome"][i] != r["outcome"][j], f"{fname}/{cname}/{pname} {name}: same branch"
                    # the pair is a pair of neighbouring floats in exactly one field
                    for i, j in pairs:
                        d = [f for f in pool.dtype.names if not bits_equal_nan(pool[f][i], pool[f][j])]
                        assert len(d) == 1, (name, d)
                        k = d[0]
                        assert np.nextafter(pool[k][i], pool[k][j]) == pool[k][j], (name, k, pool[k][i], pool[k][j])
                    if pairs:
                        thr.add(name.split(" (")[0])
        want = set(range(len(pf.OUTCOMES))) - UNREACHABLE.get(fname, set())
        assert want <= seen, f"{fname}: outcomes not reached: {[pf.OUTCOMES[o] for o in sorted(want - seen)]}"
        # a seed the plane fit rejects (zero normal) has view_cos 0, and initialize_surfels tests view_cos first
        assert seen_seed >= set(range(len(pf.SEED_OUTCOMES))) - {pf.S_ZERO_NORMAL}, fname
        for cname in fi.CONSTANTS:
            sd = _seeded(fname, cname)[4]
            zero = (sd["norm_x"] == 0) & (sd["norm_y"] == 0) & (sd["norm_z"] == 0)
            assert (sd["view_cos"][zero] == 0).all()
        want_thr = {"near", "far", "too_near", "too_far", "ndc", "u 0|1", "u W-2|W-1", "v 0|1", "v H-2|H-1", "size"}
        if pf.OCCLUDING not in UNREACHABLE.get(fname, set()):
            want_thr.add("occlusion")
        assert want_thr <= thr, f"{fname}: thresholds without a pair: {sorted(want_thr - thr)}"
        report.append(f"{fname}: {len(seen)} outcomes, {len(seen_seed)} seed outcomes, {len(thr)} thresholds")
    # the tolerance threshold on both sides of the min_tolerate_diff clamp, for each constant set
    for cname in fi.CONSTANTS:
        sides = set()
        for fname in fi.FRAMES:
            for pname in fi.POSES:
                sides |= {n for n, p in _case(fname, cname, pname)[2].items() if p and n.startswith("too_")}
        assert sides == {f"{n} ({s})" for n in ("too_near", "too_far") for s in ("clamped", "computed")}, (cname, sides)
    print("\n".join(report))


def test_stability_and_odd_surfels():
    """ref - last_update at 5 and 6 with update_times 4 and 5 (only 6 / 4 is unstable), update_times 0, projections
    outside the image and the int range, NaN and infinite positions, and a NaN normal that fuses and spreads NaN."""
    fr, pool, _ = _case("vga", "drive", "general")
    r = fr.run(pool)
    o = r["outcome"]
    age = REF_FRAME - pool["last_update"]
    for a, t, want_unstable in ((5, 4, False), (5, 5, False), (6, 4, True), (6, 5, False)):
        sel = (age == a) & (pool["update_times"] == t)
        assert sel.any() and ((o[sel] == pf.UNSTABLE) == want_unstable).all(), (a, t)
    assert (o[pool["update_times"] == 0] <= pf.DEAD).all() and (o == pf.DEAD).any()
    with np.errstate(invalid="ignore"):
        bad = ~np.isfinite(pool["px"]) | ~np.isfinite(pool["py"]) | ~np.isfinite(pool["pz"])
    assert bad.sum() >= 7 and np.isin(o[bad], [pf.NEAR, pf.FAR, pf.BORDER]).all()
    assert (np.abs(r["ui"]) >= 2 ** 31 - 1).any() or (r["ui"] == pf.INT_MIN).any()
    nan_n = np.isnan(pool["nx"])
    assert nan_n.sum() == 1 and o[nan_n][0] >= pf.FUSED_SHRUNK and np.isnan(r["pool"]["nx"][nan_n]).all()
    # mean depths on both sides of get_weight's clamp among the fused surfels
    mds = np.concatenate([_case(f, "drive", "identity")[0].run(_case(f, "drive", "identity")[1])["md"] for f in ("vga", "near")])
    assert (mds[np.isfinite(mds)] < 1).any() and (mds[np.isfinite(mds)] > 1).any()


def test_inverse_pose_is_the_adjugate_rule():
    """inverse4f restates the Eigen stand-in's inverse: the general pose's inverse times the pose is the identity to
    float rounding, and the reference's fuse under that pose (test_model_equals_reference) pins it bit for bit."""
    p = fi.POSES["general"].reshape(4, 4).T.astype(np.float64)
    q = pf.inverse4f(fi.POSES["general"]).reshape(4, 4).T.astype(np.float64)
    assert np.abs(q @ p - np.eye(4)).max() < 1e-6


# Mutations left out because they provably cannot change the output on any input the frames allow:
#   `(double)ndc < 0.1` and `view_cos < 0.1` as `<=`, or as float compares: 0.1 is not a float and no float lies
#     between 0.1 and 0.1f, so every float compares alike;
#   `(double)tol < min_tolerate_diff` as `<=`: neither 0.1 nor 0.05 is a float;
#   `(int)(pu + 0.5f)` in float: pu = x fx / z + cx with cx = 319.5, 601.8873 or 639.5 lies, near the border
#     columns, on a grid no finer than 2^-15, where pu + 0.5 is exact in float; it differs from the double sum only
#     beyond 2^23, far outside the image;
#   `new_size < size` as `<=`: on equality both keep the same size;
#   the size product in float: a product of two floats is exact in double, so rounding it once to float is the
#     float product;
#   dropping `fabs` from the size: mean_depth > 0 and view_cos >= 0.1 on every path that reaches it.
@pytest.mark.parametrize("mutation", pf.MUTATIONS)
def test_mutation_is_caught(mutation):
    """Each single mutation of the model changes the output (pool, new surfels or fused flags) on the committed
    inputs: the same inputs would catch that mistake in the kernels."""
    combos = [("case",) + c for c in CASES] + [("init", c, p) for c in fi.CONSTANTS for p in fi.INIT_PATTERNS]
    for combo in combos:
        fr, pool = (_case(*combo[1:])[:2] if combo[0] == "case" else _init_case(*combo[1:]))
        a, b = fr.run(pool), fr.run(pool, mutation)
        if (canon(a["pool"]) != canon(b["pool"]) or canon(a["new"]) != canon(b["new"])
                or not (a["fused"] == b["fused"]).all()):
            return
    pytest.fail(f"mutation {mutation} changes nothing on the committed inputs")
