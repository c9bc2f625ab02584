"""Output side of the path (SURVEY.md §8f row 4): the PCD / PLY writers of the C ABI against the numpy
restatement of SurfelMap::save_cloud / save_mesh, and (on the GPU) the device-side cloud export of the
resident pool.  The writers are host code: their tests need no GPU."""
import os

import numpy as np
import pytest

import pyoracle
from densesurfelmapping_b200 import capi, synth
from densesurfelmapping_b200.elements import POINT_DTYPE, SURFEL_DTYPE


def random_surfels(n, seed=0):
    rng = np.random.RandomState(seed)
    s = np.zeros(n, SURFEL_DTYPE)
    for f in ("px", "py", "pz"):
        s[f] = rng.uniform(-40, 40, n)
    nr = rng.normal(size=(n, 3))
    nr /= np.linalg.norm(nr, axis=1, keepdims=True)
    s["nx"], s["ny"], s["nz"] = nr[:, 0], nr[:, 1], nr[:, 2]
    s["size"] = rng.uniform(0.01, 0.6, n)
    s["color"] = rng.randint(0, 256, n) + rng.choice([0.0, 0.25, 0.75], n)  # averaged intensities are not integers
    s["weight"] = rng.uniform(0.01, 30, n)
    s["update_times"] = rng.randint(0, 12, n)
    s["last_update"] = rng.randint(0, 9, n)
    if n >= 4:
        s["nx"][0], s["ny"][0], s["nz"][0] = 0, 0, 1    # x_dir = 0: normalize() must leave it alone, not make NaN
        s["nx"][1], s["ny"][1], s["nz"][1] = 1, 0, 0
        s["px"][2], s["py"][2], s["pz"][2] = 1e-7, -123456.78, 3.0e5  # exponent formats in %g
        s["size"][3] = 0
    return s


def test_mesh_vertices_match_push_a_surfel():
    s = random_surfels(3000, 1)
    got = capi.mesh_vertices(s)
    want = pyoracle.mesh_vertices(s)
    assert got.shape == want.shape == (3000, 6, 6)
    assert np.isfinite(got).all()
    assert got.tobytes() == want.tobytes()  # same float operations in the same order: bit-identical
    # geometry: a planar regular hexagon of circumradius `size` centred on the surfel, perpendicular to its normal
    c = np.stack([s["px"], s["py"], s["pz"]], -1).astype(np.float64)
    nr = np.stack([s["nx"], s["ny"], s["nz"]], -1).astype(np.float64)
    ok = (np.hypot(s["nx"], s["ny"]) > 1e-3) & (np.abs(c).max(axis=1) < 100)  # float32 positions: skip the 3e5 m outlier
    d = got[:, :, :3].astype(np.float64) - c[:, None, :]
    r = np.linalg.norm(d, axis=2)
    assert np.allclose(r[ok], s["size"][ok, None], rtol=1e-4, atol=1e-4)
    assert np.abs(np.einsum("nkc,nc->nk", d, nr))[ok].max() < 1e-3


def test_ply_mesh_file_is_byte_identical_to_save_mesh(tmp_path):
    s = random_surfels(500, 2)
    path = tmp_path / "mesh.ply"
    capi.write_ply_mesh(str(path), s)
    got = path.read_bytes().decode()
    want = pyoracle.ply_mesh_text(s)
    assert got == want
    head = got.split("end_header\n")[0].splitlines()
    assert head[0] == "ply" and "element vertex 3000" in head and "element face 2000" in head
    # structural read-back: 3000 vertex rows of 6 numbers, 2000 faces over valid vertex ids
    body = got.split("end_header\n")[1].splitlines()
    verts = np.array([[float(x) for x in l.split()] for l in body[:3000]])
    faces = np.array([[int(x) for x in l.split()] for l in body[3000:]])
    assert verts.shape == (3000, 6) and faces.shape == (2000, 4)
    assert (faces[:, 0] == 3).all() and faces[:, 1:].min() == 0 and faces[:, 1:].max() == 2999
    assert (verts[:, 3] == verts[:, 4]).all() and (verts[:, 3] == np.floor(verts[:, 3])).all()
    # empty map: header only, like the reference
    capi.write_ply_mesh(str(path), np.zeros(0, SURFEL_DTYPE))
    assert path.read_text() == pyoracle.ply_mesh_text(np.zeros(0, SURFEL_DTYPE))


def test_pcd_file_matches_pcl_ascii_layout_and_round_trips(tmp_path):
    s = random_surfels(2000, 3)
    pts = pyoracle.cloud_points(s, 5)
    pts[7, 1] = np.nan
    pts[8, 2] = -np.nan
    pts[9, 0] = np.inf
    rec = np.zeros(len(pts), POINT_DTYPE)
    rec["x"], rec["y"], rec["z"], rec["intensity"] = pts.T
    path = tmp_path / "cloud.pcd"
    capi.write_pcd(str(path), rec)
    text = path.read_text()
    assert text == pyoracle.pcd_text(pts)
    lines = text.splitlines()
    assert lines[:11] == ["# .PCD v0.7 - Point Cloud Data file format", "VERSION 0.7", "FIELDS x y z intensity", "SIZE 4 4 4 4",
                          "TYPE F F F F", "COUNT 1 1 1 1", f"WIDTH {len(pts)}", "HEIGHT 1", "VIEWPOINT 0 0 0 1 0 0 0",
                          f"POINTS {len(pts)}", "DATA ascii"]
    back = np.array([[float(x) for x in l.split()] for l in lines[11:]], dtype=np.float32)
    assert back.shape == pts.shape
    fin = np.isfinite(pts)
    assert (np.isnan(back) == np.isnan(pts)).all()
    assert np.allclose(back[fin], pts[fin], rtol=1e-7, atol=0)  # 8 significant digits: at most 1 ulp off
    # binary flavour: same header, DATA binary, then the packed 16-byte records
    capi.write_pcd(str(path), rec, binary=True)
    raw = path.read_bytes()
    k = raw.index(b"DATA binary\n") + len(b"DATA binary\n")
    assert raw[:k].decode().splitlines()[:10] == lines[:10]
    assert raw[k:] == rec.tobytes()
    capi.write_pcd(str(path), np.zeros(0, POINT_DTYPE))
    assert path.read_text() == pyoracle.pcd_text(np.zeros((0, 4), np.float32))


def test_writers_report_errors(tmp_path):
    with pytest.raises(capi.DsmError) as e:
        capi.write_pcd(str(tmp_path / "no_such_dir" / "x.pcd"), np.zeros(3, POINT_DTYPE))
    assert e.value.code == -9
    with pytest.raises(capi.DsmError):
        capi.write_ply_mesh(str(tmp_path / "no_such_dir" / "x.ply"), random_surfels(3))
    L = capi.load_library()
    assert L.dsm_write_pcd(None, None, 0, 0) == -1
    assert L.dsm_write_pcd(os.fsencode(str(tmp_path / "a.pcd")), None, 5, 0) == -1
    assert L.dsm_strerror(-9).decode().startswith("file")


@pytest.mark.gpu
def test_pool_export_cloud_on_device(tmp_path):
    """publish_active_pointcloud / publish_neighbor_pointcloud / save_cloud on the resident pool: filter and
    compaction on the device, exact and in pool order; the pool itself stays untouched."""
    from util import oracle_for
    cam = synth.VGA
    orc = oracle_for(cam)
    pool = np.zeros(0, SURFEL_DTYPE)
    ctx = capi.Context(cam, max_batch=2, max_local_surfels=60000)
    ctx.pool_upload(pool)
    for t in range(7):  # same view seven times: most surfels reach update_times >= 5, later ones do not
        pose = synth.pose_stream(t // 3)
        gray, depth = synth.make_frame(cam, 700 + t // 3, pose)
        ctx.fuse_frame_resident(t // 2, gray, depth, pose)
    pool = ctx.pool_download()
    ut = pool["update_times"]
    assert (ut >= 5).sum() > 100 and (ut < 5).sum() > 100, "test pool does not exercise the filter"
    for min_ut in (5, 1, 3, 1000):
        want = pyoracle.cloud_points(pool, min_ut)
        got = ctx.pool_export_cloud(min_ut)
        assert got.dtype == POINT_DTYPE and got.tobytes() == want.tobytes(), f"min_update_times={min_ut}"
        sel = ctx.pool_export_surfels(min_ut)
        assert sel.tobytes() == pool[ut >= min_ut].tobytes()
    # truncated output: count reported in full, the first `cap` records written and nothing past them
    L = capi.load_library()
    import ctypes
    for fn, dtype, want in ((L.dsm_pool_export_cloud, POINT_DTYPE, pyoracle.cloud_points(pool, 5)),
                            (L.dsm_pool_export_surfels, SURFEL_DTYPE, pool[ut >= 5])):
        buf = np.frombuffer(b"\xab" * (12 * dtype.itemsize), dtype).copy()
        n = ctypes.c_int(0)
        assert fn(ctx.h, 5, buf.ctypes.data, 10, ctypes.byref(n)) == 0
        assert n.value == int((ut >= 5).sum()) and buf[:10].tobytes() == want[:10].tobytes()
        assert buf[10:].tobytes() == b"\xab" * (2 * dtype.itemsize)
    assert ctx.pool_download().tobytes() == pool.tobytes()
    # and straight into the reference's file: save_cloud == export(5) -> PCD
    path = tmp_path / "active.pcd"
    capi.write_pcd(str(path), ctx.pool_export_cloud(5))
    assert path.read_text() == pyoracle.pcd_text(pyoracle.cloud_points(pool, 5))
    # a further frame still works after the exports borrowed the alternate pool buffer
    gray, depth = synth.make_frame(cam, 709, synth.pose_stream(3))
    lo, no = orc.fuse(4, gray, depth, synth.pose_stream(3), pool)
    want_pool = pyoracle.fuse_map_poststep(lo, no)
    n_new = ctx.fuse_frame_resident(4, gray, depth, synth.pose_stream(3), want_count=True)
    assert n_new == len(no) and ctx.pool_size() == len(want_pool)
    ctx.close()
