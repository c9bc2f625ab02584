"""include/dsm_surfel_node.hpp: dsm::SurfelMapNode, the reference's SurfelMap node callback for callback.

CPU: tests/cpp/node_main.cpp with no context (pose logic only) against the reference's own SurfelMap
(pyoracle_window.RefMapWindow, libdsm_refmap_window.so) fed the same messages: after every message the local window, the
pending fuse pose (bit for bit), the window lists from every root and the active loop-closure warp (bit for bit, read
through probe surfels) agree.  The GPU half is tests/test_gpu_surfel_node.py."""
import subprocess

import numpy as np
import pytest

import pyoracle_window
from densesurfelmapping_b200 import synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE
from node_drive import Script, build_adapter, drive, read_dumps, run_node

needs_window_oracle = pytest.mark.skipif(not pyoracle_window.have_refmap_window(),
                                         reason="oracle/_ref/libdsm_refmap_window.so not built (needs the reference sources)")

SMALL = synth.Camera(64, 48, 52.5, 52.5, 31.5, 23.5, 0.5, 30.0)   # pose logic only: images count for their stamps


PROBE_W = 3


def probe_surfels():
    """Three surfels at the origin with normals e_x, e_y, e_z: the active warp W moves them to W[:3, 3] and W[:3, j]
    exactly (every other product is a zero), so W's top three rows can be read back bit for bit."""
    s = np.zeros(PROBE_W, SURFEL_DTYPE)
    s["nx"][0], s["ny"][1], s["nz"][2] = 1, 1, 1
    s["update_times"], s["last_update"], s["size"] = 1, 10 ** 6, 1
    return s


def probe_warp(local):
    W = np.zeros((4, 4), np.float32)
    W[:3, 3] = [local["px"][0], local["py"][0], local["pz"][0]]
    for j, f in enumerate(("nx", "ny", "nz")):
        W[:3, j] = [local["nx"][j], local["ny"][j], local["nz"][j]]
    return W


# ---- CPU: pose logic against the reference node ----
@needs_window_oracle
@pytest.mark.parametrize("drift_free_poses", [1, 2, 10])
def test_pose_logic_equals_the_reference_node(tmp_path, drift_free_poses):
    cam = SMALL
    msgs = drive()
    gray, depth = synth.make_frame(cam, 0)
    sc = Script()
    for stamp, is_kf, ref, p7, path, loops in msgs:
        sc.orb(stamp, is_kf, ref, p7, path, loops)
        sc.dump()
        sc.images(stamp, gray, depth)
        sc.dump()
    _, raw = run_node(str(tmp_path), cam, sc, drift_free_poses)
    dumps = iter(read_dumps(raw, [(True, False)] * (2 * len(msgs))))

    m = pyoracle_window.RefMapWindow(cam, drift_free_poses=drift_free_poses)
    seen = {"warps": 0, "propagated": 0, "retired_twice": False, "kf0_back": False}
    retired = {}
    for t, (stamp, is_kf, ref, p7, path, loops) in enumerate(msgs):
        m.set_local(probe_surfels())
        m.frame(stamp, None, None, p7, is_kf, ref, path7=np.array(path).reshape(-1, 7), loops=loops)
        for stage in ("orb", "images"):
            d = next(dumps)
            what = f"frame {t}, after the {stage} message"
            assert d["rc"] == 0, what
            assert len(d["cam"]) == m.num_poses(), what
            assert d["local"] == m.local_pose_indexs(), f"{what}: local_surfels_indexs"
            want = m.pending_frame()
            got = d["pending"]
            assert (got is None) == (want is None), f"{what}: pending frame"
            if want is not None:
                assert got[0] == want[0] and got[2:] == want[2:], f"{what}: pending reference / window lists"
                assert got[1].tobytes() == want[1].tobytes(), f"{what}: fuse pose differs {got[1]} {want[1]}"
            for root in range(m.num_poses()):
                assert d["lists"][root] == m.window_lists(root), f"{what}: window lists from root {root}"
                rem, add = d["lists"][root]
                df = d["driftfree"][root]
                assert [p for p in df if p not in d["local"]] == add and sorted(set(d["local"]) - set(df)) == rem
            if stage == "orb":
                local = m.local()
                moved = local[:PROBE_W].tobytes() != probe_surfels().tobytes()
                assert moved == bool(d["warp"]), f"{what}: loop closure"
                if moved:
                    seen["warps"] += 1
                    assert d["warp"][0][0] == -1
                    Wn = d["warp"][0][1].reshape(4, 4).T
                    assert Wn[:3].tobytes() == probe_warp(local)[:3].tobytes(), f"{what}: active warp matrix"
                    assert all(p not in d["local"] for p, _ in d["warp"][1:])
                    # every pose whose position moved took its loop pose
                    assert all(np.array_equal(c, l) for c, l in zip(d["cam"], d["loop"]))
                if len(path) < len(d["cam"]) - (1 if is_kf else 0) and len(path):
                    seen["propagated"] += 1
                for p in (want[2] if want else []):
                    retired[p] = retired.get(p, 0) + 1
                if want and 0 in want[3] and t > 0:
                    seen["kf0_back"] = True
                m.images(stamp, gray, depth)
        if any(n >= 2 for n in retired.values()):
            seen["retired_twice"] = True
    m.close()
    assert seen["warps"] >= 2 and seen["propagated"] >= 2
    if drift_free_poses == 2:
        assert seen["retired_twice"] and seen["kf0_back"]


def test_stalled_sync_drops_the_pose(tmp_path):
    """An image and a depth newer than the oldest pose: the reference spins forever (synchronize_msgs has no `>`
    branch); the node drops that pose without a fuse and fuses the next one."""
    cam = SMALL
    gray, depth = synth.make_frame(cam, 0)
    msgs = drive(4)
    sc = Script()
    sc.orb(*msgs[0])
    sc.images(msgs[0][0], gray, depth)
    sc.dump()
    sc.orb(*msgs[1])                                       # its images never come
    sc.dump()
    sc.images(msgs[2][0], gray, depth)                     # newer than the pending pose
    sc.dump()
    sc.orb(*msgs[2])
    sc.dump()
    _, raw = run_node(str(tmp_path), cam, sc, 2)
    d0, d1, d2, d3 = read_dumps(raw, [(True, False)] * 4)
    assert d0["pending"] is None and d1["pending"][0] == msgs[1][2]
    assert d2["pending"] is None and d2["fuse_pose"].tobytes() == d0["fuse_pose"].tobytes()  # dropped, nothing fused
    assert d3["pending"] is None and d3["fuse_pose"].tobytes() != d0["fuse_pose"].tobytes()  # frame 2 fused
    assert all(d["rc"] == 0 for d in (d0, d1, d2, d3))


def test_out_of_range_input_is_rejected(tmp_path):
    cam = SMALL
    msgs = drive(3)
    sc = Script()
    sc.orb(*msgs[0])
    sc.dump()
    stamp, is_kf, _, p7, path, _ = msgs[1]
    sc.orb(stamp, is_kf, 5, p7, path, [])                 # reference keyframe that does not exist
    sc.dump()
    sc.orb(stamp, is_kf, 0, p7, path, [0, -1])            # negative loop index
    sc.dump()
    _, raw = run_node(str(tmp_path), cam, sc, 2)
    d0, d1, d2 = read_dumps(raw, [(True, False)] * 3)
    assert d0["rc"] == 0 and d1["rc"] == -1 and d2["rc"] == -1
    assert len(d1["cam"]) == len(d2["cam"]) == 1


def test_pose_math_equals_the_oracle_stand_in():
    """node_math restates the Eigen stand-in of the reference build operation for operation: quaternion <-> matrix,
    products, adjugate inverse and the cast, bit for bit on random poses (tests/cpp/node_math_main.cpp)."""
    r = subprocess.run([build_adapter("node_math_main"), "2000"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "2000 poses" in r.stdout
