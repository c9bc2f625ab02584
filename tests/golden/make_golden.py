"""Mints the committed golden vectors from the SERIALISED REFERENCE (oracle/_ref/libdsm_ref_serial.so,
i.e. the reference's own fusion_functions.cpp compiled where its sources are, see oracle/Makefile).
Run where oracle/_ref/ holds the reference builds:  python tests/golden/make_golden.py

vga_two_pass.npz : BASELINE config 1 — one synthetic 640x480 frame, identity pose, empty pool
                   (pure initialise), then the same frame again against the surfels it produced
                   (pure fuse).  Full labels (u16), seeds (60-byte records), surfels (44-byte records).
checksums.json   : CRC32 of labels / seeds / surfels for larger frames (KITTI 1226x370 stream of 3,
                   flat KITTI, HD 1280x720) so that the oracle can be re-pinned anywhere cheaply.
reference_checksums.json : CRC32s of what the serialised reference ("serial": the scenarios of
                   tests/test_oracle.py, both constant sets) and the reference's SurfelMap ("map": the
                   pinned members of tests/test_refmap.py) compute, so those tests run without them.
"""
import json
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import pyoracle  # noqa: E402
from densesurfelmapping_b200 import synth  # noqa: E402
from densesurfelmapping_b200.elements import SURFEL_DTYPE  # noqa: E402


def canon(a):
    """field-by-field bytes (struct padding excluded) with every NaN canonicalised: NaN payload/sign
    and padding bytes are not part of the contract."""
    parts = []
    for f in a.dtype.names:
        v = np.ascontiguousarray(a[f]).copy()
        if v.dtype.kind == "f":
            v[np.isnan(v)] = np.float32(np.nan)
        parts.append(v.tobytes())
    return b"".join(parts)


def crc(x):
    return zlib.crc32(x if isinstance(x, (bytes, bytearray)) else np.ascontiguousarray(x).tobytes()) & 0xFFFFFFFF


def stream_checksums(cam, n, flat):
    rs = pyoracle.RefSerial(cam)
    pool = np.zeros(0, SURFEL_DTYPE)
    out = []
    for t in range(n):
        pose = synth.pose_stream(t)
        g, d = synth.make_frame(cam, t, pose, flat=flat)
        loc, new = rs.fuse(t // 2, g, d, pose, pool)
        out.append(dict(frame=t, gray_crc=crc(g), depth_crc=crc(d), labels_crc=crc(rs.labels()),
                        seeds_crc=crc(canon(rs.seeds())), local_crc=crc(canon(loc)), new_crc=crc(canon(new)),
                        n_local=int(len(loc)), n_new=int(len(new)), n_fused=int((loc["update_times"] > 1).sum()) if len(loc) else 0,
                        n_killed=int((loc["update_times"] == 0).sum()) if len(loc) else 0))
        keep = loc[loc["update_times"] > 0] if len(loc) else loc
        pool = np.concatenate([keep, new])
    return out


def main():
    assert pyoracle.have_reference(), "needs oracle/_ref/libdsm_ref_serial.so (make -C oracle)"
    cam = synth.VGA
    g, d = synth.make_frame(cam, 0)
    pose = synth.identity_pose()
    rs = pyoracle.RefSerial(cam)
    _, new0 = rs.fuse(0, g, d, pose, np.zeros(0, SURFEL_DTYPE))
    labels0, seeds0 = rs.labels(), rs.seeds()
    loc1, new1 = rs.fuse(1, g, d, pose, new0)
    labels1, seeds1 = rs.labels(), rs.seeds()
    np.savez_compressed(os.path.join(HERE, "vga_two_pass.npz"), gray_crc=crc(g), depth_crc=crc(d),
                        labels0=labels0.astype(np.uint16), seeds0=seeds0.view(np.uint8), new0=new0.view(np.uint8),
                        labels1=labels1.astype(np.uint16), seeds1=seeds1.view(np.uint8), local1=loc1.view(np.uint8), new1=new1.view(np.uint8))
    sums = {"kitti": stream_checksums(synth.KITTI, 3, False), "kitti_flat": stream_checksums(synth.KITTI, 2, True),
            "hd": stream_checksums(synth.HD, 2, False), "vga_flat": stream_checksums(synth.VGA, 2, True)}
    json.dump(sums, open(os.path.join(HERE, "checksums.json"), "w"), indent=1)
    reference_checksums()
    print("golden written:", os.listdir(HERE))


def reference_checksums():
    import test_oracle
    import test_refmap
    serial = {}
    for key, (c, rgbd, run) in test_oracle.scenarios().items():
        ref = test_oracle.reference_serial(c, rgbd)
        assert ref is not None, "needs oracle/_ref/libdsm_ref_serial{,_rgbd}.so"
        serial[key] = [test_oracle.digest(r) for r in run(ref)]
    assert pyoracle.have_refmap(), "needs oracle/_ref/libdsm_refmap.so"
    m = pyoracle.RefMap(test_refmap.CAM)
    json.dump({"serial": serial, "map": test_refmap.map_pins(m)}, open(os.path.join(HERE, "reference_checksums.json"), "w"), indent=1)
    m.close()


if __name__ == "__main__":
    main()
