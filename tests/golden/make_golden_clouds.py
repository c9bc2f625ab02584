"""Mints tests/golden/raw_cloud_checksums.json: the CRC32 of what the reference's own publish_raw_pointcloud
(surfel_map.cpp:1115-1151, compiled in place: oracle/_ref/libdsm_refmap_clouds.so, see oracle/clouds.mk) publishes for
the cases of tests/test_node_clouds.py::raw_cases, so that the numpy restatement is pinned on a checkout without it.
Run where oracle/_ref/ holds that build:  python tests/golden/make_golden_clouds.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import pyoracle_clouds  # noqa: E402
import test_node_clouds  # noqa: E402
from test_oracle import crc  # noqa: E402


def main():
    assert pyoracle_clouds.have_refmap_clouds(), "needs oracle/_ref/libdsm_refmap_clouds.so (make -C oracle -f clouds.mk clouds)"
    sums = {}
    for name, (cam, gray, depth, p7) in test_node_clouds.raw_cases().items():
        m = pyoracle_clouds.RefMapClouds(cam)
        sums[name] = crc(test_node_clouds.canon_points(m.publish_raw(gray, depth, p7)))
        m.close()
    json.dump(sums, open(os.path.join(HERE, "raw_cloud_checksums.json"), "w"), indent=1)
    print("golden written:", sums)


if __name__ == "__main__":
    main()
