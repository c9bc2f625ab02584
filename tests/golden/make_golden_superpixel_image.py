"""Mints tests/golden/superpixel_image_checksums.json: the CRC32 of the image the reference's own debug_show
(fusion_functions.cpp:977-1006, compiled in place: oracle/_ref/libdsm_ref_show.so, see oracle/show.mk) draws for the
cases of tests/test_superpixel_image.py::image_cases, so that the numpy restatement is pinned on a checkout without it.
Run where oracle/_ref/ holds that build:  python tests/golden/make_golden_superpixel_image.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import pyoracle_show  # noqa: E402
import test_superpixel_image  # noqa: E402
from test_oracle import crc  # noqa: E402


def main():
    assert pyoracle_show.have_ref_show(), "needs oracle/_ref/libdsm_ref_show.so (make -C oracle -f show.mk show)"
    sums = {}
    for name, (cam, gray, depth) in test_superpixel_image.image_cases().items():
        m = pyoracle_show.RefShow(cam)
        m.superpixels(gray, depth)
        sums[name] = crc(m.debug_show().tobytes())
        m.close()
    json.dump(sums, open(os.path.join(HERE, "superpixel_image_checksums.json"), "w"), indent=1)
    print("golden written:", sums)


if __name__ == "__main__":
    main()
