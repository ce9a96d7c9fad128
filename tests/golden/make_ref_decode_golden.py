"""Regenerates tests/golden/ref_decode.npz from the REFERENCE ITSELF: oracle/_ref/liblkref_decode.so is the reference's own
legkilo/src/preprocess/lidar_processing.cc compiled unmodified (oracle/ref_decode/Makefile), fed one PointCloud2 per
call. Run where the reference sources are; boxes without them read the committed fixture (tests/test_decode_oracle.py
on CPU, tests/test_gpu_decode_batch.py under -m gpu).

  <name>__data, __layout, __time_scale, __stamp   the message of tests/decode_cases.py and how it is decoded
  <name>__<c>__pts, __intensity, __times          the reference's output for decode_cases.COMBOS[c] (times = begin, end)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in ("leg-kilo_b200/python", "oracle", "tests"):
    sys.path.insert(0, os.path.join(ROOT, p))
import decode_cases  # noqa: E402
import lkref_decode  # noqa: E402


def main():
    arrays = {}
    for name, layout, data, ts, stamp in decode_cases.messages():
        arrays[f"{name}__data"] = data
        arrays[f"{name}__layout"] = decode_cases.layout_array(layout)
        arrays[f"{name}__time_scale"] = np.float64(ts)
        arrays[f"{name}__stamp"] = np.float64(stamp)
        for c, (blind, fn) in enumerate(decode_cases.COMBOS):
            pts, inten, b, e = lkref_decode.decode_pointcloud2(data, layout, blind, fn, ts, stamp)
            arrays[f"{name}__{c}__pts"] = pts
            arrays[f"{name}__{c}__intensity"] = inten
            arrays[f"{name}__{c}__times"] = np.array([b, e])
    np.savez_compressed(os.path.join(HERE, "ref_decode.npz"), **arrays)
    print("reference-made decode fixture written")


if __name__ == "__main__":
    main()
