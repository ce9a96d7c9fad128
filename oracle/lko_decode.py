"""oracle/lko_decode.py — TEST INFRASTRUCTURE ONLY.

The PointCloud2 decode of the CPU restatement with the header stamp applied: lko.decode_pointcloud2 returns the first /
last point times without the stamp (as lk_decode_pointcloud2 does); this adds it the way lidar_processing.cc does, so the
result is lidar_begin_time_ / lidar_end_time_ of a message with that stamp. Pinned to the reference's own source by
tests/test_decode_oracle.py (oracle/lkref_decode.py, tests/golden/ref_decode.npz).
"""
import lko


def decode_pointcloud2(data, layout, blind, filter_num, time_scale, stamp=0.0):
    """lko.decode_pointcloud2 of a message with header stamp `stamp`. Returns (float4 points, intensity, begin, end):
    begin / end = stamp + the first / last point time for Velodyne and Ouster (:34-35, :62-63), the point time alone for
    Hesai (:90-91)."""
    pts, inten, first, last = lko.decode_pointcloud2(data, layout, blind, filter_num, time_scale)
    if layout.lidar_type != 3:
        first, last = stamp + first, stamp + last
    return pts, inten, first, last
