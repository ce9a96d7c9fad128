"""Writes tests/golden/ref_map_insert.npz from the reference itself (oracle/_ref/liblkref_insert.so: oracle/ref_insert/):
the UpdateVoxelMap of point sets placed at explicit poses (lk_map_insert), on the cases of tests/map_insert_cases.py. Per
case <name>: the call's buffers (<name>_pts, _set_offsets, _rot, _pos, _rot_cov, _pos_cov), for a case on top of a map
the first-frame cloud (<name>_pw, _pb) and the digest of the map BuildVoxelMap made from it (<name>_map0), and the digest
of the map after the insert (<name>_map1). Writes only this new file; the output is the same bytes on every run."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in ("leg-kilo_b200/python", "oracle", "tests"):
    sys.path.insert(0, os.path.join(ROOT, p))
import general_prior as gp  # noqa: E402
import lkref_insert  # noqa: E402
import map_insert_cases as mic  # noqa: E402
import mapcmp  # noqa: E402


def main():
    out = {}
    for name in mic.NAMES:
        cfg, c = mic.case(name)
        r = lkref_insert.Reference(cfg)
        if "pw" in c:
            r.build_voxel_map(c["pw"], c["pb"], R=mic.G, rot_cov=gp.map_covs(mic.G)[0], pos_cov=gp.map_covs(mic.G)[1])
            out[f"{name}_map0"] = mapcmp.digest(r.map_export())
        r.map_insert(*mic.call(c))
        out[f"{name}_map1"] = mapcmp.digest(r.map_export())
        for k, v in c.items():
            out[f"{name}_{k}"] = v
        print(name, "points", len(c["pts"]), "nodes", len(out[f"{name}_map1"]))
    np.savez_compressed(os.path.join(HERE, "ref_map_insert.npz"), **out)


if __name__ == "__main__":
    main()
