"""Regenerates tests/golden/ref_leg_kinematics.npz from the REFERENCE ITSELF: oracle/_ref/liblkref_leg.so is the
reference's own legkilo/src/preprocess/kinematics.cc compiled unmodified (oracle/ref_leg/Makefile), driven from its
initial state with the redundancy drop of RosInterface::kinematicImuCallBack. Run where the reference sources are;
boxes without them read the committed fixture (tests/test_leg_kinematics.py: oracle on CPU, CUDA path under -m gpu).

  <cfg>_states  seeded leg-state stream (synth.leg_state_stream, 1 s at 500 Hz), raw lk_leg_state bytes
  <cfg>_kin     the reference's kinematic-inertial samples, raw lk_kinimu_meas bytes
  <cfg>_track   the lk_leg_track after the stream, raw bytes
for cfg in leg_fusion, diter (redundancy on, as every shipped config sets it).
"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in ("leg-kilo_b200/python", "oracle"):
    sys.path.insert(0, os.path.join(ROOT, p))
import lkref_leg  # noqa: E402
from legkilo_b200 import abi, synth  # noqa: E402

CASES = {"leg_fusion": 9300, "diter": 9301}


def main():
    arrays = {}
    for name, stream in CASES.items():
        states = synth.leg_state_stream(30.0, 31.0, 500.0, name, stream)
        kin, tr = lkref_leg.leg_kinematics(states, abi.CONFIGS[name], redundancy=True)
        arrays[f"{name}_states"] = states.view(np.uint8)
        arrays[f"{name}_kin"] = kin.view(np.uint8)
        arrays[f"{name}_track"] = np.frombuffer(C.string_at(C.addressof(tr), C.sizeof(tr)), np.uint8)
    np.savez_compressed(os.path.join(HERE, "ref_leg_kinematics.npz"), **arrays)
    print("reference-made leg-kinematics fixture written")


if __name__ == "__main__":
    main()
