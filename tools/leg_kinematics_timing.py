"""Times one lk_leg_kinematics call at two sizes: n = 50 (one scan's queue of leg states at 500 Hz) and n = 600 000
(a 20-minute recording). Device time from CUDA events on the library's stream (lk_timer_start / lk_timer_stop around
`--reps` calls, so it includes the host gaps between calls) and host wall-clock per call, both after warm-up. Prints
the card's name and power limit from the same run, then one JSON line per size.

    python tools/leg_kinematics_timing.py [--reps R]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "leg-kilo_b200", "python"))
from legkilo_b200 import Engine, abi, synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = (x.strip() for x in q.split(","))
    return name, limit


def time_calls(eng, states, cfg, reps, warmup=5):
    for _ in range(warmup):
        eng.leg_kinematics(states, cfg)
    walls = []
    eng.timer_start()
    for _ in range(reps):
        t = time.perf_counter()
        kin, _ = eng.leg_kinematics(states, cfg)
        walls.append(time.perf_counter() - t)
    dev = eng.timer_stop()
    walls.sort()
    return dict(n=len(states), n_out=len(kin), reps=reps, device_ms_per_call=dev["total_ms"] / reps,
                host_ms_per_call_mean=1e3 * sum(walls) / reps, host_ms_per_call_p50=1e3 * walls[reps // 2])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200, help="calls timed at n = 50 (a tenth of them at n = 600 000)")
    args = ap.parse_args()
    name, limit = card()
    print(f"card: {name}, power limit {limit}")
    cfg = abi.CONFIGS["leg_fusion"]
    eng = Engine(cfg)
    one_scan = synth.leg_state_stream(0.0, 0.1, 500.0, "leg_fusion", 80)
    recording = synth.leg_state_stream(0.0, 1200.0, 500.0, "leg_fusion", 81)
    assert len(one_scan) == 50 and len(recording) == 600_000
    for states, reps in ((one_scan, args.reps), (recording, max(args.reps // 10, 3))):
        r = time_calls(eng, states, cfg, reps)
        r.update(card=name, power_limit=limit)
        print(json.dumps(r))
    eng.close()


if __name__ == "__main__":
    main()
