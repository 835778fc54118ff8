"""Knob sweep on the bench workload: tokens/s of the device-resident greedy decode for a list of
(option=value,...) settings.  usage: python sweep.py 7b 64 "tile_bytes=20480,stages=8" "tile_bytes=40960" ..."""
import importlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
workload, steps = sys.argv[1], int(sys.argv[2])
L, E = bench.SHAPES[workload]
ab = bench.algorithmic_bytes_per_token(L, E)
DEFAULTS = {"window": 2, "bwindow": 1, "pf_dist": 4, "poll_first": 2, "issue_gap": 0, "grid": 132}
eng = pkg.Engine(bench.model_path(workload, pkg))
stages0 = None
for spec in sys.argv[3:]:
    try:
        for k, v in DEFAULTS.items():  # every spec starts from the defaults
            eng.set_option(k, v)
        for kv in spec.split(","):
            if kv:
                k, v = kv.split("=")
                eng.set_option(k, v)
        eng.state_zero()
        eng.decode_timed([bench.SEED_TOKEN] * 8, teacher_forced=False)
        eng.state_zero()
        ms = eng.decode_timed([bench.SEED_TOKEN] * steps, teacher_forced=False)
        tps = steps / (ms / 1e3)
        print("%-60s %8.1f tok/s  %7.3f ms/tok  %6.0f GB/s" % (spec, tps, ms / steps, ab * tps / 1e9), flush=True)
    except Exception as ex:  # noqa: BLE001
        print("%-60s FAILED: %s" % (spec, ex), flush=True)
