"""Per-sequence detection parameters: ticks/s of eight 120 k-point HDL-64 sequences through lmot_seq_dev (frames resident on the device),
three arms alternated round by round:
  (a) default    no sequence has its own values: today's kernels
  (b) same       every sequence given lmot_params' own values: the per-frame kernel variants, the same outputs
  (c) distinct   eight different sets (range window, ROI, L-shape and rule values)
Host clock around the timed ticks, bracketed by device synchronisations.  After each round the final track tables of (a) and (b) are
compared (they must be equal).  Prints the card name and power limit beside the numbers.  Needs a CUDA device; there is no CPU path.

    python scripts/seq_detect_params_measure.py [--ticks 30] [--rounds 3] [--warm 4]
"""
import argparse
import importlib
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
lmot = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")

ap = argparse.ArgumentParser()
ap.add_argument("--ticks", type=int, default=30)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--warm", type=int, default=4)
a = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("seq_detect_params_measure.py: no CUDA device")
card = torch.cuda.get_device_name(0)
try:
    pl = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                        capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as ex:                  # the numbers below still stand, without the power limit
    pl = f"unavailable ({type(ex).__name__})"

S = 8
SETS = [dict(), dict(t_hmin=-1.9, t_hmax=-1.0, h_sensor=1.73, roi_m=30.0, l_slope_dist=3, l_num_points=300, sensor_height=1.73),
        dict(r_min=2.0, r_max=50.0, roi_m=40.0, t_pt_per_m3=2.0, ram_points=200), dict(r_max=80.0, roi_m=44.0, t_len_max=12.0),
        dict(rule_filter=1), dict(r_min=10.0, r_max=60.0), dict(min_cluster_points=12, ground_tolerance=0.3), dict(roi_m=60.0)]
n_t = a.warm + a.ticks
streams = [[p for _, p in synth.frames(synth.SceneConfig(seed=211 + 13 * k), n_t)] for k in range(S)]
n = len(streams[0][0])
dev = [torch.from_numpy(np.stack(s)).cuda() for s in streams]
ts = lambda k, t: 1.0e6 * (k + 1) + 1.0e5 * t
ego = lambda k, t: (2.0 + k, 0.01 * (k - 3) * t)
torch.cuda.synchronize()

ctx = lmot.Lmot()
stream = torch.cuda.Stream()
ctx.set_stream(stream.cuda_stream)
own = lmot.default_detect_params(ctx.params)


def arm_setup(arm):
    ctx.seq_open(S, ring=8)
    for k in range(S):
        if arm == "same":
            ctx.seq_set_detect_params(k, **own)
        elif arm == "distinct":
            ctx.seq_set_detect_params(k, **{**own, **SETS[k]})


def run(args, t0, t1):
    for t in range(t0, t1):
        ctx.seq_dev(args[t], [ts(k, t) for k in range(S)], [ego(k, t)[0] for k in range(S)], [ego(k, t)[1] for k in range(S)])


print(f"card: {card}; power limit, max SM clock: {pl}")
print(f"S={S} sequences, {n} points per frame, {a.ticks} timed ticks after {a.warm} warm-up ticks, {a.rounds} rounds alternating the arms")
ctx.seq_open(S, ring=8)
args = [ctx.seq_prepare([(dev[k][t].data_ptr(), n) for k in range(S)]) for t in range(n_t)]
rates = {"default": [], "same": [], "distinct": []}
for rnd in range(a.rounds):
    tables = {}
    for arm in rates:
        arm_setup(arm)
        run(args, 0, a.warm)
        torch.cuda.synchronize()
        h0 = time.perf_counter()
        run(args, a.warm, n_t)
        torch.cuda.synchronize()
        rates[arm].append(a.ticks / (time.perf_counter() - h0))
        tables[arm] = [ctx.seq_tracker_dump(k) for k in range(S)]
    for k in range(S):
        da, db = tables["default"][k], tables["same"][k]
        if da.shape != db.shape or not np.array_equal(da.view(np.uint64), db.view(np.uint64)):
            raise SystemExit(f"round {rnd}: sequence {k}: (a) and (b) end with different tables")
print(f"(a) and (b) end with equal tables in every round ({[len(t) for t in tables['default']]} tracks)")
for arm, v in rates.items():
    v = np.array(v)
    print(f"{arm:9s} ticks/s median {np.median(v):8.1f}  (min {v.min():8.1f}, max {v.max():8.1f})")
ctx.set_stream(None)
ctx.close()
