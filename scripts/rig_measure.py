"""Batched ticks of a sensor rig: ticks/s of 8 x 120 k-point frames through lmot_batch_dev in three configurations, alternated round
by round on one context each (CUDA events on the launching stream, frames resident on the device):
  none      no sensors (lmot_params for every frame; the kernels without the rig code)
  identity  8 sensors equal to lmot_default_sensor (the rig kernels, identity poses)
  distinct  8 different poses and mounting heights
Prints the card name and power limit beside the numbers.  Needs a CUDA device; there is no CPU path.

    python scripts/rig_measure.py [--ticks 20] [--rounds 5]
"""
import argparse
import importlib
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
lmot = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")

ap = argparse.ArgumentParser()
ap.add_argument("--ticks", type=int, default=20)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--warm", type=int, default=3)
a = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("rig_measure.py: no CUDA device")
F = 8
card = torch.cuda.get_device_name(0)
try:
    pl = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                        capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as ex:                  # the numbers below still stand, without the power limit
    pl = f"unavailable ({type(ex).__name__})"

n_t = a.warm + a.ticks
streams = [[p for _, p in synth.frames(synth.SceneConfig(seed=101 + s), n_t)] for s in range(F)]
n = len(streams[0][0])
dev = [torch.from_numpy(np.stack(s)).cuda() for s in streams]
stream = torch.cuda.Stream()


def yaw_pose(yaw, tx, ty, tz):
    c, s = np.cos(yaw), np.sin(yaw)
    return np.array([[c, -s, 0, tx], [s, c, 0, ty], [0, 0, 1, tz]], np.float32)


heights = [2.0, 1.2, 0.8, 1.8, 1.6, 1.0, 2.2, 1.4]
configs = {"none": None, "identity": dict(poses=[np.eye(3, 4, dtype=np.float32)] * F),
           "distinct": dict(poses=[yaw_pose(k * np.pi / 4, 1.5 * np.cos(k), 0.8 * np.sin(k), h) for k, h in enumerate(heights)],
                            h_sensor=heights, t_hmin=[-2.0 + 2.0 - h for h in heights], t_hmax=[-0.4 + 2.0 - h for h in heights],
                            sensor_height=heights)}
ctxs = {}
for name, cfg in configs.items():
    ctx = lmot.Lmot()
    ctx.set_stream(stream.cuda_stream)
    if cfg is not None:
        ctx.set_sensors(cfg["poses"], **{k: v for k, v in cfg.items() if k != "poses"})
    ctxs[name] = (ctx, [ctx.batch_prepare([(dev[s][t].data_ptr(), n) for s in range(F)]) for t in range(n_t)])

e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
rates = {k: [] for k in configs}
for rnd in range(a.rounds):
    for name, (ctx, args) in ctxs.items():
        ctx.tracker_reset()
        for t in range(a.warm):
            ctx.batch_dev(args[t], 1e5 * (t + 1))
        ctx.flush(); torch.cuda.synchronize()
        e0.record(stream)
        for t in range(a.warm, n_t):
            ctx.batch_dev(args[t], 1e5 * (t + 1))
        ctx.flush()
        e1.record(stream)
        torch.cuda.synchronize()
        rates[name].append(1e3 * a.ticks / e0.elapsed_time(e1))
        r = ctx.batch_fetch(want_boxes=False)
        if rnd == 0:
            print(f"{name:9s} boxes per frame {r['n_boxes']}, tracks {len(r['track_manage'])}")
print(f"card: {card}; power limit, max SM clock: {pl}")
print(f"{F} x {n} points per tick, {a.ticks} timed ticks per round, {a.rounds} rounds alternating the configurations")
for name, v in rates.items():
    v = np.array(v)
    print(f"{name:9s} ticks/s median {np.median(v):8.1f}  min {v.min():8.1f}  max {v.max():8.1f}")
for ctx, _ in ctxs.values():
    ctx.set_stream(None)
    ctx.close()
