"""Sequence ticks with sensor tables: frames/s and ticks/s of 8 x 120 k-point frames per tick (frames resident on the device), four
arms alternated round by round:
  A  one context, lmot_seq_dev: 2 vehicles x 4 sensors (each vehicle its own sensor table and track table)
  B  two contexts, one per vehicle, each lmot_batch_dev with its rig (lmot_set_sensors) on its own stream
  C  one context, lmot_seq_dev: 8 one-sensor sequences, each with its own mounting height and pose
  D  the same 8 sequences without tables (lmot_params' thresholds; the kernels without the rig code)
Host clock around the timed ticks, bracketed by device synchronisations.  After each round the final track tables of A and B are
compared (they must be equal; C and D run different thresholds on different clouds and are not comparable).  Prints the card name and
power limit beside the numbers.  Needs a CUDA device; there is no CPU path.

    python scripts/seq_rig_measure.py [--ticks 30] [--rounds 3] [--warm 4]
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
    raise SystemExit("seq_rig_measure.py: no CUDA device")
card = torch.cuda.get_device_name(0)
try:
    pl = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                        capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as ex:                  # the numbers below still stand, without the power limit
    pl = f"unavailable ({type(ex).__name__})"

F = 8
n_t = a.warm + a.ticks
heights = [2.0, 1.2, 0.8, 1.8, 1.6, 1.0, 2.2, 1.4]


def yaw_pose(yaw, tx, ty, tz):
    c, s = np.cos(yaw), np.sin(yaw)
    return np.array([[c, -s, 0, tx], [s, c, 0, ty], [0, 0, 1, tz]], np.float32)


def table(idx):
    return dict(poses=[yaw_pose(k * np.pi / 4, 1.5 * np.cos(k), 0.8 * np.sin(k), heights[k]) for k in idx],
                h_sensor=[heights[k] for k in idx], t_hmin=[-2.0 + 2.0 - heights[k] for k in idx],
                t_hmax=[-0.4 + 2.0 - heights[k] for k in idx], sensor_height=[heights[k] for k in idx])


raw = [np.stack([p for _, p in synth.frames(synth.SceneConfig(seed=301 + 11 * s), n_t)]) for s in range(F)]
n = raw[0].shape[1]
shifted = []
for s in range(F):                       # sensor s's clouds as seen from its mounting height
    q = raw[s].copy()
    q[..., 2] += np.float32(2.0 - heights[s])
    shifted.append(q)
dev_raw = [torch.from_numpy(x).cuda() for x in raw]
dev_rig = [torch.from_numpy(x).cuda() for x in shifted]
del raw, shifted
torch.cuda.synchronize()
VEH = [list(range(0, 4)), list(range(4, 8))]
ts = lambda k, t: 1.0e6 * (k + 1) + 1.0e5 * t                    # own start stamp per sequence / vehicle
ego = lambda k, t: (2.0 + k, 0.01 * (k - 3) * t)                 # own ego speed and yaw per sequence / vehicle


def seq_scalars(S, t):
    return (lmot.Lmot.seq_scalars(S, [ts(k, t) for k in range(S)]), lmot.Lmot.seq_scalars(S, [ego(k, t)[0] for k in range(S)]),
            lmot.Lmot.seq_scalars(S, [ego(k, t)[1] for k in range(S)]))


def open_a(ctx):
    ctx.seq_open(2, ring=8)
    for v, idx in enumerate(VEH):
        ctx.seq_set_sensors(v, **table(idx))


def open_c(ctx):
    ctx.seq_open(F, ring=8)
    for k in range(F):
        ctx.seq_set_sensors(k, **table([k]))


def open_d(ctx):
    ctx.seq_open(F, ring=8)


# A: one context, two vehicles of four sensors
ca = lmot.Lmot(); sa = torch.cuda.Stream(); ca.set_stream(sa.cuda_stream); open_a(ca)
args_a = [ca.seq_prepare([[(dev_rig[s][t].data_ptr(), n) for s in idx] for idx in VEH]) for t in range(n_t)]
scal_2 = [seq_scalars(2, t) for t in range(n_t)]
# B: one context per vehicle, its own stream
cb = []
for v, idx in enumerate(VEH):
    c = lmot.Lmot(); st = torch.cuda.Stream(); c.set_stream(st.cuda_stream)
    t_ = table(idx)
    c.set_sensors(t_.pop("poses"), **t_)
    cb.append((c, [c.batch_prepare([(dev_rig[s][t].data_ptr(), n) for s in idx]) for t in range(n_t)]))
# C / D: eight one-sensor sequences with and without tables
cc = lmot.Lmot(); sc = torch.cuda.Stream(); cc.set_stream(sc.cuda_stream); open_c(cc)
args_c = [cc.seq_prepare([(dev_rig[s][t].data_ptr(), n) for s in range(F)]) for t in range(n_t)]
cd = lmot.Lmot(); sd = torch.cuda.Stream(); cd.set_stream(sd.cuda_stream); open_d(cd)
args_d = [cd.seq_prepare([(dev_raw[s][t].data_ptr(), n) for s in range(F)]) for t in range(n_t)]
scal_8 = [seq_scalars(F, t) for t in range(n_t)]


def run_a(t0, t1):
    for t in range(t0, t1):
        ca.seq_dev(args_a[t], *scal_2[t])


def run_b(t0, t1):
    for t in range(t0, t1):
        for v, (c, args) in enumerate(cb):
            c.batch_dev(args[t], ts(v, t), *ego(v, t))


def run_c(t0, t1):
    for t in range(t0, t1):
        cc.seq_dev(args_c[t], *scal_8[t])


def run_d(t0, t1):
    for t in range(t0, t1):
        cd.seq_dev(args_d[t], *scal_8[t])


arms = {"A seq 2x4": (lambda: open_a(ca), run_a), "B 2 contexts": (lambda: [c.tracker_reset() for c, _ in cb], run_b),
        "C seq 8x1 rig": (lambda: open_c(cc), run_c), "D seq 8x1 none": (lambda: open_d(cd), run_d)}
rates = {k: [] for k in arms}
print(f"card: {card}; power limit, max SM clock: {pl}")
print(f"{F} x {n} points per tick, {a.ticks} timed ticks after {a.warm} warm-up ticks, {a.rounds} rounds alternating the arms")
for rnd in range(a.rounds):
    for name, (reset, run) in arms.items():
        reset()
        run(0, a.warm)
        torch.cuda.synchronize()
        h0 = time.perf_counter()
        run(a.warm, n_t)
        torch.cuda.synchronize()
        rates[name].append(a.ticks / (time.perf_counter() - h0))
    for v, (c, _) in enumerate(cb):
        da, db = ca.seq_tracker_dump(v), c.tracker_dump()
        if da.shape != db.shape or not np.array_equal(da.view(np.uint64), db.view(np.uint64)):
            raise SystemExit(f"round {rnd}: vehicle {v} of A differs from its context in B ({da.shape} vs {db.shape} rows)")
print(f"A and B: final tables equal in every round ({[len(ca.seq_tracker_dump(v)) for v in range(2)]} tracks); "
      f"A's last tick: boxes per vehicle {[len(x['boxes']) for x in ca.seq_fetch()]}")
for name, v in rates.items():
    v = np.array(v)
    print(f"{name:15s} frames/s median {F * np.median(v):8.1f}  min {F * v.min():8.1f}  max {F * v.max():8.1f}   "
          f"ticks/s median {np.median(v):7.1f}  min {v.min():7.1f}  max {v.max():7.1f}")
for c in [ca, cc, cd] + [c for c, _ in cb]:
    c.set_stream(None)
    c.close()
