"""Sweep accumulation on the GPU: what an accumulating frame costs, and what it finds on a sparse sensor.

  1. lmot_frame_dev frames/s on the bench scene (120 k points, the sensor driving at 5 m/s) at K = 1, 2, 4, 8, in alternating rounds
  2. one 8-sequence lmot_seq_dev tick, no sequence accumulating vs all eight at K = 4
  3. accumulate_kernel's device time (torch.profiler) at K = 2, 4, 8
  4. boxes, tracks and (frame, static object) pairs with a box centre within 1 m on the sparse 16-beam scene of the tests, K = 1 and 4
  5. the card's name and power limit, read in the same call
Prints one JSON object (and writes it to --out); every time is a median over rounds with its min / max.
"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
from accumulate_scenes import hits, sparse_frames  # noqa: E402

KS = (1, 2, 4, 8)


def spread(xs):
    return dict(median=statistics.median(xs), min=min(xs), max=max(xs), rounds=len(xs))


def frame_rounds(frames, rounds, steps):
    d = [torch.from_numpy(p).cuda() for _, p in frames]
    ctx = {}
    for K in KS:
        c = pkg.Lmot()
        c.set_accumulate(sweeps=K)
        ctx[K] = c
    res = {K: [] for K in KS}
    ts = 0.0
    for r in range(rounds + 1):
        for K, c in ctx.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(steps):
                ts += 1e5
                x = d[i % len(d)]
                c.frame_dev(x.data_ptr(), x.shape[0], ts, 5.0, 0.0)
            c.frame_fetch()
            dt = time.perf_counter() - t0
            if r > 0:                        # round 0 warms up (and allocates the rings)
                res[K].append(steps / dt)
    for c in ctx.values():
        c.close()
    return {f"K{K}": spread(v) for K, v in res.items()}


def seq_rounds(frames, rounds, steps):
    """one 8-sequence lmot_seq_dev tick of the bench frames, no sequence accumulating vs all eight at K = 4 (ticks/s)"""
    d = [torch.from_numpy(p).cuda() for _, p in frames]
    ctx = {}
    for arm in ("none", "all"):
        c = pkg.Lmot()
        c.seq_open(8)
        if arm == "all":
            for k in range(8):
                c.seq_set_accumulate(k, sweeps=4)
        ctx[arm] = c
    res = {arm: [] for arm in ctx}
    ts = 0.0
    for r in range(rounds + 1):
        for arm, c in ctx.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(steps):
                ts += 1e5
                c.seq_dev([(x.data_ptr(), x.shape[0]) for x in d], [ts] * 8, [5.0] * 8, [0.0] * 8)
            c.seq_fetch()
            dt = time.perf_counter() - t0
            if r > 0:
                res[arm].append(steps / dt)
    for c in ctx.values():
        c.close()
    return {arm: spread(v) for arm, v in res.items()}


def kernel_times(frames, steps):
    from torch.profiler import ProfilerActivity, profile
    d = [torch.from_numpy(p).cuda() for _, p in frames]
    out = {}
    for K in KS[1:]:
        c = pkg.Lmot()
        c.set_accumulate(sweeps=K)
        ts = 0.0
        for i in range(2 * K):
            ts += 1e5
            c.frame_dev(d[i % len(d)].data_ptr(), d[i % len(d)].shape[0], ts, 5.0, 0.0)
        c.frame_fetch()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(steps):
                ts += 1e5
                c.frame_dev(d[i % len(d)].data_ptr(), d[i % len(d)].shape[0], ts, 5.0, 0.0)
            c.frame_fetch()
            torch.cuda.synchronize()
        us = [e.device_time for e in prof.events() if "accumulate_kernel" in e.name]
        out[f"K{K}"] = spread(us) if us else None
        c.close()
    return out


def sparse(n_frames):
    out = {}
    for K in (1, 4):
        boxes = tracks = pairs = 0
        for kind in ("straight", "turn"):
            c = pkg.Lmot()
            c.set_accumulate(sweeps=K)
            for ts, v, yaw, pts, _, objs in sparse_frames(pkg, synth, kind, n_frames):
                r = c.frame(pts, ts, v, yaw)
                boxes += len(r["boxes"])
                pairs += hits(r["boxes"], objs)
            tracks += c.tracker_num_tracks()
            c.close()
        out[f"K{K}"] = dict(boxes=boxes, tracks_in_table=tracks, static_pairs_within_1m=pairs)
    return out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode == 0 and q.stdout.strip():
        name, power = (x.strip() for x in q.stdout.strip().splitlines()[0].split(",", 1))
        return dict(name=name, power_limit=power)
    return dict(name=torch.cuda.get_device_name(0), power_limit="unknown (nvidia-smi did not answer)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    frames = list(synth.frames(synth.SceneConfig(seed=1), 8))         # the bench scene: 64 x 1875 = 120 k points
    out = dict(card=card(), frame_dev_fps=frame_rounds(frames, a.rounds, a.steps),
               seq_dev_8x120k_ticks_per_s=seq_rounds(frames, a.rounds, a.steps // 4), accumulate_kernel_us=kernel_times(frames, 50),
               sparse_16_beam=sparse(16))
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
