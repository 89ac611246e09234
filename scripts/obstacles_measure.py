"""Obstacle footprints on the GPU: what they cost.

  1. lmot_frame_dev frames/s on the bench scene (120 k points) with obstacles off and on, in alternating rounds
  2. 8 x 120 k sequence ticks (lmot_seq_dev) per second with obstacles off and on for every sequence, in alternating rounds
  3. device time (torch.profiler) of obstacles_kernel per launch: one unit (lmot_frame_dev) and eight units (one tick)
  4. the card's name and power limit, read in the same call
Prints one JSON object (and writes it to --out); every rate and time is a median over rounds with its min / max.
"""
import argparse
import importlib
import json
import os
import re
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")

ARMS = ("off", "on")


def spread(xs):
    return dict(median=statistics.median(xs), min=min(xs), max=max(xs), rounds=len(xs))


def _ctx(arm, n_seq=0):
    c = pkg.Lmot()
    if n_seq:
        c.seq_open(n_seq)
    if arm == "on":
        c.set_obstacles(on=1)
        for k in range(n_seq):
            c.seq_set_obstacles(k, on=1)
    return c


def frame_rounds(d, rounds, steps):
    ctx = {arm: _ctx(arm) for arm in ARMS}
    res = {arm: [] for arm in ARMS}
    ts = 0.0
    for r in range(rounds + 1):
        for arm, c in ctx.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(steps):
                ts += 1e5
                x = d[i % len(d)]
                c.frame_dev(x.data_ptr(), x.shape[0], ts)
            c.frame_fetch()
            dt = time.perf_counter() - t0
            if r > 0:                        # round 0 warms up
                res[arm].append(steps / dt)
    for c in ctx.values():
        c.close()
    return {arm: spread(v) for arm, v in res.items()}


def tick_rounds(d, rounds, steps):
    ctx = {arm: _ctx(arm, 8) for arm in ARMS}
    res = {arm: [] for arm in ARMS}
    ts = 0.0
    frames = [(x.data_ptr(), x.shape[0]) for x in d[:8]]
    for r in range(rounds + 1):
        for arm, c in ctx.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(steps):
                ts += 1e5
                c.seq_dev(frames, [ts] * 8)
            c.seq_fetch()
            dt = time.perf_counter() - t0
            if r > 0:
                res[arm].append(steps / dt)
    for c in ctx.values():
        c.close()
    return {arm: spread(v) for arm, v in res.items()}


def kernel_times(d, steps):
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for units in (1, 8):
        c = _ctx("on", 8 if units == 8 else 0)
        ts = [0.0]

        def run():
            for i in range(steps):
                ts[0] += 1e5
                if units == 1:
                    c.frame_dev(d[i % len(d)].data_ptr(), d[i % len(d)].shape[0], ts[0])
                else:
                    c.seq_dev([(x.data_ptr(), x.shape[0]) for x in d[:8]], [ts[0]] * 8)
            c.frame_fetch() if units == 1 else c.seq_fetch()
        run()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run()
            torch.cuda.synchronize()
        ev = [e.device_time for e in prof.events() if e.device_type.name == "CUDA" and re.search(r"\bobstacles_kernel\b", e.name)]
        out[f"obstacles_kernel_{units}_unit{'s' if units > 1 else ''}_us"] = spread(ev)
        c.close()
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
    bench = [torch.from_numpy(p).cuda() for _, p in synth.frames(synth.SceneConfig(seed=1), 8)]   # 64 x 1875 = 120 k points
    out = dict(card=card(), frame_dev_fps=frame_rounds(bench, a.rounds, a.steps),
               seq_tick_8x120k_per_s=tick_rounds(bench, a.rounds, a.steps // 4), kernel_times=kernel_times(bench, 40))
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
