"""Box search on the GPU: what a searching frame costs.

  1. lmot_frame_dev frames/s on the bench scene (120 k points) with the search off, at A = 90 and at A = 360, in alternating rounds
  2. one 8-sequence lmot_seq_dev tick of the bench frames, no sequence searching vs all eight at A = 90
  3. box_search_kernel's device time (torch.profiler) at those sizes, and for one cluster of 110 k points
  4. the card's name and power limit, read in the same call
Prints one JSON object (and writes it to --out); every rate and time is a median over rounds with its min / max.
"""
import argparse
import importlib
import json
import math
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")

ARMS = (("off", 0), ("A90", 90), ("A360", 360))


def spread(xs):
    return dict(median=statistics.median(xs), min=min(xs), max=max(xs), rounds=len(xs))


def _ctx(A, params=None):
    c = pkg.Lmot(params)
    if A:
        c.set_box_search(on=1, n_angles=A)
    return c


def frame_rounds(frames, rounds, steps):
    d = [torch.from_numpy(p).cuda() for _, p in frames]
    ctx = {name: _ctx(A) for name, A in ARMS}
    res = {name: [] for name in ctx}
    ts = 0.0
    for r in range(rounds + 1):
        for name, c in ctx.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(steps):
                ts += 1e5
                x = d[i % len(d)]
                c.frame_dev(x.data_ptr(), x.shape[0], ts)
            c.frame_fetch()
            dt = time.perf_counter() - t0
            if r > 0:                        # round 0 warms up
                res[name].append(steps / dt)
    for c in ctx.values():
        c.close()
    return {name: spread(v) for name, v in res.items()}


def seq_rounds(frames, rounds, steps):
    d = [torch.from_numpy(p).cuda() for _, p in frames]
    ctx = {}
    for arm in ("none", "all_A90"):
        c = pkg.Lmot()
        c.seq_open(8)
        if arm != "none":
            for k in range(8):
                c.seq_set_box_search(k, on=1, n_angles=90)
        ctx[arm] = c
    res = {arm: [] for arm in ctx}
    ts = 0.0
    for r in range(rounds + 1):
        for arm, c in ctx.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(steps):
                ts += 1e5
                c.seq_dev([(x.data_ptr(), x.shape[0]) for x in d], [ts] * 8)
            c.seq_fetch()
            dt = time.perf_counter() - t0
            if r > 0:
                res[arm].append(steps / dt)
    for c in ctx.values():
        c.close()
    return {arm: spread(v) for arm, v in res.items()}


def _profile(run, names):
    from torch.profiler import ProfilerActivity, profile
    run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    out = {}
    for key, sub in names.items():
        us = [e.device_time for e in prof.events() if sub in e.name]
        out[key] = spread(us) if us else None
    return out


def kernel_times(frames, steps):
    d = [torch.from_numpy(p).cuda() for _, p in frames]
    out = {}
    for name, A in ARMS:
        c = _ctx(A)
        ts = [0.0]

        def run():
            for i in range(steps):
                ts[0] += 1e5
                c.frame_dev(d[i % len(d)].data_ptr(), d[i % len(d)].shape[0], ts[0])
            c.frame_fetch()
        out[f"frame_{name}"] = _profile(run, dict(box_search_kernel_us="box_search_kernel", box_fit_kernel_us="box_fit_kernel"))
        c.close()
    c = pkg.Lmot()
    c.seq_open(8)
    for k in range(8):
        c.seq_set_box_search(k, on=1, n_angles=90)
    ts = [0.0]

    def run_seq():
        for i in range(steps // 4):
            ts[0] += 1e5
            c.seq_dev([(x.data_ptr(), x.shape[0]) for x in d], [ts[0]] * 8)
        c.seq_fetch()
    out["seq_8x120k_A90"] = _profile(run_seq, dict(box_search_kernel_us="box_search_kernel"))
    c.close()
    # one cluster of 110 k points (a car-sized block) on a ground grid
    rng = np.random.default_rng(11)
    g = np.arange(-24.0, 24.0, 0.5)
    gx, gy = np.meshgrid(g, g)
    ground = np.zeros((gx.size, 4), np.float32)
    ground[:, 0], ground[:, 1], ground[:, 2] = gx.ravel(), gy.ravel(), -1.73
    n = 110_000
    u, w = rng.uniform(-2.25, 2.25, n), rng.uniform(-0.9, 0.9, n)
    blk = np.zeros((n, 4), np.float32)
    blk[:, 0] = 12.0 + math.cos(0.8) * u - math.sin(0.8) * w
    blk[:, 1] = -6.0 + math.sin(0.8) * u + math.cos(0.8) * w
    blk[:, 2] = rng.uniform(-1.3, -0.2, n)
    big = torch.from_numpy(np.concatenate([ground, blk])).cuda()
    for name, A in ARMS[1:]:
        p = pkg.default_params()
        p.max_points = 1 << 18
        c = _ctx(A, p)
        ts = [0.0]

        def run_big():
            for _ in range(10):
                ts[0] += 1e5
                c.frame_dev(big.data_ptr(), big.shape[0], ts[0])
            c.frame_fetch()
        out[f"cluster_110k_{name}"] = _profile(run_big, dict(box_search_kernel_us="box_search_kernel"))
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
    frames = list(synth.frames(synth.SceneConfig(seed=1), 8))         # the bench scene: 64 x 1875 = 120 k points
    out = dict(card=card(), frame_dev_fps=frame_rounds(frames, a.rounds, a.steps),
               seq_dev_8x120k_ticks_per_s=seq_rounds(frames, a.rounds, a.steps // 4), kernel_times=kernel_times(frames, 40))
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
