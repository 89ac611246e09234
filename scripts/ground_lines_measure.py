"""Ground lines on the GPU: what a frame with the lines on costs.

  1. lmot_frame_dev frames/s on the bench scene (120 k points) with the lines off and on, in alternating rounds
  2. one 8-sequence lmot_seq_dev tick of the bench frames, no sequence with lines vs all eight
  3. device time (torch.profiler) of the ground kernel (off: ground_fused_kernel, on: ground_fused_lines_kernel, whose phase 2 is the
     serial fp64 walk of each channel) and of box fitting (box_fit_kernel / box_fit_lines_kernel), per frame and per 8-sequence tick
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
        c.set_ground_lines(on=1)
        for k in range(n_seq):
            c.seq_set_ground_lines(k, on=1)
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


def seq_rounds(d, rounds, steps):
    ctx = {arm: _ctx(arm, 8) for arm in ARMS}
    res = {arm: [] for arm in ARMS}
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


KERNELS = dict(ground_us=("ground_fused_kernel", "ground_fused_lines_kernel", "ground_fused_frame_kernel"),
               box_fit_us=("box_fit_kernel", "box_fit_lines_kernel"))


def _profile(run):
    from torch.profiler import ProfilerActivity, profile
    run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    out = {}
    for key, subs in KERNELS.items():
        ev = [e for e in prof.events() if e.device_type.name == "CUDA" and any(s in e.name for s in subs)]
        out[key] = spread([e.device_time for e in ev]) if ev else None
        out[key.replace("_us", "_kernels")] = sorted({re.search(r"(\w+_kernel)", e.name).group(1) for e in ev})
    return out


def kernel_times(d, steps):
    out = {}
    for arm in ARMS:
        c = _ctx(arm)
        ts = [0.0]

        def run():
            for i in range(steps):
                ts[0] += 1e5
                c.frame_dev(d[i % len(d)].data_ptr(), d[i % len(d)].shape[0], ts[0])
            c.frame_fetch()
        out[f"frame_{arm}"] = _profile(run)
        c.close()
        c = _ctx(arm, 8)

        def run_seq():
            for i in range(steps // 4):
                ts[0] += 1e5
                c.seq_dev([(x.data_ptr(), x.shape[0]) for x in d], [ts[0]] * 8)
            c.seq_fetch()
        out[f"seq_8x120k_{arm}"] = _profile(run_seq)
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
    d = [torch.from_numpy(p).cuda() for _, p in frames]
    out = dict(card=card(), frame_dev_fps=frame_rounds(d, a.rounds, a.steps),
               seq_dev_8x120k_ticks_per_s=seq_rounds(d, a.rounds, a.steps // 4), kernel_times=kernel_times(d, 40))
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
