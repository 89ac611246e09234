#!/usr/bin/env python3
"""Merging rigs (lmot_set_rig_merge / lmot_seq_set_rig_merge): ticks/s with separate and with merged detection.

Three comparisons over device data, each timed with a host clock around work that ends in a result wait (batch_fetch / seq_fetch wait for
the last submission, which is published after every earlier one).  The arms alternate round by round; round 0 warms up.

  (a) a 4 x 120 k lmot_batch_dev tick of a 4-sensor rig, separate against merged;
  (b) the same with 8 sensors (8 x 120 k);
  (c) a two-sequence lmot_seq_dev tick, each sequence a 4-sensor rig (8 x 120 k in all), neither merging against both.

Every sensor's frame is a bench scene (synth.py, 64 x 1875 points) of its own seed, mounted at a quarter-turn yaw.  Prints one JSON line
per comparison with the card name, power limit and max SM clock.  --trace: one torch.profiler run of (b) merged instead, printing the
mean GPU time of every kernel of a tick (rig_merge_kernel's among them).  Needs a GPU; there is no CPU fallback.
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")

QUARTER = [(1, 0), (0, 1), (-1, 0), (0, -1)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def poses(n):
    out = []
    for k in range(n):
        c, s = QUARTER[k % 4]
        out.append(np.array([[c, -s, 0, 0.5 * c], [s, c, 0, 0.5 * s], [0, 0, 1, 0]], np.float32))
    return out


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=300, help="ticks per round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--trace", action="store_true")
    args = ap.parse_args()
    info = card()
    host = [[p for _, p in synth.frames(synth.SceneConfig(seed=400 + k), 4)] for k in range(8)]
    dev = [[torch.from_numpy(p).cuda() for p in fr] for fr in host]
    n0 = len(host[0][0])
    torch.cuda.synchronize()

    def batch_ctx(F, merge):
        c = pkg.Lmot(pkg.default_params())
        c.set_sensors(poses(F))
        c.set_rig_merge(merge)
        return c

    def batch_run(c, F, clock, n):
        for _ in range(n):
            t = clock[0]
            c.batch_dev([(dev[k][t % 4].data_ptr(), n0) for k in range(F)], 1.0e6 + 1.0e5 * t, 5.0, 0.01 * t)
            clock[0] += 1
        c.batch_fetch(want_boxes=False)

    if args.trace:
        from torch.profiler import ProfilerActivity, profile
        c = batch_ctx(8, 1)
        clock = [0]
        batch_run(c, 8, clock, 50)
        torch.cuda.synchronize()
        n = 100
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            batch_run(c, 8, clock, n)
            torch.cuda.synchronize()
        tot = {}
        for e in prof.events():
            if str(e.device_type).endswith("CUDA"):
                tot.setdefault(e.name, []).append(e.device_time)
        print(json.dumps({"trace": "b_batch_dev_8x120k_merged", "gpu": info, "ticks": n,
                          "kernels_us_per_tick": {k[:60]: round(sum(v) / n, 2) for k, v in sorted(tot.items(), key=lambda kv: -sum(kv[1]))}}))
        c.close()
        return

    def timed(run):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run()
        return time.perf_counter() - t0

    def compare(name, make, run):
        ctxs = {arm: make(arm == "merged") for arm in ("separate", "merged")}
        clocks = {arm: [0] for arm in ctxs}
        arms = {arm: [] for arm in ctxs}
        for r in range(args.rounds + 1):
            for arm in (("separate", "merged") if r % 2 else ("merged", "separate")):
                dt = timed(lambda: run(ctxs[arm], clocks[arm], args.ticks))
                if r:
                    arms[arm].append(dt)
        for c in ctxs.values():
            c.close()
        out = {"comparison": name, "gpu": info, "rounds": args.rounds, "per_round": args.ticks}
        for arm, xs in arms.items():
            s = np.array(xs)
            out[arm] = {"ticks_per_s_median": round(float(args.ticks / np.median(s)), 1), "min": round(float(args.ticks / s.max()), 1),
                        "max": round(float(args.ticks / s.min()), 1), "us_per_tick_median": round(float(np.median(s)) * 1e6 / args.ticks, 2)}
        print(json.dumps(out), flush=True)

    for F in (4, 8):
        compare(f"{'a' if F == 4 else 'b'}_batch_dev_{F}x120k", lambda m, F=F: batch_ctx(F, int(m)),
                lambda c, clock, n, F=F: batch_run(c, F, clock, n))

    def seq_ctx(merge):
        c = pkg.Lmot(pkg.default_params())
        c.seq_open(2, ring=8)
        for k in range(2):
            c.seq_set_sensors(k, poses(4))
            c.seq_set_rig_merge(k, int(merge))
        return c

    def seq_run(c, clock, n):
        for _ in range(n):
            t = clock[0]
            fr = [[(dev[4 * s + j][t % 4].data_ptr(), n0) for j in range(4)] for s in range(2)]
            c.seq_dev(fr, [1.0e6 + 1.0e5 * t] * 2, [5.0] * 2, [0.01 * t, 0.5 + 0.01 * t])
            clock[0] += 1
        c.seq_fetch(want_boxes=False)

    compare("c_seq_dev_2x4x120k", seq_ctx, seq_run)


if __name__ == "__main__":
    main()
