#!/usr/bin/env python3
"""Sweep deskew (lmot_set_deskew / lmot_seq_set_deskew): what the extra pass costs.

Two comparisons over device data, each timed with a host clock around work that ends in a result wait (frame_fetch / seq_fetch wait
for the last submission, which is published after every earlier one).  The arms alternate round by round; round 0 warms up.

  (a) frames/s through lmot_frame_dev on the bench scene (synth.py, 64 x 1875 = 120 k points), deskew off against on;
  (b) ticks/s of an 8 x 120 k lmot_seq_dev tick, no sequence deskewing against all eight.

With deskew on, every point's time comes from its azimuth column (a 100 ms sweep) and the ego moves at 12 m/s, turning at 0.2 rad/s.
Prints one JSON line per comparison with the card name, power limit and max SM clock.  Needs a GPU; there is no CPU fallback.
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def with_time(p, azimuths):
    p = np.ascontiguousarray(p).copy()
    tau = (-0.1 + (np.arange(azimuths) + 0.5) / azimuths * 0.1).astype(np.float32)
    p[:, 3] = np.tile(tau, len(p) // azimuths)
    return p


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=400, help="frames per round in (a)")
    ap.add_argument("--ticks", type=int, default=100, help="ticks per round in (b)")
    ap.add_argument("--rounds", type=int, default=6)
    args = ap.parse_args()
    info = card()
    cfg = synth.SceneConfig()                                    # the bench scene: 64 x 1875
    host = [with_time(p, cfg.azimuths) for _, p in synth.frames(cfg, 16)]
    dev = [torch.from_numpy(p).cuda() for p in host]
    seq_host = [[with_time(p, cfg.azimuths) for _, p in synth.frames(synth.SceneConfig(seed=300 + k), 4)] for k in range(8)]
    seq_dev = [[torch.from_numpy(p).cuda() for p in fr] for fr in seq_host]
    torch.cuda.synchronize()
    ego = lambda t: (12.0, 0.02 * t)                             # 0.2 rad/s at 10 Hz

    def timed(run):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run()
        return time.perf_counter() - t0

    def report(name, arms, unit, n):
        out = {"comparison": name, "gpu": info, "rounds": args.rounds, "per_round": n}
        for arm, xs in arms.items():
            s = np.array(xs)
            out[arm] = {f"{unit}_per_s_median": round(float(n / np.median(s)), 1), "min": round(float(n / s.max()), 1),
                        "max": round(float(n / s.min()), 1), "us_per_" + unit + "_median": round(float(np.median(s)) * 1e6 / n, 2)}
        print(json.dumps(out), flush=True)

    # (a) lmot_frame_dev, deskew off / on
    ctxs = {}
    for arm in ("off", "on"):
        p = pkg.default_params()
        ctxs[arm] = pkg.Lmot(p)
        if arm == "on":
            ctxs[arm].set_deskew(on=1)
    clock = {"off": 0, "on": 0}

    def run_frames(arm):
        c = ctxs[arm]
        for _ in range(args.frames):
            t = clock[arm]
            d = dev[t % len(dev)]
            c.frame_dev(d.data_ptr(), len(host[0]), 1.0e6 + 1.0e5 * t, *ego(t))
            clock[arm] += 1
        c.frame_fetch(want_boxes=False)

    arms = {"off": [], "on": []}
    for r in range(args.rounds + 1):
        for arm in (("off", "on") if r % 2 else ("on", "off")):
            dt = timed(lambda: run_frames(arm))
            if r:
                arms[arm].append(dt)
    for c in ctxs.values():
        c.close()
    report("a_frame_dev_120k", arms, "frame", args.frames)

    # (b) an 8 x 120 k lmot_seq_dev tick, no sequence deskewing / all eight
    ctxs = {}
    for arm in ("off", "on"):
        p = pkg.default_params()
        p.max_points = 1 << 17
        p.max_tracks = 2048
        c = pkg.Lmot(p)
        c.seq_open(8, ring=8)
        if arm == "on":
            for k in range(8):
                c.seq_set_deskew(k, on=1)
        ctxs[arm] = c
    clock = {"off": 0, "on": 0}

    def run_ticks(arm):
        c = ctxs[arm]
        for _ in range(args.ticks):
            t = clock[arm]
            fr = [(seq_dev[k][t % 4].data_ptr(), len(seq_host[k][0])) for k in range(8)]
            c.seq_dev(fr, [1.0e6 + 1.0e5 * t] * 8, [12.0] * 8, [0.02 * t + 0.1 * k for k in range(8)])
            clock[arm] += 1
        c.seq_fetch(want_boxes=False)

    arms = {"off": [], "on": []}
    for r in range(args.rounds + 1):
        for arm in (("off", "on") if r % 2 else ("on", "off")):
            dt = timed(lambda: run_ticks(arm))
            if r:
                arms[arm].append(dt)
    for c in ctxs.values():
        c.close()
    report("b_seq_dev_8x120k", arms, "tick", args.ticks)


if __name__ == "__main__":
    main()
