"""Detection areas on the GPU: what a masked submission costs, and what the area removes on a cluttered scene.

  1. lmot_frame_dev on the bench scene (120 k points), area off and on (a 5-vertex road polygon), in alternating rounds
  2. one tick of 8 x 120 k points through lmot_seq_dev, no sequence masked vs all eight masked with polygons that change every tick
  3. detect_area_kernel's device time (torch.profiler) at 16, 256 and 1024 vertices
  4. boxes and spawned tracks on the roadside clutter scene of the tests, without and with the road corridor as the area
Prints one JSON object (and writes it to --out); every time is a median over rounds with its min / max.
"""
import argparse
import importlib
import json
import math
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
from detect_area_scenes import CORRIDOR, cluttered_frames, near_clutter  # noqa: E402

ROAD = [np.array([[-24.0, -7.0], [24.0, -9.0], [24.0, 8.0], [0.0, 6.0], [-24.0, 9.0]])]


def polygon(nv, r=20.0, phase=0.0):
    t = np.linspace(0.0, 2 * math.pi, nv, endpoint=False) + phase
    rr = r * (1.0 + 0.2 * np.cos(5 * t))
    return [np.stack([rr * np.cos(t), 0.5 * rr * np.sin(t)], 1)]


def spread(xs):
    return dict(median=statistics.median(xs), min=min(xs), max=max(xs), rounds=len(xs))


def frame_rounds(frames, rounds, steps):
    d = [torch.from_numpy(p).cuda() for _, p in frames]
    ctx = {arm: pkg.Lmot() for arm in ("off", "on")}
    ctx["on"].set_detect_area(ROAD)
    res = {arm: [] for arm in ctx}
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
            dt = (time.perf_counter() - t0) / steps * 1e6
            if r > 0:                        # round 0 warms up
                res[arm].append(dt)
    for c in ctx.values():
        c.close()
    return {arm: spread(v) for arm, v in res.items()}


def seq_rounds(frames, rounds, steps):
    d = [torch.from_numpy(p).cuda() for _, p in frames]
    dev = [(x.data_ptr(), x.shape[0]) for x in d[:8]]
    out = {}
    res = {"none": [], "all8_changing": []}
    ctxs = {}
    for arm in res:
        c = pkg.Lmot()
        c.seq_open(8, ring=8)
        ctxs[arm] = c
    ts = 0.0
    for r in range(rounds + 1):
        for arm, c in ctxs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(steps):
                ts += 1e5
                if arm != "none":
                    for k in range(8):
                        c.seq_set_detect_area(k, polygon(16, 20.0, 0.01 * i + k))
                c.seq_dev(dev, [ts] * 8)
            c.seq_fetch()
            dt = (time.perf_counter() - t0) / steps * 1e6
            if r > 0:
                res[arm].append(dt)
    for c in ctxs.values():
        c.close()
    out.update({arm: spread(v) for arm, v in res.items()})
    return out


def kernel_times(frames, steps):
    from torch.profiler import ProfilerActivity, profile
    x = torch.from_numpy(frames[0][1]).cuda()
    out = {}
    for nv in (16, 256, 1024):
        c = pkg.Lmot()
        c.set_detect_area(polygon(nv))
        for i in range(5):
            c.frame_dev(x.data_ptr(), x.shape[0], (i + 1) * 1e5)
        c.frame_fetch()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(steps):
                c.frame_dev(x.data_ptr(), x.shape[0], (i + 10) * 1e5)
            c.frame_fetch()
            torch.cuda.synchronize()
        us = [e.device_time for e in prof.events() if "detect_area_kernel" in e.name]
        out[str(nv)] = spread(us)
        c.close()
    return out


def clutter(n_frames):
    res = {}
    for arm in ("no_area", "corridor"):
        c = pkg.Lmot()
        if arm == "corridor":
            c.set_detect_area(CORRIDOR)
        boxes = clutter_boxes = 0
        r = None
        for ts, p in cluttered_frames(synth, n_frames):
            r = c.frame(p, ts)
            boxes += len(r["boxes"])
            clutter_boxes += int(near_clutter(r["boxes"]).sum())
        tg = np.asarray(r["targets"]).reshape(-1, 3)
        res[arm] = dict(frames=n_frames, boxes=boxes, boxes_on_clutter=clutter_boxes, tracks_spawned=int(len(tg)),
                        tracks_outside_corridor=int((np.abs(tg[:, 1]) > 8.0).sum()))
        c.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = torch.cuda.get_device_name(0)
    frames = list(synth.frames(synth.SceneConfig(seed=1), 8))         # the bench scene: 64 x 1875 = 120 k points
    out = dict(gpu=gpu, frame_dev_us=frame_rounds(frames, a.rounds, a.steps), seq_dev_8x120k_us=seq_rounds(frames, a.rounds, a.steps // 4),
               detect_area_kernel_us=kernel_times(frames, 50), clutter=clutter(20))
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
