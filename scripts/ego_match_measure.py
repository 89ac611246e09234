"""Cost of scan-matched ego motion on the GPU (lmot_ego_estimate_dev, lmot_seq_ego_estimate_dev) at its default settings.

  * time per estimate on the 120 k-point synth scene (64 x 1875 rays, device frames): one stream, and 8 sequences in one call.  The calls
    are synchronous (they end in a synchronisation of the matcher stream), so a host clock around each call measures the device work plus
    the host's share of it; median and p90 over `--iters` calls after `--warmup`, consecutive frames of a moving-object scene;
  * lmot_frame_dev frames/s with and without an estimate of the same frame before each frame, in alternating rounds.
Writes measure_out/ego_match_measure.json (or --out) and prints it, with the device name and power limit."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:                      # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--out", default=os.path.join(ROOT, "measure_out", "ego_match_measure.json"))
    a = ap.parse_args()
    n_fr = 16
    frames = [p for _, p in synth.frames(synth.SceneConfig(seed=1), n_fr)]
    dev = [torch.from_numpy(p).cuda() for p in frames]
    torch.cuda.synchronize()
    res = dict(gpu=gpu_info(), points=len(frames[0]))

    ctx = pkg.Lmot()
    t_us, outs = [], []
    for i in range(a.warmup + a.iters):
        f = i % n_fr
        t0 = time.perf_counter()
        o = ctx.ego_estimate_dev(dev[f].data_ptr(), len(frames[f]), (i + 1) * 1e5)
        t1 = time.perf_counter()
        if i >= a.warmup:
            t_us.append((t1 - t0) * 1e6)
            outs.append(o)
    res["one_stream_us"] = dict(median=float(np.median(t_us)), p90=float(np.percentile(t_us, 90)))
    res["one_stream_ok_frac"] = float(np.mean([o["ok"] for o in outs]))
    res["n_used_median"] = float(np.median([o["n_used"] for o in outs]))
    ctx.seq_open(8, ring=2)
    t_us = []
    for i in range(a.warmup + a.iters):
        ptrs = [dev[(i + k) % n_fr].data_ptr() for k in range(8)]
        t0 = time.perf_counter()
        ctx.seq_ego_estimate_dev(ptrs, [len(frames[0])] * 8, [(i + 1) * 1e5] * 8)
        t1 = time.perf_counter()
        if i >= a.warmup:
            t_us.append((t1 - t0) * 1e6)
    res["eight_sequences_us"] = dict(median=float(np.median(t_us)), p90=float(np.percentile(t_us, 90)))
    ctx.close()

    rates = {"plain": [], "with_estimate": []}
    for r in range(a.rounds):
        for arm in ("plain", "with_estimate") if r % 2 == 0 else ("with_estimate", "plain"):
            ctx = pkg.Lmot()
            for i in range(30):                  # warm-up: every slot and the matcher's first-call allocations
                if arm == "with_estimate":
                    ctx.ego_estimate_dev(dev[i % n_fr].data_ptr(), len(frames[0]), (i + 1) * 1e5)
                ctx.frame_dev(dev[i % n_fr].data_ptr(), len(frames[0]), (i + 1) * 1e5)
                ctx.frame_fetch()
            ctx.sync()
            t0 = time.perf_counter()
            for i in range(30, 30 + a.frames):
                ts = (i + 1) * 1e5
                if arm == "with_estimate":
                    ctx.ego_estimate_dev(dev[i % n_fr].data_ptr(), len(frames[0]), ts)
                ctx.frame_dev(dev[i % n_fr].data_ptr(), len(frames[0]), ts)
                ctx.frame_fetch()
            ctx.sync()
            rates[arm].append(a.frames / (time.perf_counter() - t0))
            ctx.close()
    res["frame_dev_fps"] = {k: dict(median=float(np.median(v)), rounds=[round(x, 1) for x in v]) for k, v in rates.items()}
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
