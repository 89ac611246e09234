"""Layered clustering on the GPU: what it costs and what it recovers.

  1. device time (torch.profiler) of clustering per unit: layer_mark_kernel + ccl_layer_kernel with layers on (S = 32, g = 2) against
     ccl_dense_kernel with them off, on the bench scene (120 k points) and on tests/layer_scenes.py's canopy scene, for one unit
     (lmot_frame_dev) and for 8 units (one 8-sequence lmot_seq_dev tick).  The profiled runs set LMOT_FUSE_CCL=0, so that the unlayered
     clustering is a launch of its own rather than the ground kernel's tail
  2. lmot_frame_dev frames/s on the bench scene with layers off and on, in alternating rounds (clustering fused, as the library runs)
  3. objects of the canopy scene (64- and 32-beam) with a box, off and on, through lmot_frame
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
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
import layer_scenes as ls  # noqa: E402

ARMS = ("off", "on")


def spread(xs):
    return dict(median=statistics.median(xs), min=min(xs), max=max(xs), rounds=len(xs))


def _ctx(arm, n_seq=0):
    c = pkg.Lmot()
    if n_seq:
        c.seq_open(n_seq)
    if arm == "on":
        c.set_layers(on=1)
        for k in range(n_seq):
            c.seq_set_layers(k, on=1)
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


KERNELS = ("layer_mark_kernel", "ccl_layer_kernel", "ccl_dense_kernel")


def _profile(run):
    from torch.profiler import ProfilerActivity, profile
    run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    out = {}
    for k in KERNELS:
        ev = [e.device_time for e in prof.events() if e.device_type.name == "CUDA" and re.search(rf"\b{k}\b", e.name)]
        if ev:
            out[k + "_us"] = spread(ev)
    return out


def kernel_times(scenes, steps):
    out = {}
    for name, d in scenes.items():
        for arm in ARMS:
            c = _ctx(arm)
            ts = [0.0]

            def run():
                for i in range(steps):
                    ts[0] += 1e5
                    c.frame_dev(d[i % len(d)].data_ptr(), d[i % len(d)].shape[0], ts[0])
                c.frame_fetch()
            out[f"{name}_1_unit_{arm}"] = _profile(run)
            c.close()
            c = _ctx(arm, 8)

            def run_seq():
                for i in range(steps // 4):
                    ts[0] += 1e5
                    c.seq_dev([(d[j % len(d)].data_ptr(), d[j % len(d)].shape[0]) for j in range(8)], [ts[0]] * 8)
                c.seq_fetch()
            out[f"{name}_8_units_{arm}"] = _profile(run_seq)
            c.close()
    return out


def objects():
    out = {}
    for sensor in ("64", "32"):
        pts, objs = ls.render(sensor)
        for arm in ARMS:
            c = _ctx(arm)
            r = c.frame(pts, 1e6)
            c.close()
            out[f"{sensor}_beam_{arm}"] = {k: ls.found(r["boxes"], objs, k) for k in
                                           ("car_canopy", "ped_shelter", "car_gantry", "truck", "car_open", "ped_open")}
        out[f"{sensor}_beam_objects"] = {k: sum(o[2] == k for o in objs) for k in out[f"{sensor}_beam_on"]}
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
    ap.add_argument("--kernels", action="store_true", help="internal: only the profiled kernel times (run with LMOT_FUSE_CCL=0)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    bench = [torch.from_numpy(p).cuda() for _, p in synth.frames(synth.SceneConfig(seed=1), 8)]   # 64 x 1875 = 120 k points
    canopy = [torch.from_numpy(ls.render("64", seed=s)[0]).cuda() for s in (7, 8)]
    if a.kernels:
        print(json.dumps(kernel_times(dict(bench=bench, canopy=canopy), 40)))
        return
    env = dict(os.environ, LMOT_FUSE_CCL="0")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--kernels"], env=env, capture_output=True, text=True, timeout=1200)
    if r.returncode != 0:
        raise RuntimeError(r.stderr[-2000:])
    out = dict(card=card(), kernel_times=json.loads(r.stdout.strip().splitlines()[-1]),
               frame_dev_fps=frame_rounds(bench, a.rounds, a.steps), objects=objects())
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
