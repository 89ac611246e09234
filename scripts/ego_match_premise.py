"""Premise of scan-matched ego motion (include/lmot.h, lmot_ego_estimate), on the CPU: does the matcher at its defaults recover the fold's
motion well enough to stand in for GPS ego?

Drives: accumulate_scenes' straight (4 m/s) and turning (3 m/s, 0.04 rad per step) routes through its static scene, rendered from the
library's fold (tests/ego_match_scenes.py drive_frames) at 16, 32 and 64 beams, plus the 32-beam drives with 12 of synth's movers.  Per
drive of 40 steps, with the NumPy restatement of the estimator:
  * v / dtheta errors of each matched step against the fold's true delta (median and max, steps 2..40);
  * the fold after 40 steps fed with matched ego and with v = 0 (constant yaw), against the GPS fold: position (m) and yaw (rad);
  * the reference tracker's (oracle port) static-flag count over the drive (sum over steps of the tracks flagged static) with GPS ego,
    matched ego and v = 0.
Prints one JSON line per drive and a summary table.  Usage: python scripts/ego_match_premise.py [--steps 40] [--beams 16 32 64]"""
import argparse
import importlib
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import ego_match_scenes as em  # noqa: E402
from oracle import ref  # noqa: E402

synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")


def static_count(oracle, frames, ego):
    oracle.tracker_reset()
    tot = 0
    for (ts, _, _, pts, _, _), (v, yaw) in zip(frames, ego):
        e, _ = oracle.ground_remove(pts)
        grid, k = oracle.component_clustering(e)
        boxes, _ = oracle.box_fitting(e, grid, k)
        r = oracle.tracker_step(boxes, ts, v, yaw)
        tot += int(np.sum(r["is_static"] == 1))
    return tot


def fold_of(frames, ego):
    h = dict(init=False, ts=0.0, pre_yaw=0.0, fold=None)
    f = None
    for (ts, *_), (v, yaw) in zip(frames, ego):
        f = em.fold_step(h, ts, v, yaw)
    return f


def one(kind, beams, movers, steps, oracle):
    frames = em.drive_frames(synth, kind, steps, beams=beams, movers=movers)
    m = em.Matcher()
    outs = [m.estimate(f[3], f[0]) for f in frames]
    ev, eth, oks = [], [], 0
    for t in range(1, steps):
        dt = (frames[t][0] - frames[t - 1][0]) / 1e6
        _, _, dth = em.true_delta(frames[t - 1][4], frames[t][4], dt, frames[t][1])
        ev.append(abs(outs[t]["v"] - frames[t][1]))
        eth.append(abs(outs[t]["dtheta"] - dth))
        oks += outs[t]["ok"]
    gps = [(f[1], f[2]) for f in frames]
    mat = [(o["v"], o["yaw"]) for o in outs]
    zero = [(0.0, 0.0)] * steps
    fg, fm, f0 = fold_of(frames, gps), fold_of(frames, mat), fold_of(frames, zero)
    row = dict(kind=kind, beams=beams, movers=movers, steps=steps, ok=oks, n_used_med=int(np.median([o["n_used"] for o in outs[1:]])),
               v_err_med=float(np.median(ev)), v_err_max=float(max(ev)), th_err_med=float(np.median(eth)), th_err_max=float(max(eth)),
               fold_pos_err_matched=float(math.hypot(fm[0] - fg[0], fm[1] - fg[1])), fold_yaw_err_matched=float(abs(fm[2] - fg[2])),
               fold_pos_err_v0=float(math.hypot(f0[0] - fg[0], f0[1] - fg[1])), fold_yaw_err_v0=float(abs(f0[2] - fg[2])))
    if oracle is not None:
        row.update(static_gps=static_count(oracle, frames, gps), static_matched=static_count(oracle, frames, mat),
                   static_v0=static_count(oracle, frames, zero))
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--beams", type=int, nargs="+", default=[16, 32, 64])
    ap.add_argument("--no-tracker", action="store_true", help="skip the static-flag runs")
    a = ap.parse_args()
    oracle = None if a.no_tracker else (ref.RefOracle("intended") if ref.have_ref("intended") else ref.PortOracle())
    cases = [(k, b, 0) for b in a.beams for k in ("straight", "turn")]
    if 32 in a.beams:
        cases += [(k, 32, 12) for k in ("straight", "turn")]
    rows = []
    for kind, beams, movers in cases:
        r = one(kind, beams, movers, a.steps, oracle)
        rows.append(r)
        print(json.dumps(r), flush=True)
    print(f"{'drive':<22}{'ok':>4}{'n_used':>7}{'|dv| med/max':>16}{'|dth| med/max':>20}{'fold m/v0 (m)':>18}{'static gps/m/v0':>18}")
    for r in rows:
        st = f"{r.get('static_gps', '-')}/{r.get('static_matched', '-')}/{r.get('static_v0', '-')}"
        print(f"{r['kind'] + ' ' + str(r['beams']) + ('+movers' if r['movers'] else ''):<22}{r['ok']:>4}{r['n_used_med']:>7}"
              f"{r['v_err_med']:>8.3f}/{r['v_err_max']:<7.3f}{r['th_err_med']:>10.5f}/{r['th_err_max']:<9.5f}"
              f"{r['fold_pos_err_matched']:>8.3f}/{r['fold_pos_err_v0']:<9.2f}{st:>18}")


if __name__ == "__main__":
    main()
