"""Does background subtraction let a stationary sensor box what moves and stop boxing what stands?  Measured on the CPU with the
reference's own chain.

A sensor that does not move sees synth.py's scene (40 objects inside +-25 m) plus static structure that never moves: poles and hedges,
tree trunks and canopies, shelter roofs and a sign gantry, and parked cars (tests/background_scenes.py).  It is rendered by the 64- and
the 32-beam sensor of tests/weather_scenes.py.  The first L frames learn the background table (the NumPy restatement of DESIGN.md §6n's
definition); the next frames are scored.  On each scored frame the reference's groundRemove -> componentClustering -> boxFitting runs on
E and on E_fg, the points of E in front of the background, for every margin_m and nbr_cols of the sweep.  An object is found when a box
centre lies within 1 m of its centre; a ghost is a box within 1 m of no scored object.  The scored objects are the objects that move,
including those that park or leave in the two changing scenes:
  moving: every mover moves through learning and scoring;
  leave:  every second mover stands parked through learning, then drives off;
  arrive: every second mover is absent during learning, then appears and parks.
Per cell: objects found, ghost boxes, objects found only on E_fg (+), objects lost on E_fg (-), of those the objects that stand where
they stood through all of learning (learned), and the share of E removed.
Needs oracle/_ref (built by build()).
"""
import argparse
import importlib
import json
import os
import sys
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import background_scenes as bs  # noqa: E402

MARGINS = (0.2, 0.3, 0.5)
NBR_COLS = (0, 1, 2)


def run_one(job):
    sensor, mode, seed, learn, scored = job
    from oracle import ref
    synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
    oracle = ref.RefOracle("intended")
    learner = bs.Learner(learn_frames=learn)
    arms = {(m, n): dict(found=0, ghosts=0, recovered=0, lost=0, lost_learned=0, removed=0) for m in MARGINS for n in NBR_COLS}
    row = dict(sensor=sensor, mode=mode, seed=seed, objects=0, learned=0, found=0, ghosts=0, points=0)
    tables = None
    for pts, obj, learned, learning in bs.stationary_frames(synth, sensor, mode, learn, scored, seed):
        e, g = oracle.ground_remove(pts)
        if learning:
            learner.learn(np.concatenate([e, g]))
            continue
        if tables is None:
            tables = {n: learner.freeze(nbr_cols=n) for n in NBR_COLS}
        fe, ge = bs.matched(bs.ref_boxes(oracle, e), obj)
        row["objects"] += len(obj); row["learned"] += int(learned.sum())
        row["found"] += int(fe.sum()); row["ghosts"] += ge; row["points"] += len(e)
        for (m, n), q in arms.items():
            ef = bs.foreground(e, tables[n], margin_m=m)
            fk, gk = bs.matched(bs.ref_boxes(oracle, ef), obj)
            q["found"] += int(fk.sum()); q["ghosts"] += gk
            q["recovered"] += int((fk & ~fe).sum()); q["lost"] += int((fe & ~fk).sum())
            q["lost_learned"] += int((fe & ~fk & learned).sum()); q["removed"] += len(e) - len(ef)
    row["arms"] = {f"m={m} c={n}": q for (m, n), q in arms.items()}
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, nargs="+", default=[5, 6])
    ap.add_argument("--learn", type=int, default=bs.DEFAULTS["learn_frames"])
    ap.add_argument("--scored", type=int, default=20)
    ap.add_argument("--jobs", type=int, default=os.cpu_count())
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    jobs = [(s, m, seed, a.learn, a.scored) for s in bs.ws.SENSORS for m in bs.MODES for seed in a.seeds]
    with ProcessPoolExecutor(min(a.jobs, len(jobs))) as ex:
        rows = list(ex.map(run_one, jobs))
    table = []
    for s in bs.ws.SENSORS:
        for m in bs.MODES:
            rs = [r for r in rows if r["sensor"] == s and r["mode"] == m]
            tot = {f: sum(r[f] for r in rs) for f in ("objects", "learned", "found", "ghosts", "points")}
            tot.update(sensor=s, mode=m, arms={})
            for k in rs[0]["arms"]:
                tot["arms"][k] = {f: sum(r["arms"][k][f] for r in rs) for f in rs[0]["arms"][k]}
            table.append(tot)
            print(f"{s:>2} {m:>7}  objects {tot['objects']:4d} (learned {tot['learned']})  "
                  f"E: found {tot['found']:4d} ghosts {tot['ghosts']:4d}", flush=True)
            for k, q in tot["arms"].items():
                print(f"    {k}: found {q['found']:4d} ghosts {q['ghosts']:4d} +{q['recovered']} -{q['lost']} "
                      f"(learned {q['lost_learned']}) removed {100.0 * q['removed'] / max(tot['points'], 1):.1f} %", flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(seeds=a.seeds, learn=a.learn, scored=a.scored, table=table), f, indent=1)


if __name__ == "__main__":
    main()
