"""Does a radius outlier filter in front of clustering recover what snow costs?  Measured on the CPU with the reference's own chain.

For synth.py's scene (60 cars and pedestrians inside +-25 m) rendered by a 64- and a 32-beam sensor, clean and with light, moderate and
heavy snow (tests/weather_scenes.py), the reference's groundRemove -> componentClustering -> boxFitting runs on E and on E_kept, the
points of E the filter keeps (the NumPy restatement of include/lmot.h's definition), for the defaults and for other settings.  An object
is found when a box centre lies within 1 m of its centre; a ghost is a box within 1 m of no object.  Per cell: objects found, ghost
boxes, objects found only with the filter (+), objects lost to it (-) and points removed.  Needs oracle/_ref (built by build()).
"""
import argparse
import importlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
import weather_scenes as ws  # noqa: E402
from oracle import ref  # noqa: E402

SETTINGS = {"defaults": {}, "k=2": dict(min_neighbors=2), "k=1": dict(min_neighbors=1), "beta=5": dict(beta=5.0)}


def matched(boxes, obj):
    c = ws.centres(boxes)
    d = np.hypot(c[:, None, 0] - obj[None, :, 0], c[:, None, 1] - obj[None, :, 1]) <= 1.0
    return d.any(0), int((~d.any(1)).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, nargs="+", default=[5, 6])
    ap.add_argument("--frames", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    oracle = ref.RefOracle("intended")
    table = []
    for sensor in ws.SENSORS:
        for level in [None, *ws.SNOW]:
            row = dict(sensor=sensor, snow=level or "clean", found=0, ghosts=0, arms={k: dict(found=0, ghosts=0, recovered=0, lost=0, removed=0)
                                                                                      for k in SETTINGS})
            for seed in a.seeds:
                for pts, obj in ws.scene_frames(synth, sensor, a.frames, seed=seed, level=level):
                    _, b, e = ws.ref_detect(oracle, pts)
                    fe, ge = matched(b, obj)
                    row["found"] += int(fe.sum()); row["ghosts"] += ge
                    for name, s in SETTINGS.items():
                        _, bk, ek = ws.ref_detect(oracle, pts, dict(ws.DEFAULTS, **s))
                        fk, gk = matched(bk, obj)
                        q = row["arms"][name]
                        q["found"] += int(fk.sum()); q["ghosts"] += gk
                        q["recovered"] += int((fk & ~fe).sum()); q["lost"] += int((fe & ~fk).sum()); q["removed"] += len(e) - len(ek)
            table.append(row)
            print(f"{sensor:>2} {row['snow']:>8}  E: found {row['found']:3d} ghosts {row['ghosts']:3d}  | " +
                  " | ".join(f"{k}: {q['found']:3d} {q['ghosts']:3d} +{q['recovered']} -{q['lost']} rm {q['removed']}"
                             for k, q in row["arms"].items()), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(seeds=a.seeds, frames=a.frames, table=table), f, indent=1)


if __name__ == "__main__":
    main()
