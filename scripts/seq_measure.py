"""Independent sequences on one GPU: frames/s of S independent 120 k-point HDL-64 streams (S = 1, 2, 4, 8; different synth seeds and ego
motions, frames resident on the device), two arms alternated round by round:
  contexts  S contexts, each fed by lmot_frame_dev on its own caller stream
  seq       one context, one lmot_seq_dev tick per S frames (one tracker chain for all S tables)
Frames/s = S x ticks/s, host clock around the timed ticks, bracketed by device synchronisations.  After each round the final track
tables of the two arms are compared (they must be equal).  Prints the card name and power limit beside the numbers.  Needs a CUDA
device; there is no CPU path.

    python scripts/seq_measure.py [--ticks 30] [--rounds 3] [--warm 4]
"""
import argparse
import importlib
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
lmot = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")

ap = argparse.ArgumentParser()
ap.add_argument("--ticks", type=int, default=30)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--warm", type=int, default=4)
ap.add_argument("--sizes", default="1,2,4,8")
a = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("seq_measure.py: no CUDA device")
card = torch.cuda.get_device_name(0)
try:
    pl = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                        capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as ex:                  # the numbers below still stand, without the power limit
    pl = f"unavailable ({type(ex).__name__})"

sizes = [int(s) for s in a.sizes.split(",")]
S_MAX = max(sizes)
n_t = a.warm + a.ticks
streams = [[p for _, p in synth.frames(synth.SceneConfig(seed=211 + 13 * k), n_t)] for k in range(S_MAX)]
n = len(streams[0][0])
dev = [torch.from_numpy(np.stack(s)).cuda() for s in streams]
ts = lambda k, t: 1.0e6 * (k + 1) + 1.0e5 * t                    # own start stamp per stream
ego = lambda k, t: (2.0 + k, 0.01 * (k - 3) * t)                 # own ego speed and yaw per stream
torch.cuda.synchronize()


def run_contexts(ctxs, S, t0, t1):
    for t in range(t0, t1):
        for k in range(S):
            ctxs[k][0].frame_dev(dev[k][t].data_ptr(), n, ts(k, t), *ego(k, t))


def run_seq(ctx, args, S, t0, t1):
    for t in range(t0, t1):
        ctx.seq_dev(args[t], [ts(k, t) for k in range(S)], [ego(k, t)[0] for k in range(S)], [ego(k, t)[1] for k in range(S)])


print(f"card: {card}; power limit, max SM clock: {pl}")
print(f"{n} points per frame, {a.ticks} timed ticks after {a.warm} warm-up ticks, {a.rounds} rounds alternating the arms")
for S in sizes:
    ctxs = []
    for k in range(S):
        c = lmot.Lmot()
        st = torch.cuda.Stream()
        c.set_stream(st.cuda_stream)
        ctxs.append((c, st))
    seq = lmot.Lmot()
    seq_stream = torch.cuda.Stream()
    seq.set_stream(seq_stream.cuda_stream)
    seq.seq_open(S, ring=8)
    args = [seq.seq_prepare([(dev[k][t].data_ptr(), n) for k in range(S)]) for t in range(n_t)]
    rates = {"contexts": [], "seq": []}
    for rnd in range(a.rounds):
        for arm in ("contexts", "seq"):
            if arm == "contexts":
                for c, _ in ctxs:
                    c.tracker_reset()
                run = lambda t0, t1: run_contexts(ctxs, S, t0, t1)
            else:
                seq.seq_open(S, ring=8)
                run = lambda t0, t1: run_seq(seq, args, S, t0, t1)
            run(0, a.warm)
            torch.cuda.synchronize()
            h0 = time.perf_counter()
            run(a.warm, n_t)
            torch.cuda.synchronize()
            rates[arm].append(S * a.ticks / (time.perf_counter() - h0))
        for k in range(S):
            da, db = ctxs[k][0].tracker_dump(), seq.seq_tracker_dump(k)
            if da.shape != db.shape or not np.array_equal(da.view(np.uint64), db.view(np.uint64)):
                raise SystemExit(f"S={S} round {rnd}: sequence {k} differs from its context ({da.shape} vs {db.shape} rows)")
    print(f"S={S}: final tables equal in every round ({[len(ctxs[k][0].tracker_dump()) for k in range(S)]} tracks)")
    for arm, v in rates.items():
        v = np.array(v)
        print(f"S={S} {arm:8s} frames/s median {np.median(v):8.1f}  min {v.min():8.1f}  max {v.max():8.1f}  (ticks/s median {np.median(v) / S:8.1f})")
    for c, _ in ctxs:
        c.set_stream(None)
        c.close()
    seq.set_stream(None)
    seq.close()
