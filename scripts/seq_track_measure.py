"""Tracking-only streams on one GPU: tracker steps/s of S independent box-list streams (S = 1, 2, 4, 8; lists resident on the device),
two arms alternated round by round:
  A  contexts  S contexts, each stepped by lmot_track_step_lists_dev (one list) on its own caller stream
  B  seq       one context, one lmot_seq_track_dev tick per S lists (one tracker chain for all S tables)
Two workloads:
  bench     about 64 tracks and 30-64 boxes per step (48 moving objects, a varying subset seen, a few clutter boxes)
  stress    BASELINE.json configs[2]: 1024 mature tracks on a 32 x 32 lattice, 256 detections per step.  Unobserved tracks die within a
            few steps, so the timed ticks run in bursts of --burst ticks, each starting from the same 1024-track table (loaded untimed
            with lmot_tracker_load / lmot_seq_tracker_load, as bench.py's tracker_stress re-loads it before every step)
Steps/s = S x ticks/s, host clock around the timed ticks (summed over the bursts), bracketed by device synchronisations.  After each
round the final track tables of the two arms are compared (they must be equal).  Prints the card name, power limit and max SM clock
beside the numbers.  Needs a CUDA device; there is no CPU path.

    python scripts/seq_track_measure.py [--ticks 200] [--rounds 3] [--warm 10]
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


# the workloads (also imported by scripts/tracker_params_measure.py)
def boxes_at(c):
    out = np.zeros((len(c), 8, 3), np.float32)
    sign = np.array([[-1.0, -0.5], [-1.0, 0.5], [1.0, 0.5], [1.0, -0.5]])
    for k in range(4):
        out[:, k, :2] = c + sign[k]; out[:, k, 2] = -2.0
        out[:, 4 + k, :2] = c + sign[k]; out[:, 4 + k, 2] = 0.0
    return out


def bench_lists(k, n_t):
    rng = np.random.default_rng(700 + k)
    start = rng.uniform((8.0, -40.0), (60.0, 40.0), (48, 2))
    vel = rng.uniform(-1.0, 1.0, (48, 2))
    out = []
    for t in range(n_t):
        seen = np.sort(rng.choice(48, int(rng.integers(30, 49)), replace=False))
        c = start[seen] + vel[seen] * 0.1 * t + rng.normal(0, 0.03, (len(seen), 2))
        junk = rng.uniform((-80.0, -60.0), (-30.0, 60.0), (int(rng.integers(0, 17)), 2))
        out.append(boxes_at(np.concatenate([c, junk])))
    return out


LAT = np.stack(np.meshgrid(np.arange(32) * 8.0 - 124.0, np.arange(32) * 8.0 - 124.0, indexing="ij"), -1).reshape(-1, 2)
OFF = -0.63035 - np.pi / 2


def stress_lists(k, n_t):
    rng = np.random.default_rng(900 + k)
    return [boxes_at(LAT[np.sort(rng.choice(len(LAT), 256, replace=False))] + rng.normal(0, 0.15, (256, 2))) for _ in range(n_t)]


def stress_state():
    """the mature 1024-track table: frame 1 spawns, then every lattice site is observed until the tracks are mature"""
    rng = np.random.default_rng(0)
    c = lmot.Lmot()
    t = 0.0
    for _ in range(8):
        t += 1e5
        c.track_step(boxes_at(LAT + rng.normal(0, 0.02, LAT.shape)), t)
    st = c.tracker_dump()
    c.close()
    return st, t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warm", type=int, default=10)
    ap.add_argument("--sizes", default="1,2,4,8")
    ap.add_argument("--workloads", default="bench,stress")
    ap.add_argument("--burst", type=int, default=8)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("seq_track_measure.py: no CUDA device")
    card = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:                  # the numbers below still stand, without the power limit
        pl = f"unavailable ({type(ex).__name__})"

    STATE, TS_STATE = stress_state()

    print(f"card: {card}; power limit, max SM clock: {pl}")
    print(f"{a.ticks} timed ticks after {a.warm} warm-up ticks, {a.rounds} rounds alternating the arms")
    sizes = [int(s) for s in a.sizes.split(",")]
    S_MAX = max(sizes)
    n_t = a.warm + a.ticks
    table = []
    for wl in a.workloads.split(","):
        burst = a.ticks if wl == "bench" else a.burst
        if wl == "bench":
            ts = lambda k, t: 1.0e6 * (k + 1) + 1.0e5 * t                # own start stamp per stream
            ego = lambda k, t: (2.0 + k, 0.01 * (k - 3) * t)             # own ego speed and yaw per stream
        else:
            ts = lambda k, t: TS_STATE + 1.0e5 * ((t - a.warm) % burst + 1 if t >= a.warm else t + 1)   # each burst restarts at the table
            ego = lambda k, t: (0.0, 0.0)
        lists = [bench_lists(k, n_t) if wl == "bench" else stress_lists(k, n_t) for k in range(S_MAX)]
        cap = max(len(b) for l in lists for b in l)
        pad = np.zeros((n_t, S_MAX, cap, 8, 3), np.float32)
        cnt = np.zeros((n_t, S_MAX), np.int32)
        for k in range(S_MAX):
            for t in range(n_t):
                pad[t, k, : len(lists[k][t])] = lists[k][t]
                cnt[t, k] = len(lists[k][t])
        d_pad, d_cnt = torch.from_numpy(pad).cuda(), torch.from_numpy(cnt).cuda()
        torch.cuda.synchronize()
        lp = lambda t, k: d_pad[t, k].data_ptr()
        cp = lambda t, k: d_cnt[t, k:].data_ptr()
        for S in sizes:
            ctxs = []
            for k in range(S):
                c = lmot.Lmot()
                st = torch.cuda.Stream()
                c.set_stream(st.cuda_stream)
                ctxs.append(c)
            seq = lmot.Lmot()
            seq_stream = torch.cuda.Stream()
            seq.set_stream(seq_stream.cuda_stream)
            scal = [[lmot.Lmot.seq_scalars(S, [f(k, t) for k in range(S)]) for f in (ts, lambda k, t: ego(k, t)[0], lambda k, t: ego(k, t)[1])]
                    for t in range(n_t)]

            def run_a(t0, t1):
                for t in range(t0, t1):
                    for k in range(S):
                        ctxs[k].track_step_lists_dev(lp(t, k), cp(t, k), 1, cap, ts(k, t), *ego(k, t))

            def run_b(t0, t1):
                for t in range(t0, t1):
                    seq.seq_track_dev(lp(t, 0), cp(t, 0), cap, *scal[t])

            rates = {"A contexts": [], "B seq": []}
            def start(arm):
                """each arm's tables at the start of a burst: empty (bench) or the 1024-track table (stress)"""
                if arm.startswith("A"):
                    for c in ctxs:
                        c.tracker_reset() if wl == "bench" else c.tracker_load(STATE, 1, TS_STATE, 0.0, OFF, OFF, -np.pi / 2)
                else:
                    if wl == "bench":
                        seq.seq_open(S, ring=8)
                    else:
                        for k in range(S):
                            seq.seq_tracker_load(k, STATE, 1, TS_STATE, 0.0, OFF, OFF, -np.pi / 2)

            seq.seq_open(S, ring=8)
            for rnd in range(a.rounds):
                for arm in rates:
                    run = run_a if arm.startswith("A") else run_b
                    start(arm)
                    run(0, a.warm)
                    el = 0.0
                    for b0 in range(a.warm, n_t, burst):
                        if b0 > a.warm or wl != "bench":
                            start(arm)
                        torch.cuda.synchronize()
                        h0 = time.perf_counter()
                        run(b0, min(b0 + burst, n_t))
                        torch.cuda.synchronize()
                        el += time.perf_counter() - h0
                    rates[arm].append(S * a.ticks / el)
                for k in range(S):
                    da, db = ctxs[k].tracker_dump(), seq.seq_tracker_dump(k)
                    if da.shape != db.shape or not np.array_equal(da.view(np.uint64), db.view(np.uint64)):
                        raise SystemExit(f"{wl} S={S} round {rnd}: sequence {k} differs from its context ({da.shape} vs {db.shape} rows)")
            live = [int((ctxs[k].tracker_dump()[:, 0] > 0).sum()) for k in range(S)]
            print(f"{wl} S={S}: final tables equal in every round (live tracks {live})")
            row = [wl, S]
            for arm, v in rates.items():
                v = np.array(v)
                row.append((np.median(v), v.min(), v.max()))
                print(f"{wl} S={S} {arm:10s} steps/s median {np.median(v):9.1f}  min {v.min():9.1f}  max {v.max():9.1f}")
            table.append(row)
            for c in ctxs:
                c.set_stream(None)
                c.close()
            seq.set_stream(None)
            seq.close()

    print()
    print("| workload | S | A: S contexts, steps/s median (min-max) | B: one context, seq_track_dev, steps/s median (min-max) | B / A |")
    print("|---|---|---|---|---|")
    for wl, S, ra, rb in table:
        print(f"| {wl} | {S} | {ra[0]:.0f} ({ra[1]:.0f}-{ra[2]:.0f}) | {rb[0]:.0f} ({rb[1]:.0f}-{rb[2]:.0f}) | {rb[0] / ra[0]:.2f} |")


if __name__ == "__main__":
    main()
