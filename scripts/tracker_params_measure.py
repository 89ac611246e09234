"""Tunable tracker parameters on one GPU (DESIGN.md §6c).  Two arms, each alternated round by round after a warm-up:

  arm 1  cost of the tuned kernels.  One context, pipelined lmot_track_step_lists_dev (one list per step), on the bench and stress
         workloads of seq_track_measure.py: the defaults (the default kernels) against a no-op tuned set (distance_thres = 1e9, the
         tuned kernels with the same results).  The final tables of the two must be equal.
  arm 2  a parameter sweep: eight parameter sets over one box stream (the bench workload's stream 0).
           A  8 contexts, each with its set, on their own streams, lmot_track_step_lists_dev
           B  one context, 8 sequences with the 8 sets, lmot_seq_track_dev (one tracker chain per tick)
         The final table of sequence k must equal context k's.

Steps/s = tables x steps / host time around the timed steps, bracketed by device synchronisations (stress: summed over bursts that
each start from the same 1024-track table, as in seq_track_measure.py).  Prints the card name, power limit and max SM clock beside
the numbers.  Needs a CUDA device; there is no CPU path.

    python scripts/tracker_params_measure.py [--ticks 200] [--rounds 3] [--warm 10]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from seq_track_measure import OFF, bench_lists, lmot, stress_lists, stress_state  # noqa: E402

NOOP = dict(distance_thres=1e9)
SWEEP = [                                   # arm 2: the defaults, the reference's commented alternatives, and single-field moves
    {},
    dict(gamma_g=5.99, p_g=0.95),                                                       # imm_ukf_jpda.cpp:31-32
    dict(gamma_g=15.22),                                                                # :33
    dict(distance_thres=1.0, lifetime_thres=8),                                         # :39, :42
    dict(std_a=[0.8, 0.8, 5.0], std_yawdd=[0.8, 0.8, 3.0]),                             # ukf.cpp:53-58
    dict(std_a=[3.0, 3.0, 3.0], std_yawdd=[3.0, 3.0, 3.0]),                             # :75-80
    dict(std_las_x=0.3, std_las_y=0.3),                                                 # :92, :95
    dict(trans=[[0.8, 0.1, 0.1], [0.8, 0.1, 0.1], [0.1, 0.1, 0.8]], p0_diag=[0.5, 0.5, 1.0, 1.0, 1.0]),   # :156-166, :263-267
]


def pad_device(lists_per_step):
    """[t][k] box arrays -> device (T, K, cap, 8, 3) and counts (T, K)"""
    n_t, K = len(lists_per_step), len(lists_per_step[0])
    cap = max(len(b) for row in lists_per_step for b in row)
    pad = np.zeros((n_t, K, cap, 8, 3), np.float32)
    cnt = np.zeros((n_t, K), np.int32)
    for t, row in enumerate(lists_per_step):
        for k, b in enumerate(row):
            pad[t, k, : len(b)] = b
            cnt[t, k] = len(b)
    d_pad, d_cnt = torch.from_numpy(pad).cuda(), torch.from_numpy(cnt).cuda()
    torch.cuda.synchronize()
    return d_pad, d_cnt, cap


def timed(run, start, warm, n_t, burst):
    """warm-up steps, then the timed steps in bursts (each burst starts with start()); -> seconds"""
    start()
    run(0, warm)
    el = 0.0
    for b0 in range(warm, n_t, burst):
        if b0 > warm or burst < n_t - warm:
            start()
        torch.cuda.synchronize()
        h0 = time.perf_counter()
        run(b0, min(b0 + burst, n_t))
        torch.cuda.synchronize()
        el += time.perf_counter() - h0
    return el


def stats(v):
    v = np.array(v)
    return np.median(v), v.min(), v.max()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warm", type=int, default=10)
    ap.add_argument("--burst", type=int, default=8)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tracker_params_measure.py: no CUDA device")
    card = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:                  # the numbers below still stand, without the power limit
        pl = f"unavailable ({type(ex).__name__})"
    print(f"card: {card}; power limit, max SM clock: {pl}")
    print(f"{a.ticks} timed steps after {a.warm} warm-up steps, {a.rounds} rounds alternating the arms")
    n_t = a.warm + a.ticks
    STATE, TS_STATE = stress_state()
    rows = []

    # ---- arm 1: defaults against a no-op tuned set, one context
    for wl in ("bench", "stress"):
        burst = a.ticks if wl == "bench" else a.burst
        lists = bench_lists(0, n_t) if wl == "bench" else stress_lists(0, n_t)
        d_pad, d_cnt, cap = pad_device([[b] for b in lists])
        if wl == "bench":
            ts = lambda t: 1.0e6 + 1.0e5 * t
            ego = lambda t: (2.0, -0.03 * t)
        else:
            ts = lambda t: TS_STATE + 1.0e5 * ((t - a.warm) % burst + 1 if t >= a.warm else t + 1)
            ego = lambda t: (0.0, 0.0)
        ctxs = {"default": lmot.Lmot(), "no-op tuned": lmot.Lmot()}
        ctxs["no-op tuned"].set_tracker_params(**NOOP)
        streams = []
        for c in ctxs.values():
            streams.append(torch.cuda.Stream())
            c.set_stream(streams[-1].cuda_stream)
        rates = {k: [] for k in ctxs}
        for rnd in range(a.rounds):
            for arm, c in ctxs.items():
                def run(t0, t1, c=c):
                    for t in range(t0, t1):
                        c.track_step_lists_dev(d_pad[t, 0].data_ptr(), d_cnt[t, 0:].data_ptr(), 1, cap, ts(t), *ego(t))

                def start(c=c):
                    c.tracker_reset() if wl == "bench" else c.tracker_load(STATE, 1, TS_STATE, 0.0, OFF, OFF, -np.pi / 2)
                rates[arm].append(a.ticks / timed(run, start, a.warm, n_t, burst))
            da, db = (c.tracker_dump() for c in ctxs.values())
            if da.shape != db.shape or not np.array_equal(da.view(np.uint64), db.view(np.uint64)):
                raise SystemExit(f"arm 1 {wl} round {rnd}: the no-op tuned table differs from the default one")
        print(f"arm 1 {wl}: final tables of the two arms equal in every round ({int((da[:, 0] > 0).sum())} live tracks)")
        for arm, v in rates.items():
            m, lo, hi = stats(v)
            print(f"arm 1 {wl} {arm:12s} steps/s median {m:9.1f}  min {lo:9.1f}  max {hi:9.1f}")
            rows.append(("1", wl, arm, m, lo, hi))
        for c in ctxs.values():
            c.set_stream(None)
            c.close()

    # ---- arm 2: eight parameter sets over one box stream
    S = len(SWEEP)
    lists = bench_lists(0, n_t)
    d_pad, d_cnt, cap = pad_device([[b] * S for b in lists])
    ts = lambda t: 1.0e6 + 1.0e5 * t
    ctxs, streams = [], []
    for k in range(S):
        c = lmot.Lmot()
        if SWEEP[k]:
            c.set_tracker_params(**SWEEP[k])
        streams.append(torch.cuda.Stream())
        c.set_stream(streams[-1].cuda_stream)
        ctxs.append(c)
    seq = lmot.Lmot()
    seq_stream = torch.cuda.Stream()
    seq.set_stream(seq_stream.cuda_stream)
    scal = [[lmot.Lmot.seq_scalars(S, v) for v in (ts(t), 2.0, -0.03 * t)] for t in range(n_t)]

    def run_a(t0, t1):
        for t in range(t0, t1):
            for k in range(S):
                ctxs[k].track_step_lists_dev(d_pad[t, k].data_ptr(), d_cnt[t, k:].data_ptr(), 1, cap, ts(t), 2.0, -0.03 * t)

    def start_a():
        for c in ctxs:
            c.tracker_reset()

    def run_b(t0, t1):
        for t in range(t0, t1):
            seq.seq_track_dev(d_pad[t, 0].data_ptr(), d_cnt[t, 0:].data_ptr(), cap, *scal[t])

    def start_b():
        seq.seq_open(S, ring=8)
        for k in range(S):
            if SWEEP[k]:
                seq.seq_set_tracker_params(k, **SWEEP[k])

    rates = {"A 8 contexts": [], "B 8 sequences": []}
    for rnd in range(a.rounds):
        rates["A 8 contexts"].append(S * a.ticks / timed(run_a, start_a, a.warm, n_t, a.ticks))
        rates["B 8 sequences"].append(S * a.ticks / timed(run_b, start_b, a.warm, n_t, a.ticks))
        for k in range(S):
            da, db = ctxs[k].tracker_dump(), seq.seq_tracker_dump(k)
            if da.shape != db.shape or not np.array_equal(da.view(np.uint64), db.view(np.uint64)):
                raise SystemExit(f"arm 2 round {rnd}: sequence {k} differs from its context")
    live = [int((seq.seq_tracker_dump(k)[:, 0] > 0).sum()) for k in range(S)]
    print(f"arm 2: final tables of A and B equal in every round (live tracks per set {live})")
    for arm, v in rates.items():
        m, lo, hi = stats(v)
        print(f"arm 2 {arm:14s} steps/s median {m:9.1f}  min {lo:9.1f}  max {hi:9.1f}")
        rows.append(("2", "bench x 8 sets", arm, m, lo, hi))
    for c in ctxs:
        c.set_stream(None)
        c.close()
    seq.set_stream(None)
    seq.close()

    print()
    print("| arm | workload | configuration | steps/s median (min-max) |")
    print("|---|---|---|---|")
    for arm, wl, name, m, lo, hi in rows:
        print(f"| {arm} | {wl} | {name} | {m:.0f} ({lo:.0f}-{hi:.0f}) |")


if __name__ == "__main__":
    main()
