#!/usr/bin/env python3
"""Sequence ticks on each stream's own clock (lmot_seq_tick_dev): what a subset or mixed tick costs next to today's alternatives.

Three comparisons, each timed over device data with a host clock around work that ends in a result wait (seq_fetch waits for the last
tick, which is published after every earlier one).  The arms alternate round by round, and after every round the arms' final tables are
compared bit for bit (a timing of different work is not a comparison).

  (a) no regression: an 8-sequence all-frames tick through lmot_seq_tick_dev against lmot_seq_dev (the same launches);
  (b) a two-rate fleet, 4 sequences at 20 Hz and 4 at 10 Hz over 2 s of stream time: one set with subset ticks against today's
      alternative, one context with one set per rate;
  (c) a mixed tick, 4 sequences from frames + 4 from box lists, against an 8-frames tick.

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
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def params():
    p = pkg.default_params()
    p.max_points = 1 << 17
    p.max_tracks = 2048
    return p


def boxes_of(rng, n):
    from test_seq_track_gpu import boxes_at
    return boxes_at(rng.uniform((8.0, -30.0), (40.0, 30.0), (n, 2)))


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=40, help="ticks per round in (a) and (c); (b) is 2 s of stream time at 20 Hz")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    T = args.ticks
    cfgs = [synth.SceneConfig(seed=300 + k, n_objects=30, rings=64, azimuths=1800) for k in range(8)]
    host = [[p for _, p in synth.frames(c, max(T, 40))] for c in cfgs]
    dev = [[torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in fr] for fr in host]
    rng = np.random.default_rng(1)
    lists = [[boxes_of(rng, 20 + k) for _ in range(max(T, 40))] for k in range(8)]
    dl = [[torch.from_numpy(b).cuda() for b in ls] for ls in lists]
    dn = [[torch.tensor([len(b)], dtype=torch.int32).cuda() for b in ls] for ls in lists]
    torch.cuda.synchronize()
    ts = lambda k, t: 1.0e6 * (1 + k) + 50000.0 * t
    fr = lambda k, t: (dev[k][t].data_ptr(), len(host[k][t]))
    li = lambda k, t: dict(lists=[dl[k][t].data_ptr()], d_counts=dn[k][t].data_ptr(), cap=len(lists[k][t]), timestamp=ts(k, t))
    info = card()

    def opened(S):
        c = pkg.Lmot(params())
        c.seq_open(S, ring=8)
        return c

    def timed(run):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run()
        return time.perf_counter() - t0

    def same_tables(pairs):
        for (ca, ka), (cb, kb) in pairs:
            a, b = ca.seq_tracker_dump(ka), cb.seq_tracker_dump(kb)
            assert a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64)), (ka, kb)

    def report(name, arms, unit_ticks):
        out = {"comparison": name, "gpu": info, "rounds": args.rounds}
        for arm, xs in arms.items():
            ms = np.array(xs) * 1e3
            out[arm] = {"ms_per_round_median": round(float(np.median(ms)), 3), "min": round(float(ms.min()), 3), "max": round(float(ms.max()), 3),
                        "us_per_tick_median": round(float(np.median(ms)) * 1e3 / unit_ticks, 1)}
        print(json.dumps(out), flush=True)

    # (a) all-frames tick: lmot_seq_tick_dev against lmot_seq_dev
    arms = {"seq_dev": [], "seq_tick_dev": []}
    for r in range(args.rounds + 1):
        a, b = opened(8), opened(8)
        run_a = lambda: [a.seq_dev([fr(k, t) for k in range(8)], [ts(k, t) for k in range(8)]) for t in range(T)] and a.seq_fetch()
        run_b = lambda: [b.seq_tick_dev([dict(frames=fr(k, t), timestamp=ts(k, t)) for k in range(8)]) for t in range(T)] and b.seq_fetch()
        order = [("seq_dev", run_a), ("seq_tick_dev", run_b)] if r % 2 else [("seq_tick_dev", run_b), ("seq_dev", run_a)]
        for arm, run in order:
            dt = timed(run)
            if r:                                   # round 0 warms every shape up
                arms[arm].append(dt)
        same_tables([((a, k), (b, k)) for k in range(8)])
        a.close(); b.close()
    report("a_all_frames_tick", arms, T)

    # (b) two-rate fleet over 2 s: sequences 0-3 at 20 Hz (every tick), 4-7 at 10 Hz (even ticks)
    N = 40
    arms = {"one_set_subset_ticks": [], "one_context_per_rate": []}
    for r in range(args.rounds + 1):
        one = opened(8)
        fast, slow = opened(4), opened(4)

        def run_one():
            for t in range(N):
                one.seq_tick_dev([dict(frames=fr(k, t), timestamp=ts(k, t)) if k < 4 or t % 2 == 0 else None for k in range(8)])
            one.seq_fetch()

        def run_two():
            for t in range(N):
                fast.seq_dev([fr(k, t) for k in range(4)], [ts(k, t) for k in range(4)])
                if t % 2 == 0:
                    slow.seq_dev([fr(k, t) for k in range(4, 8)], [ts(k, t) for k in range(4, 8)])
            fast.seq_fetch(); slow.seq_fetch()

        order = [("one_set_subset_ticks", run_one), ("one_context_per_rate", run_two)]
        for arm, run in (order if r % 2 else order[::-1]):
            dt = timed(run)
            if r:
                arms[arm].append(dt)
        same_tables([((one, k), (fast, k)) for k in range(4)] + [((one, k), (slow, k - 4)) for k in range(4, 8)])
        one.close(); fast.close(); slow.close()
    report("b_two_rate_fleet_2s", arms, N)

    # (c) a mixed tick (sequences 0-3 frames, 4-7 box lists) against an 8-frames tick
    arms = {"frames_8": [], "frames_4_lists_4": []}
    for r in range(args.rounds + 1):
        a, b, ref = opened(8), opened(8), opened(8)
        run_a = lambda: [a.seq_tick_dev([dict(frames=fr(k, t), timestamp=ts(k, t)) for k in range(8)]) for t in range(T)] and a.seq_fetch()
        run_b = lambda: [b.seq_tick_dev([dict(frames=fr(k, t), timestamp=ts(k, t)) if k < 4 else li(k, t) for k in range(8)])
                         for t in range(T)] and b.seq_fetch()
        order = [("frames_8", run_a), ("frames_4_lists_4", run_b)]
        for arm, run in (order if r % 2 else order[::-1]):
            dt = timed(run)
            if r:
                arms[arm].append(dt)
        for t in range(T):              # the mixed tick's tables against the same steps as separate all-frames / all-lists ticks
            ref.seq_tick_dev([dict(frames=fr(k, t), timestamp=ts(k, t)) if k < 4 else None for k in range(8)])
            ref.seq_tick_dev([li(k, t) if k >= 4 else None for k in range(8)])
        ref.seq_fetch()
        same_tables([((a, k), (ref, k)) for k in range(4)] + [((b, k), (ref, k)) for k in range(8)])
        a.close(); b.close(); ref.close()
    report("c_mixed_tick", arms, T)


if __name__ == "__main__":
    main()
