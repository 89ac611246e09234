"""Track retirement (lmot_set_track_retirement): what it buys on a long stream and what the retire phase costs on the tracker chain.
Arms alternated round by round (off, on), box lists resident on the device, steps/s from the host clock between device
synchronisations.  Prints the card name and power limit beside the numbers.  Needs a CUDA device; there is no CPU path.
  (a) long   one context, --long steps of the bench workload (scripts/seq_track_measure.py), default max_tracks: steps/s per
             1,000-step window, the table's rows at the end of each window, and the step at which the table without retirement fills
  (b) chain  the bench workload from an empty table (--steps steps), and the stress table (1,024 mature tracks, 256 boxes per step,
             bursts of 8 steps from the loaded table: most tracks die and hundreds of records move per step)
  (c) seq    S = 8 tracking-only sequence ticks (lmot_seq_track_dev) of the bench workload, every sequence off / on

    python scripts/retire_measure.py [--long 20000] [--steps 2000] [--rounds 3]
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))
lmot = importlib.import_module("3d-lidar-multi-object-tracking_b200")
from seq_track_measure import OFF, bench_lists, stress_lists, stress_state   # noqa: E402


def padded(lists):
    cap = max(1, max(len(b) for b in lists))
    pad = np.zeros((len(lists), cap, 8, 3), np.float32)
    for t, b in enumerate(lists):
        pad[t, : len(b)] = b
    cnt = np.array([len(b) for b in lists], np.int32)
    return torch.from_numpy(pad).cuda(), torch.from_numpy(cnt).cuda(), cap


def ctx(retire):
    c = lmot.Lmot()
    st = torch.cuda.Stream()
    c.set_stream(st.cuda_stream)
    c.set_track_retirement(retire)
    return c


def step(c, d, n, cap, t, ts):
    c.track_step_lists_dev(d[t].data_ptr(), n[t:].data_ptr(), 1, cap, ts, 2.0, 0.001 * t)


def first_full_step(lists):
    """the step whose spawns first exceed the table without retirement (LMOT_WARN_TRACK_TABLE_FULL), stepped synchronously"""
    c = lmot.Lmot()
    try:
        for t, b in enumerate(lists):
            c.track_step(b, 1.0e6 + 1.0e5 * t, 2.0, 0.001 * t)
            if c.last_warning == lmot.WARN_TRACK_TABLE_FULL:
                return t
        return None
    finally:
        c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--long", type=int, default=20000)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window", type=int, default=1000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("retire_measure.py: no CUDA device")
    card = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:
        pl = f"unavailable ({type(ex).__name__})"
    print(f"card: {card}; power limit, max SM clock: {pl}; {a.rounds} rounds alternating off / on")

    # ---- (a) the long run
    lists = bench_lists(0, a.long)
    d, n, cap = padded(lists)
    full_at = first_full_step(lists)
    W = a.long // a.window
    rates = {False: np.zeros((a.rounds, W)), True: np.zeros((a.rounds, W))}
    rows = {False: [], True: []}
    for r in range(a.rounds):
        for arm in (False, True):
            c = ctx(arm)
            for w in range(W):
                torch.cuda.synchronize()
                h0 = time.perf_counter()
                for t in range(w * a.window, (w + 1) * a.window):
                    step(c, d, n, cap, t, 1.0e6 + 1.0e5 * t)
                torch.cuda.synchronize()
                rates[arm][r, w] = a.window / (time.perf_counter() - h0)
                if r == 0:
                    rows[arm].append(c.tracker_num_tracks())
            c.set_stream(None)
            c.close()
    print(f"\n(a) bench workload, {a.long} steps, max_tracks {lmot.default_params().max_tracks}: without retirement the table is full "
          f"from step {full_at} on (LMOT_WARN_TRACK_TABLE_FULL: no new track after that)")
    print("| steps | off: steps/s median (min-max) | off: rows | on: steps/s median (min-max) | on: rows |")
    print("|---|---|---|---|---|")
    for w in range(W):
        o, i = rates[False][:, w], rates[True][:, w]
        print(f"| {w * a.window}-{(w + 1) * a.window} | {np.median(o):.0f} ({o.min():.0f}-{o.max():.0f}) | {rows[False][w]} | "
              f"{np.median(i):.0f} ({i.min():.0f}-{i.max():.0f}) | {rows[True][w]} |")
    del d, n

    # ---- (b) the retire phase on the chain
    print("\n(b) one context, steps/s median (min-max)")
    lists = bench_lists(1, a.steps)
    d, n, cap = padded(lists)
    state, ts_state = stress_state()
    sl = stress_lists(0, a.steps)
    sd, sn, scap = padded(sl)
    res = {("bench", False): [], ("bench", True): [], ("stress", False): [], ("stress", True): []}
    for r in range(a.rounds):
        for arm in (False, True):
            c = ctx(arm)
            torch.cuda.synchronize()
            h0 = time.perf_counter()
            for t in range(a.steps):
                step(c, d, n, cap, t, 1.0e6 + 1.0e5 * t)
            torch.cuda.synchronize()
            res[("bench", arm)].append(a.steps / (time.perf_counter() - h0))
            el = 0.0
            for b0 in range(0, a.steps, 8):
                c.tracker_load(state, 1, ts_state, 0.0, OFF, OFF, -np.pi / 2)
                torch.cuda.synchronize()
                h0 = time.perf_counter()
                for t in range(b0, b0 + 8):
                    sd_t = t % len(sl)
                    c.track_step_lists_dev(sd[sd_t].data_ptr(), sn[sd_t:].data_ptr(), 1, scap, ts_state + 1.0e5 * (t - b0 + 1), 0.0, 0.0)
                torch.cuda.synchronize()
                el += time.perf_counter() - h0
            res[("stress", arm)].append(a.steps / el)
            c.set_stream(None)
            c.close()
    print("| workload | off | on | on / off |")
    print("|---|---|---|---|")
    for wl in ("bench", "stress"):
        o, i = np.array(res[(wl, False)]), np.array(res[(wl, True)])
        print(f"| {wl} | {np.median(o):.0f} ({o.min():.0f}-{o.max():.0f}) | {np.median(i):.0f} ({i.min():.0f}-{i.max():.0f}) | "
              f"{np.median(i) / np.median(o):.3f} |")
    del d, n, sd, sn

    # ---- (c) S = 8 sequence ticks
    S, n_t = 8, a.steps
    lists = [bench_lists(k, n_t) for k in range(S)]
    cap = max(len(b) for l in lists for b in l)
    pad = np.zeros((n_t, S, cap, 8, 3), np.float32)
    cnt = np.zeros((n_t, S), np.int32)
    for k in range(S):
        for t in range(n_t):
            pad[t, k, : len(lists[k][t])] = lists[k][t]
            cnt[t, k] = len(lists[k][t])
    d, n = torch.from_numpy(pad).cuda(), torch.from_numpy(cnt).cuda()
    rs = {False: [], True: []}
    for r in range(a.rounds):
        for arm in (False, True):
            c = lmot.Lmot()
            st = torch.cuda.Stream()
            c.set_stream(st.cuda_stream)
            c.seq_open(S, ring=8)
            for k in range(S):
                c.seq_set_track_retirement(k, arm)
            torch.cuda.synchronize()
            h0 = time.perf_counter()
            for t in range(n_t):
                scal = [lmot.Lmot.seq_scalars(S, [f(k) for k in range(S)]) for f in
                        (lambda k: 1.0e6 * (k + 1) + 1.0e5 * t, lambda k: 2.0 + k, lambda k: 0.01 * (k - 3) * t)]
                c.seq_track_dev(d[t, 0].data_ptr(), n[t, 0:].data_ptr(), cap, *scal)
            torch.cuda.synchronize()
            rs[arm].append(S * n_t / (time.perf_counter() - h0))
            c.set_stream(None)
            c.close()
    o, i = np.array(rs[False]), np.array(rs[True])
    print(f"\n(c) S = 8 tracking-only sequence ticks, {n_t} ticks: steps/s off {np.median(o):.0f} ({o.min():.0f}-{o.max():.0f}), "
          f"on {np.median(i):.0f} ({i.min():.0f}-{i.max():.0f}), on / off {np.median(i) / np.median(o):.3f}")


if __name__ == "__main__":
    main()
