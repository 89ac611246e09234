"""Track prediction (lmot_predict_tracks*): what one prediction costs and what predicting after every step costs the tracker chain.
Prints the card name and power limit beside the numbers.  Needs a CUDA device; there is no CPU path.
  (a) call   us per lmot_predict_tracks_dev call (CUDA events over back-to-back calls on the context's stream) for a 64-row table, the
             1,024-track stress table, and an 8,192-row append-only table (the bench table padded with dead rows), at n_t = 1, 8, 32
  (b) chain  bench-workload steps/s through lmot_track_step_lists_dev, without and with an n_t = 8 prediction after every step;
             the two arms alternate, --rounds rounds
  (c) seq    S = 8 tracking-only sequence ticks (lmot_seq_track_dev), without and with one lmot_seq_predict_tracks_dev per tick

    python scripts/predict_measure.py [--steps 2000] [--rounds 3] [--calls 200]
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
from seq_track_measure import OFF, bench_lists, stress_state   # noqa: E402


def padded(lists):
    cap = max(1, max(len(b) for b in lists))
    pad = np.zeros((len(lists), cap, 8, 3), np.float32)
    for t, b in enumerate(lists):
        pad[t, : len(b)] = b
    cnt = np.array([len(b) for b in lists], np.int32)
    return torch.from_numpy(pad).cuda(), torch.from_numpy(cnt).cuda(), cap


class DevOut:
    """device outputs of n_t times x cap rows"""

    def __init__(self, n_t, cap):
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device="cuda")
        self.t = [z(cap, torch.int64), z(cap, torch.int32), z((n_t, cap), torch.uint8), z((n_t, cap, 5), torch.float64),
                  z((n_t, cap, 25), torch.float64), z((n_t, cap, 3), torch.float64), z((n_t, cap, 2), torch.float64), z((n_t, cap, 4), torch.float64)]
        names = ("ids", "track_manage", "flags", "x", "P", "mode_prob", "gate_z", "gate_S")
        self.out = lmot.pred_out(cap, {k: v.data_ptr() for k, v in zip(names, self.t)})


def ctx(max_tracks=8192):
    p = lmot.default_params()
    p.max_tracks = max_tracks
    c = lmot.Lmot(p)
    st = torch.cuda.Stream()
    c.set_stream(st.cuda_stream)
    return c, st


def call_us(c, st, ts, n_t, cap, calls):
    o = DevOut(n_t, cap)
    times = [ts + 1e5 * (j + 1) for j in range(n_t)]
    torch.cuda.synchronize()
    for _ in range(10):
        c.predict_tracks_dev(times, o.out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(st)
    for _ in range(calls):
        c.predict_tracks_dev(times, o.out)
    e1.record(st)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("predict_measure.py: no CUDA device")
    card = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:
        pl = f"unavailable ({type(ex).__name__})"
    print(f"card: {card}; power limit, max SM clock: {pl}")

    # ---- (a) one call
    probe = lmot.Lmot()
    for t, b in enumerate(bench_lists(0, 200)):
        probe.track_step(b, 1.0e6 + 1.0e5 * t, 2.0, 0.001 * t)
    bench_tab = probe.tracker_dump()
    probe.close()
    live = bench_tab[bench_tab[:, 0] > 0]
    small = np.concatenate([live] * (64 // len(live) + 1))[:64]
    dead = np.repeat(bench_tab[:1], 8192 - len(bench_tab), 0)
    dead[:, 0] = 0
    stress, sts = stress_state()
    tables = [("64 live rows", small, 1e6), ("1,024-track stress table", stress, sts),
              (f"8,192 rows append-only ({int((bench_tab[:, 0] > 0).sum())} live)", np.concatenate([bench_tab, dead]), 1e6)]
    print("(a) us per lmot_predict_tracks_dev call")
    for name, tab, ts in tables:
        c, st = ctx()
        c.tracker_load(tab, 1, ts, 0.0, OFF, OFF, -np.pi / 2)
        row = [f"n_t={n_t}: {call_us(c, st, ts, n_t, len(tab), a.calls):8.1f}" for n_t in (1, 8, 32)]
        print(f"  {name:40s} " + "  ".join(row))
        c.close()

    # ---- (b) the chain
    lists = bench_lists(0, a.steps)
    d, n, cap = padded(lists)
    res = {"plain": [], "predict n_t=8": []}
    for r in range(a.rounds):
        for arm in res:
            c, st = ctx()
            o = DevOut(8, 8192)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for t in range(a.steps):
                ts = 1.0e6 + 1.0e5 * t
                c.track_step_lists_dev(d[t].data_ptr(), n[t:].data_ptr(), 1, cap, ts, 2.0, 0.001 * t)
                if arm != "plain":
                    c.predict_tracks_dev([ts + 2.5e4 * (j + 1) for j in range(8)], o.out)
                if t % 4 == 3:
                    c.frame_fetch(want_boxes=False)
            torch.cuda.synchronize()
            res[arm].append(a.steps / (time.perf_counter() - t0))
            c.close()
    print(f"(b) bench steps/s through lmot_track_step_lists_dev, {a.steps} steps, {a.rounds} rounds alternating")
    for arm, v in res.items():
        print(f"  {arm:16s} " + " ".join(f"{x:8.0f}" for x in v) + f"   median {np.median(v):8.0f}")
    p, q = np.median(res["plain"]), np.median(res["predict n_t=8"])
    print(f"  chain cost per predicted step: {1e6 / q - 1e6 / p:.1f} us")

    # ---- (c) sequences
    S, ticks = 8, max(200, a.steps // 4)
    per = [bench_lists(k, ticks) for k in range(S)]
    cap = max(1, max(len(b) for lst in per for b in lst))
    pad = np.zeros((ticks, S, cap, 8, 3), np.float32)
    cnt = np.zeros((ticks, S), np.int32)
    for k in range(S):
        for t, b in enumerate(per[k]):
            pad[t, k, : len(b)] = b
            cnt[t, k] = len(b)
    dp, dc = torch.from_numpy(pad).cuda(), torch.from_numpy(cnt).cuda()
    res = {"plain": [], "predict n_t=8": []}
    for r in range(a.rounds):
        for arm in res:
            c, st = ctx(2048)
            c.seq_open(S, ring=8)
            outs = [DevOut(8, 2048) for _ in range(S)]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for t in range(ticks):
                ts = [1.0e6 + 1.0e5 * t] * S
                c.seq_track_dev(dp[t].data_ptr(), dc[t].data_ptr(), cap, ts, [2.0] * S, [0.001 * t] * S)
                if arm != "plain":
                    c.seq_predict_tracks_dev([[x + 2.5e4 * (j + 1) for j in range(8)] for x in ts], [o.out for o in outs])
                if t % 4 == 3:
                    c.seq_fetch()
            torch.cuda.synchronize()
            res[arm].append(ticks / (time.perf_counter() - t0))
            c.close()
    print(f"(c) S = {S} sequence ticks/s (lmot_seq_track_dev), {ticks} ticks, {a.rounds} rounds alternating")
    for arm, v in res.items():
        print(f"  {arm:16s} " + " ".join(f"{x:8.0f}" for x in v) + f"   median {np.median(v):8.0f}")


if __name__ == "__main__":
    main()
