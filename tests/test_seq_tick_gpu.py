"""Sequence ticks on each stream's own clock (lmot_seq_tick*): any subset of the sequences steps, each from frames or box lists, and a
sequence may restart in place.

Contract (include/lmot.h): over any schedule, sequence k gives bit for bit what a separate context with the same lmot_params, tracker
parameters, retirement and detection parameters gives when it receives only sequence k's steps, in order -- FRAMES through lmot_frame
(lmot_set_sensors(table) + lmot_batch with a table), LISTS through lmot_track_step (lmot_track_step_lists_dev with a table).  A skipped
sequence is untouched and its output is not written.

Each docstring names the one-line breakage the test is meant to catch.  These breakages were reasoned out; none was injected and run.
"""
import ctypes as C

import numpy as np
import pytest

from test_seq_detect_params_gpu import SPARSE
from test_seq_rig_gpu import _RigSeq, _params, _table_kw
from test_seq_track_gpu import _ListSeq, _pad_lists
from test_sensor_rig_gpu import RIG, RIG_B

pytestmark = pytest.mark.gpu
f32 = np.float32
FIELDS = ("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb", "boxes")
N_TICKS = 40
TUNED = dict(gamma_g=7.5, std_a=(1.5, 2.5, 3.5), std_las_x=0.2)
LAYOUTS = {"S8": [None] * 8, "mixed": [RIG, RIG_B[1:2], None, RIG_B[2:4]]}


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8) if a.dtype.itemsize == 1 else a.view(f"u{a.dtype.itemsize}")


# ------------------------------------------------------------------------------------------------ data, schedule and twins
_DATA = {}


class _Data:
    """sequence k's frames (one per sensor of `rig`) and box lists (one per sensor) for every tick, on its own clock (50 ms per tick)
    and with its own ego motion (none for sequence 0, which the reference anchors)"""

    def __init__(self, synth, k, rig, n_ticks):
        key = (k, id(rig), n_ticks)
        if key not in _DATA:
            _DATA[key] = (_RigSeq(synth, k, rig, n_ticks=n_ticks).frames, _ListSeq(k, n_ticks, n_lists=len(rig) if rig else 1).lists)
        self.frames, self.lists = _DATA[key]
        self.k, self.rig = k, rig

    def ts(self, t):
        return 1.0e6 * (1 + self.k) + 777.0 * self.k + 50000.0 * t

    def ego(self, t):
        k = self.k
        return (1.5 * k + 0.05 * t, 0.3 + 0.01 * (k - 3) * t) if k else (0.0, 0.0)

    def entry(self, kind, t, restart=False):
        v, yaw = self.ego(t)
        d = dict(timestamp=self.ts(t), v_gps=v, yaw_gps=yaw, restart=restart)
        if kind == "F":
            d["frames"] = list(self.frames[t][: len(self.rig)]) if self.rig else self.frames[t][0]
        else:
            b = self.lists[t]
            d["lists"] = b if isinstance(b, list) or not self.rig else [b]
        return d


def _schedule(S, n_ticks, seed):
    """-> [tick][k] in (None, "F", "L"): sequences 2j at 20 Hz, 2j+1 at 10 Hz (every other tick), random drops; every sequence absent on
    at least 3 ticks, every tick with one present"""
    rng = np.random.default_rng(seed)
    sch = []
    for t in range(n_ticks):
        row = [None if (k % 2 and t % 2) or rng.random() < 0.15 else ("F" if rng.random() < 0.5 else "L") for k in range(S)]
        if all(x is None for x in row):
            row[0] = "F"
        sch.append(row)
    for k in range(0, S, 2):
        while sum(r[k] is None for r in sch) < 3:
            t = int(rng.integers(1, n_ticks))
            if sum(x is not None for x in sch[t]) > 1:
                sch[t][k] = None
    return sch


class _Twin:
    """the oracle of one sequence: a context with its table, tracker parameters, retirement and detection parameters.  step ->
    (status, result dict, per-frame counts, track IDs)"""

    def __init__(self, pkg, prm, rig=None, tuned=None, retire=False):
        self.pkg, self.ctx, self.rig = pkg, pkg.Lmot(prm), rig
        if rig:
            self.ctx.set_sensors(**_table_kw(rig))
        if tuned:
            self.ctx.set_tracker_params(**tuned)
        if retire:
            self.ctx.set_track_retirement(True)

    def step(self, d):
        c, pkg = self.ctx, self.pkg
        ts, v, yaw = C.c_double(d["timestamp"]), C.c_double(d["v_gps"]), C.c_double(d["yaw_gps"])
        if "frames" in d and self.rig:
            ptrs, ns, F, stride, keep = c._batch_args(d["frames"], False)
            bo, bufs = c._batch_out(c.params.max_tracks)
            st = c.lib.lmot_batch(c.h, ptrs, ns, F, stride, ts, v, yaw, C.byref(bo))
            r = c._batch_result(bo, bufs)
            counts = [tuple(int(r[key][i]) for key in ("n_elevated", "n_ground", "num_cluster", "n_boxes")) for i in range(F)]
            r.update({key: int(sum(r[key])) for key in ("n_elevated", "n_ground", "num_cluster")})
        elif "frames" in d:
            p, n, s = pkg._pts(d["frames"])
            fo, bufs = c._frame_out(c.params.max_tracks)
            st = c.lib.lmot_frame(c.h, pkg._fp(p), n, s, ts, v, yaw, C.byref(fo))
            r = c._frame_result(fo, bufs)
            counts = [(r["n_elevated"], r["n_ground"], r["num_cluster"], fo.n_boxes)]
        elif not self.rig:
            b = np.ascontiguousarray(d["lists"], f32).reshape(-1, 8, 3)
            to, bufs = c._track_out(c.params.max_tracks)
            st = c.lib.lmot_track_step(c.h, pkg._fp(b if len(b) else np.zeros((1, 8, 3), f32)), len(b), ts, v, yaw, C.byref(to))
            r = c._track_result(to, bufs)
            r.update(boxes=b, n_elevated=0, n_ground=0, num_cluster=0)
            counts = [(0, 0, 0, len(b))]
        else:
            import torch
            lists = d["lists"]
            dl, dn, cap = _pad_lists(lists)
            c.set_stream(None)
            c.lib.lmot_track_step_lists_dev(c.h, C.c_void_p(dl.data_ptr()), C.c_void_p(dn.data_ptr()), len(lists), int(cap), ts, v, yaw)
            fo, bufs = c._frame_out(c.params.max_tracks)
            torch.cuda.synchronize()
            st = c.lib.lmot_frame_fetch(c.h, C.byref(fo))
            r = c._frame_result(fo, bufs)
            counts = [(0, 0, 0, len(b)) for b in lists]
        return st, r, counts, _ids(c.track_ids)

    def close(self):
        self.ctx.close()


def _same(got, fc, want, what):
    _, w, wc, _ = want
    assert [tuple(int(x) for x in row) for row in fc] == [tuple(int(x) for x in row) for row in wc], (what, "frame counts")
    assert (got["n_elevated"], got["n_ground"], got["num_cluster"]) == (w["n_elevated"], w["n_ground"], w["num_cluster"]), what
    for key in FIELDS:
        assert got[key].shape == w[key].shape and np.array_equal(_bits(got[key]), _bits(w[key])), (what, key)


def _ids(fn, *k):
    """track IDs of the result most recently returned, None before the first"""
    try:
        return fn(*k)
    except RuntimeError as e:
        if getattr(e, "status", None) == -4:
            return None
        raise


def _same_ids(a, b, what):
    assert (a is None) == (b is None) and (a is None or np.array_equal(a, b)), (what, "ids")


def _status(wants):
    errs = [w[0] for w in wants if w[0] < 0]
    warns = [w[0] for w in wants if w[0] > 0]
    return errs[0] if errs else (warns[0] if warns else 0)


def _raw(ctx, fn, *args):
    """a raw seq call that returns per-sequence results: -> (status, results with None for skipped sequences)"""
    so, sets = ctx._seq_out(ctx.params.max_tracks)
    st = fn(ctx.h, *args, C.byref(so))
    return st, ctx._seq_tick_result(so, sets)


def _dev_entries(entries, keep):
    """host entries -> device entries: frames as (pointer, n) tuples, lists one tensor each with device lengths and capacity + 2"""
    import torch
    out = []
    for d in entries:
        if d is None:
            out.append(None)
            continue
        e = dict(d)
        if "frames" in d:
            fr = d["frames"]
            ts = [torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in (fr if isinstance(fr, list) else [fr])]
            keep.extend(ts)
            tup = [(t.data_ptr(), len(t)) for t in ts]
            e["frames"] = tup if isinstance(fr, list) else tup[0]
        else:
            ls = d["lists"] if isinstance(d["lists"], list) else [d["lists"]]
            cap = max(len(b) for b in ls) + 2
            ts = [torch.from_numpy(np.concatenate([b, np.zeros((cap - len(b), 8, 3), f32)])).cuda() for b in ls]
            n = torch.tensor([len(b) for b in ls], dtype=torch.int32).cuda()
            keep.extend(ts + [n])
            e.update(lists=[t.data_ptr() for t in ts], d_counts=n.data_ptr(), cap=cap)
        out.append(e)
    return out


# ------------------------------------------------------------------------------------------------ 1. schedules against twins
@pytest.mark.parametrize("layout,gf,mode", [("S8", 0, "sync"), ("S8", 1, "submit"), ("S8", 0, "dev"), ("mixed", 1, "sync"),
                                            ("mixed", 0, "submit"), ("mixed", 1, "dev")])
def test_schedules_equal_twins(pkg, synth, ref_intended, layout, gf, mode):
    """Catches a per-sequence array routed by chain position instead of through the map (a subset tick hands sequence k slot j's list,
    another sequence's stamp, rig or frame counts), a skipped table that steps anyway, a mixed tick whose gate misses a semaphore, a
    stale block reported for a skipped sequence, and a kind switch that loses a table's fold order.  40 ticks of a two-rate schedule
    with drops, kinds drawn per (tick, sequence), tuned, retiring and own-detection sequences."""
    import torch
    rigs = LAYOUTS[layout]
    S = len(rigs)
    data = [_Data(synth, k, rigs[k], N_TICKS) for k in range(S)]
    sch = _schedule(S, N_TICKS, seed=7 + S + gf)
    ctx = pkg.Lmot(_params(pkg, gf))
    twins = []
    anchor = layout == "S8" and gf == 0 and mode == "sync"
    for k in range(S):
        tuned = TUNED if k in (1, 2) else None
        retire = k in (3, 4) or (S < 5 and k == 0)
        det = SPARSE if k == S - 1 else None
        prm = _params(pkg, gf)
        for name, val in (det or {}).items():
            setattr(prm, name, val)
        twins.append(_Twin(pkg, prm, rigs[k], tuned, retire))
    keep, stream = [], None
    try:
        ctx.seq_open(S, ring=N_TICKS if mode != "sync" else 4)
        for k in range(S):
            if rigs[k]:
                ctx.seq_set_sensors(k, **_table_kw(rigs[k]))
            if k in (1, 2):
                ctx.seq_set_tracker_params(k, **TUNED)
            if k in (3, 4) or (S < 5 and k == 0):
                ctx.seq_set_track_retirement(k, True)
        ctx.seq_set_detect_params(S - 1, **SPARSE)
        if anchor:
            ref_intended.tracker_reset()
        want, got = [], []
        for t in range(N_TICKS):
            entries = [data[k].entry(sch[t][k], t) if sch[t][k] else None for k in range(S)]
            want.append([twins[k].step(entries[k]) if entries[k] else None for k in range(S)])
            if mode == "sync":
                arr, stride, kp = ctx._seq_entries(entries, False)
                st, res = _raw(ctx, ctx.lib.lmot_seq_tick, arr, S, stride)
                got.append((st, res, [ctx.seq_frame_counts(k) for k in range(S)], [_ids(ctx.seq_track_ids, k) for k in range(S)],
                            ctx.seq_stepped()))
                if anchor and entries[0]:
                    d = entries[0]
                    if "frames" in d:
                        e, g = ref_intended.ground_remove(d["frames"])
                        grid, nc = ref_intended.component_clustering(e)
                        boxes, _ = ref_intended.box_fitting(e, grid, nc)
                    else:
                        boxes = d["lists"]
                    a = ref_intended.tracker_step(boxes, d["timestamp"])
                    r = res[0]
                    assert r["boxes"].shape == boxes.shape and np.array_equal(_bits(r["boxes"]), _bits(np.asarray(boxes, f32))), t
                    assert np.array_equal(r["track_manage"], a["track_manage"]), t
                    np.testing.assert_allclose(r["targets"], a["targets"], rtol=1e-4, atol=1e-4)
            elif mode == "submit":
                ctx.seq_tick_submit(entries)
                keep.append(ctx._keep)
            else:
                if stream is None:
                    stream = torch.cuda.Stream()
                    ctx.set_stream(stream.cuda_stream)
                with torch.cuda.stream(stream):
                    dev = _dev_entries(entries, keep)
                ctx.seq_tick_dev(dev)
        if mode != "sync":
            for t in range(N_TICKS):
                st, res = _raw(ctx, ctx.lib.lmot_seq_collect)
                got.append((st, res, [ctx.seq_frame_counts(k) for k in range(S)], [_ids(ctx.seq_track_ids, k) for k in range(S)],
                            ctx.seq_stepped()))
            ctx.set_stream(None)
        for t, ((st, res, fcs, ids, mask), w) in enumerate(zip(got, want)):
            stepped = [k for k in range(S) if w[k] is not None]
            assert mask == sum(1 << k for k in stepped), t
            assert st == _status([w[k] for k in stepped]), (t, st)
            for k in range(S):
                if w[k] is None:
                    assert res[k] is None and len(fcs[k]) == 0, (t, k)
                    continue
                _same(res[k], fcs[k], w[k], (t, k))
                _same_ids(ids[k], w[k][3], (t, k))
        for k in range(S):
            a, b = ctx.seq_tracker_dump(k), twins[k].ctx.tracker_dump()
            assert a.shape == b.shape and np.array_equal(_bits(a), _bits(b)), (k, "dump")
            assert np.array_equal(ctx.seq_tracker_get_ego(k), twins[k].ctx.tracker_get_ego()), (k, "ego")
    finally:
        ctx.close()
        for tw in twins:
            tw.close()


# ------------------------------------------------------------------------------------------------ 2. a skipped sequence
def test_skipped_sequence_is_untouched(pkg, synth):
    """Catches a skipped table that steps with an empty list (its tracks age), a skipped sequence's ego or stamp folded anyway, its output
    buffers written from the stale block of the ring slot, and its IDs or frame counts taken from that block."""
    S, K = 4, 2
    data = [_Data(synth, k, None, 12) for k in range(S)]
    ctx = pkg.Lmot(_params(pkg))
    try:
        ctx.seq_open(S, ring=2)
        ctx.seq_set_track_retirement(K, True)
        for t in range(4):
            ctx.seq_tick([data[k].entry("F" if (t + k) % 2 else "L", t) for k in range(S)])
        dump, ego, ids = ctx.seq_tracker_dump(K), ctx.seq_tracker_get_ego(K), ctx.seq_track_ids(K)
        t_pred = data[K].ts(11) + 1.0e5
        pred = ctx.seq_predict_tracks(K, [t_pred])
        assert len(dump) > 0 and len(ids) > 0
        so, sets = ctx._seq_out(ctx.params.max_tracks)
        for t in range(4, 10):
            bufs = sets[K][1]
            for a in bufs.values():
                if isinstance(a, np.ndarray):
                    a.view(np.uint8)[:] = 0xA5
            fo = so.seq[K]
            fo.n_elevated = fo.n_ground = fo.num_cluster = fo.n_boxes = -7
            fo.tracks.n_tracks = fo.tracks.n_vis = -7
            entries = [data[k].entry("F" if (t + k) % 2 else "L", t) if k != K else None for k in range(S)]
            arr, stride, kp = ctx._seq_entries(entries, False)
            assert ctx.lib.lmot_seq_tick(ctx.h, arr, S, stride, C.byref(so)) >= 0
            assert (fo.n_elevated, fo.n_ground, fo.num_cluster, fo.n_boxes, fo.tracks.n_tracks, fo.tracks.n_vis) == (-7,) * 6, t
            for name, a in bufs.items():
                if isinstance(a, np.ndarray):
                    assert (a.view(np.uint8) == 0xA5).all(), (t, name)
            assert ctx.seq_stepped() == (1 << S) - 1 - (1 << K)
            assert len(ctx.seq_frame_counts(K)) == 0 and len(ctx.seq_frame_counts(0)) == 1
            assert np.array_equal(ctx.seq_track_ids(K), ids)
        assert np.array_equal(_bits(ctx.seq_tracker_dump(K)), _bits(dump))
        assert np.array_equal(ctx.seq_tracker_get_ego(K), ego)
        p2 = ctx.seq_predict_tracks(K, [t_pred])
        for name in pred:
            assert np.array_equal(_bits(pred[name]), _bits(p2[name])), name
        ctx.seq_tick([data[k].entry("F", 10) for k in range(S)])         # an every-sequence tick sets every bit again
        assert ctx.seq_stepped() == (1 << S) - 1
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ 3. single-kind ticks
_NAMES_SCRIPT = r"""
import importlib, json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
sys.path[:0] = sys.argv[1:3]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
from test_seq_track_gpu import boxes_at
frames = [p for _, p in synth.frames(synth.SceneConfig(seed=5, rings=32, azimuths=900), 1)] * 8
lists = [boxes_at(np.random.default_rng(k).uniform(-30, 30, (6 + k, 2))) for k in range(8)]
arms = {"seq": lambda c, t: c.seq(frames, [t] * 8), "tick_frames": lambda c, t: c.seq_tick([dict(frames=f, timestamp=t) for f in frames]),
        "seq_track": lambda c, t: c.seq_track(lists, [t] * 8), "tick_lists": lambda c, t: c.seq_tick([dict(lists=b, timestamp=t) for b in lists])}
out = {}
for arm, fn in arms.items():
    p = pkg.default_params(); p.max_points = 1 << 16
    ctx = pkg.Lmot(p); ctx.seq_open(8, ring=4)
    fn(ctx, 1e6)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(ctx, 1.1e6)
        torch.cuda.synchronize()
    out[arm] = sorted(e.name for e in prof.events() if "_kernel" in e.name or e.name.startswith(("Memcpy", "Memset")))
    ctx.close()
print(json.dumps(out))
"""


def _kernel_names():
    """kernel, copy and memset names of one S = 8 tick per arm (torch.profiler, in a process of its own as in
    test_seq_detect_params_gpu)"""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _NAMES_SCRIPT, os.path.dirname(here), here], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_single_kind_ticks_are_todays_path(pkg, synth):
    """Catches an all-FRAMES or all-LISTS tick that issues another launch than lmot_seq_dev / lmot_seq_track_dev (an extra pack, a
    restart memset, a per-list copy) or gets other bits."""
    import torch
    names = _kernel_names()
    assert names["seq"] and names["seq"] == names["tick_frames"], names
    assert names["seq_track"] and names["seq_track"] == names["tick_lists"], names
    assert any("pack_lists_seq_kernel" in n for n in names["tick_lists"]) and not any("pack_lists" in n for n in names["tick_frames"])
    S = 4
    data = [_Data(synth, k, None, 8) for k in range(S)]
    a, b = pkg.Lmot(_params(pkg, 1)), pkg.Lmot(_params(pkg, 1))
    keep = []
    try:
        for c in (a, b):
            c.seq_open(S, ring=16)
        for t in range(8):
            kind = "F" if t < 4 else "L"
            entries = [data[k].entry(kind, t) for k in range(S)]
            dev = _dev_entries(entries, keep)
            torch.cuda.synchronize()
            ts = [e["timestamp"] for e in entries]
            v = [e["v_gps"] for e in entries]
            y = [e["yaw_gps"] for e in entries]
            if kind == "F":
                a.seq_dev([e["frames"] for e in dev], ts, v, y)
            else:
                dl, dn, cap = _pad_lists([e["lists"] for e in entries])
                keep += [dl, dn]
                a.seq_track_dev(dl.data_ptr(), dn.data_ptr(), cap, ts, v, y)
            b.seq_tick_dev(dev)
        for t in range(8):
            ra, rb = a.seq_collect(), b.seq_collect()
            for k in range(S):
                for key in FIELDS + ("n_elevated", "n_ground", "num_cluster"):
                    assert np.array_equal(_bits(np.asarray(ra[k][key])), _bits(np.asarray(rb[k][key]))), (t, k, key)
                assert np.array_equal(a.seq_frame_counts(k), b.seq_frame_counts(k)), (t, k)
        for k in range(S):
            assert np.array_equal(_bits(a.seq_tracker_dump(k)), _bits(b.seq_tracker_dump(k))), k
    finally:
        a.close(); b.close()


# ------------------------------------------------------------------------------------------------ 4. restart in a tick
def _pred_dev(pkg, ctx, S, t_us, cap=512):
    """lmot_seq_predict_tracks_dev of every sequence at t_us into fresh device arrays -> (arrays per sequence, device row counts)"""
    import torch
    n_t, bufs, outs = len(t_us), [], []
    for _ in range(S):
        b = {"ids": torch.zeros(cap, dtype=torch.int64, device="cuda"), "track_manage": torch.zeros(cap, dtype=torch.int32, device="cuda"),
             "flags": torch.zeros(n_t * cap, dtype=torch.uint8, device="cuda")}
        for name, w in pkg.PRED_FIELDS:
            b[name] = torch.zeros(n_t * cap * w, dtype=torch.float64, device="cuda")
        outs.append(pkg.pred_out(cap, {n: x.data_ptr() for n, x in b.items()}))
        bufs.append(b)
    dn = torch.zeros(S, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.seq_predict_tracks_dev(np.tile(np.asarray(t_us, np.float64), (S, 1)), outs, dn.data_ptr())
    return bufs, dn


@pytest.mark.parametrize("compat", [0, 1])
def test_restart_in_tick(pkg, synth, compat):
    """Catches a restart that drains or forgets other sequences' uncollected ticks, one that runs before a prediction queued ahead of it
    (the prediction would see the emptied table), one that keeps the old ego fold, first-frame flag or spawn counter (IDs not from 0),
    and a restart that leaks into the other tables."""
    import torch
    S, K, R = 4, 3, 9
    data = [_Data(synth, k, None, 14) for k in range(S)]
    new = _Data(synth, 7, None, 14)                   # the new stream on sequence K from tick R on
    prm = _params(pkg)
    prm.oracle_compat_first_frame = compat
    a, b = pkg.Lmot(prm), pkg.Lmot(prm)
    twin = _Twin(pkg, prm, retire=True)
    try:
        for c in (a, b):
            c.seq_open(S, ring=8)
            c.seq_set_track_retirement(K, True)
        kinds = lambda t, k: "F" if (t + k) % 3 else "L"
        for t in range(6):
            for c in (a, b):
                c.seq_tick([data[k].entry(kinds(t, k), t) for k in range(S)])
        for t in range(6, R):
            for c in (a, b):
                c.seq_tick_submit([data[k].entry(kinds(t, k), t) for k in range(S)])
        t_pred = [max(data[k].ts(R - 1) for k in range(S)) + 2.0e4]
        pa, pb = _pred_dev(pkg, a, S, t_pred), _pred_dev(pkg, b, S, t_pred)
        got_a, got_b, ids_k, want = [], [], [], []
        for t in range(R, 13):
            ea = [data[k].entry(kinds(t, k), t) if k != K else new.entry(kinds(t, k), t, restart=t == R) for k in range(S)]
            eb = [data[k].entry(kinds(t, k), t) if k != K else None for k in range(S)]
            if t == R:
                eb[K] = None
            a.seq_tick_submit(ea)
            b.seq_tick_submit(eb)
            want.append(twin.step(ea[K]))
        for t in range(6, 13):
            got_a.append(_raw(a, a.lib.lmot_seq_collect))
            ids_k.append((a.seq_track_ids(K), a.seq_frame_counts(K)) if t >= R else None)
            got_b.append(_raw(b, b.lib.lmot_seq_collect))
        assert len(got_a) == 7 and a.lib.lmot_seq_collect(a.h, None) == pkg.ERR_STATE     # nothing dropped, nothing extra
        torch.cuda.synchronize()
        for k in range(S):
            for name, x in pa[0][k].items():
                assert np.array_equal(_bits(x.cpu().numpy()), _bits(pb[0][k][name].cpu().numpy())), (k, name)
        assert torch.equal(pa[1], pb[1]) and int(pa[1][K]) > 0
        for i, ((_, ra), (_, rb)) in enumerate(zip(got_a, got_b)):
            for k in range(S):
                if k == K and i + 6 >= R:
                    continue
                for key in FIELDS:
                    assert np.array_equal(_bits(ra[k][key]), _bits(rb[k][key])), (i, k, key)
        for i, w in enumerate(want):
            ids, fc = ids_k[R - 6 + i]
            _same(got_a[R - 6 + i][1][K], fc, w, ("restart", i))
            assert np.array_equal(ids, w[3]), i
        assert len(want[-1][3]) > 0 and want[-1][3].min() >= 0 and ids_k[R - 6][0].tolist() == list(range(len(ids_k[R - 6][0])))
        for k in range(S):
            if k != K:
                assert np.array_equal(_bits(a.seq_tracker_dump(k)), _bits(b.seq_tracker_dump(k))), k
        assert np.array_equal(_bits(a.seq_tracker_dump(K)), _bits(twin.ctx.tracker_dump()))
        assert np.array_equal(a.seq_tracker_get_ego(K), twin.ctx.tracker_get_ego())
    finally:
        a.close(); b.close(); twin.close()


# ------------------------------------------------------------------------------------------------ 5. one ring for every kind of tick
def test_interleave_with_existing_ticks(pkg, synth):
    """Catches a tick kind with a ring of its own (or its own in-flight count), a full ring that does not refuse a host tick, a dev tick
    that does not drop the oldest, and fetch keeping the ticks it drops."""
    import torch
    S = 3
    data = [_Data(synth, k, None, 12) for k in range(S)]
    ctx = pkg.Lmot(_params(pkg))
    twins = [_Twin(pkg, _params(pkg)) for _ in range(S)]
    keep = []
    try:
        ctx.seq_open(S, ring=3)
        want = []

        def step_twins(entries):
            want.append([twins[k].step(entries[k]) if entries[k] else None for k in range(S)])
            return entries

        e = step_twins([data[k].entry("F", 0) for k in range(S)])
        ctx.seq_submit([x["frames"] for x in e], [x["timestamp"] for x in e], [x["v_gps"] for x in e], [x["yaw_gps"] for x in e])
        e = step_twins([data[k].entry("L", 1) for k in range(S)])
        ctx.seq_track_submit([x["lists"] for x in e], [x["timestamp"] for x in e], [x["v_gps"] for x in e], [x["yaw_gps"] for x in e])
        ctx.seq_tick_submit(step_twins([data[0].entry("F", 2), None, data[2].entry("L", 2)]))
        full = [data[k].entry("F", 3) for k in range(S)]
        arr, stride, kp = ctx._seq_entries(full, False)
        assert ctx.lib.lmot_seq_tick_submit(ctx.h, arr, S, stride) == pkg.ERR_STATE
        for t in range(3):
            st, res = _raw(ctx, ctx.lib.lmot_seq_collect)
            for k in range(S):
                if want[t][k] is None:
                    assert res[k] is None
                else:
                    _same(res[k], ctx.seq_frame_counts(k), want[t][k], (t, k))
        # fetch: the most recent tick, older ones dropped
        ctx.seq_tick_submit(step_twins([None, data[1].entry("L", 3), None]))
        ctx.seq_tick_submit(step_twins([data[0].entry("L", 4), data[1].entry("F", 4), None]))
        res = ctx.seq_fetch()
        _same(res[0], ctx.seq_frame_counts(0), want[-1][0], "fetch 0")
        _same(res[1], ctx.seq_frame_counts(1), want[-1][1], "fetch 1")
        assert res[2] is None and ctx.lib.lmot_seq_collect(ctx.h, None) == pkg.ERR_STATE
        # device form: a full ring drops the oldest tick
        for t in range(5, 9):
            entries = step_twins([data[k].entry("F" if (t + k) % 2 else "L", t) if (t + k) % 4 else None for k in range(S)])
            dev = _dev_entries(entries, keep)
            torch.cuda.synchronize()
            ctx.seq_tick_dev(dev)
        for t in range(6, 9):
            st, res = _raw(ctx, ctx.lib.lmot_seq_collect)
            w = want[t]
            for k in range(S):
                if w[k] is None:
                    assert res[k] is None, (t, k)
                else:
                    _same(res[k], ctx.seq_frame_counts(k), w[k], (t, k))
        assert ctx.lib.lmot_seq_collect(ctx.h, None) == pkg.ERR_STATE
        for k in range(S):
            assert np.array_equal(_bits(ctx.seq_tracker_dump(k)), _bits(twins[k].ctx.tracker_dump())), k
    finally:
        ctx.close()
        for tw in twins:
            tw.close()


# ------------------------------------------------------------------------------------------------ 6. validation and capacity
def test_validation_and_capacity(pkg, synth):
    """Catches a rejected tick that still took a ring slot, restarted a table or folded an ego pose, a rejection code mixed up, and a
    device list above max_boxes that fails the whole tick instead of its own sequence."""
    import torch
    S = 2
    prm = _params(pkg, max_boxes=64)
    ctx = pkg.Lmot(prm)
    keep = []
    try:
        assert ctx.lib.lmot_seq_tick_submit(ctx.h, (pkg.SeqEntry * S)(), S, 4) == pkg.ERR_INVALID          # no open set
        ctx.seq_open(S, ring=2)
        ego0 = [ctx.seq_tracker_get_ego(k) for k in range(S)]
        d = _Data(synth, 0, None, 2)
        pts = np.ascontiguousarray(d.frames[0][0], f32)
        big = np.zeros((prm.max_points + 1, 4), f32)
        many = np.zeros((65, 8, 3), f32)
        dp = torch.from_numpy(pts).cuda()
        dn = torch.tensor([3], dtype=torch.int32).cuda()
        torch.cuda.synchronize()
        ptr_arr = lambda *ps: (C.c_void_p * len(ps))(*ps)
        int_arr = lambda *ns: (C.c_int * len(ns))(*ns)

        def entries(*specs):
            arr = (pkg.SeqEntry * S)()
            for k, sp in enumerate(specs):
                for name, val in sp.items():
                    if name == "data":
                        keep.append(val)
                        val = C.cast(val, C.POINTER(C.c_void_p))
                    elif name == "n":
                        keep.append(val)
                        val = C.cast(val, C.POINTER(C.c_int))
                    setattr(arr[k], name, val)
            return arr

        F = dict(kind=pkg.SEQ_FRAMES, data=ptr_arr(pts.ctypes.data), n=int_arr(len(pts)), timestamp_us=1e6)
        L = dict(kind=pkg.SEQ_LISTS, data=ptr_arr(many.ctypes.data), n=int_arr(3), timestamp_us=1e6)
        DL = dict(kind=pkg.SEQ_LISTS, data=ptr_arr(dp.data_ptr()), d_counts=dn.data_ptr(), cap_per_list=4, timestamp_us=1e6)
        DF = dict(kind=pkg.SEQ_FRAMES, data=ptr_arr(dp.data_ptr()), n=int_arr(len(pts)), timestamp_us=1e6)
        host = [
            (pkg.ERR_INVALID, [dict(kind=3), F]), (pkg.ERR_INVALID, [dict(F, flags=2), F]), (pkg.ERR_INVALID, [{}, {}]),
            (pkg.ERR_INVALID, [dict(flags=1), F]), (pkg.ERR_INVALID, [dict(F, data=None), F]), (pkg.ERR_INVALID, [dict(F, n=None), F]),
            (pkg.ERR_INVALID, [dict(F, n=int_arr(-1)), F]), (pkg.ERR_INVALID, [F, dict(L, n=None)]),
            (pkg.ERR_INVALID, [F, dict(L, data=ptr_arr(None))]), (pkg.ERR_INVALID, [dict(L, n=int_arr(-2)), F]),
            (pkg.ERR_CAPACITY, [dict(F, data=ptr_arr(big.ctypes.data), n=int_arr(len(big))), F]),
            (pkg.ERR_CAPACITY, [F, dict(L, n=int_arr(65))]),
        ]
        for i, (code, specs) in enumerate(host):
            assert ctx.lib.lmot_seq_tick_submit(ctx.h, entries(*specs), S, 4) == code, i
        assert ctx.lib.lmot_seq_tick_submit(ctx.h, entries(F, F), 1, 4) == pkg.ERR_INVALID
        assert ctx.lib.lmot_seq_tick_submit(ctx.h, entries(F, L), S, 2) == pkg.ERR_INVALID      # stride < 3 with frames
        dev = [
            (pkg.ERR_INVALID, [dict(DL, d_counts=None), DF]), (pkg.ERR_INVALID, [dict(DL, cap_per_list=0), DF]),
            (pkg.ERR_INVALID, [DL, dict(DF, data=ptr_arr(dp.data_ptr() + 4))]), (pkg.ERR_INVALID, [dict(DL, data=ptr_arr(None)), DF]),
            (pkg.ERR_CAPACITY, [DL, dict(DF, n=int_arr(prm.max_points + 1))]),
        ]
        for i, (code, specs) in enumerate(dev):
            assert ctx.lib.lmot_seq_tick_dev(ctx.h, entries(*specs), S) == code, i
        ctx.enable_timing(True)
        assert ctx.lib.lmot_seq_tick_submit(ctx.h, entries(F, F), S, 4) == pkg.ERR_STATE
        ctx.enable_timing(False)
        assert ctx.lib.lmot_seq_collect(ctx.h, None) == pkg.ERR_STATE              # nothing was submitted
        for k in range(S):
            assert len(ctx.seq_tracker_dump(k)) == 0 and np.array_equal(ctx.seq_tracker_get_ego(k), ego0[k]), k
        # a device list above max_boxes: LMOT_ERR_CAPACITY for its sequence only
        lst = [_ListSeq(0, 2, n_obj=80).lists[0][:80], _ListSeq(1, 2).lists[0]]
        assert len(lst[0]) > 64
        twins = [_Twin(pkg, prm, rig=[RIG[0]]), _Twin(pkg, prm)]
        try:
            ctx.seq_set_sensors(0, **_table_kw([RIG[0]]))
            es = [dict(lists=[lst[0]], timestamp=2e6, v_gps=0.0, yaw_gps=0.0), dict(lists=lst[1], timestamp=2e6, v_gps=0.0, yaw_gps=0.0)]
            want = [twins[k].step(es[k]) for k in range(S)]
            assert want[0][0] == pkg.ERR_CAPACITY and want[1][0] >= 0
            devs = _dev_entries(es, keep)
            torch.cuda.synchronize()
            ctx.seq_tick_dev(devs)
            st, res = _raw(ctx, ctx.lib.lmot_seq_collect)
            assert st == pkg.ERR_CAPACITY
            for k in range(S):
                _same(res[k], ctx.seq_frame_counts(k), want[k], k)
            assert len(res[0]["boxes"]) == 64
        finally:
            for tw in twins:
                tw.close()
    finally:
        ctx.close()
