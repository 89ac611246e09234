"""GPU parity of merging rigs (lmot_set_rig_merge / lmot_seq_set_rig_merge): the sensors' elevated clouds of a tick are moved into the
vehicle frame, concatenated in table order and clustered and boxed as one cloud.

Oracle (rig_merge_scenes.merged_detection): the reference's groundRemove per sensor under its mount, the rig arithmetic on each elevated
cloud, the concatenation, then the reference's componentClustering + boxFitting with sensorHeight = the vehicle frame's height, and the
reference's immUkfJpdaf on the boxes (moved into the dead-reckoned global frame when global_frame = 1).  Sequences, switching and in-flight
ticks are compared with twin contexts.  Bars as in test_sensor_rig_gpu: counts and boxes bit-exact, identical trackManage / static /
visible flags, UKF states within 1e-4 relative on positive-definite filters.
"""
import ctypes as C

import numpy as np
import pytest

from rig_merge_scenes import boxes_per_object, doubled_view_detection, merged_detection, overlap_rig, overlap_ticks, table_kw
from test_global_frame_gpu import _ego, xf_apply, xf_pair
from test_sensor_rig_gpu import check_tick, ego_sequence
from test_tracker_gpu import INTS, STATE, TOL, _pd_tracks, _rel_err

pytestmark = pytest.mark.gpu
f32 = np.float32

HEIGHTS = [2.0, 1.2, 0.8, 1.8, 1.6, 1.0, 2.2, 1.4]
TRACK_KEYS = ("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb")


def _params(pkg, gf=0, h_vehicle=2.0, **kw):
    p = pkg.default_params()
    p.global_frame = gf
    p.sensor_height = h_vehicle
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _merging(pkg, rig, params, on=1):
    ctx = pkg.Lmot(params)
    ctx.set_sensors(**table_kw(rig))
    ctx.set_rig_merge(on)
    return ctx


def _same(a, b, what):
    for k in ("boxes",) + TRACK_KEYS:
        assert a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), (what, k)


def _seq_same(r, rows, w, wrows, what):
    """sequence result r (+ lmot_seq_frame_counts rows) against a twin's lmot_batch result w"""
    assert [tuple(x) for x in rows] == wrows, what
    assert (r["n_elevated"], r["n_ground"], r["num_cluster"]) == tuple(int(sum(x[i] for x in wrows)) for i in range(3)), what
    _same(r, w, what)


def _rows(r):
    return list(zip(r["n_elevated"], r["n_ground"], r["num_cluster"], r["n_boxes"]))


# ------------------------------------------------------------------------------------------------ 1. the oracle, F sensors
@pytest.mark.parametrize("gf", [0, 1])
@pytest.mark.parametrize("F", [1, 2, 4, 8])
def test_merged_parity(pkg, ref_intended, synth, F, gf):
    import torch
    ref = ref_intended
    h_v = 1.5 if F >= 4 else 2.0
    rig = overlap_rig(F, heights=HEIGHTS[:F], h_vehicle=h_v)
    ticks = list(overlap_ticks(synth, rig, 8, seed=11 + F))
    det = [merged_detection(ref, rig, frames, h_v) for _, frames, _, _ in ticks]
    assert sum(len(b) for _, b, _, _ in det) > 0
    egos = ego_sequence(pkg, [(t[0], None) for t in ticks]) if gf else [None] * len(ticks)
    ref.tracker_reset()
    want = []
    for f, ((ts, _, _, _), (rows, b, _, _)) in enumerate(zip(ticks, det)):
        v, yaw = _ego(f)
        fwd, back = xf_pair(egos[f]) if gf else (None, None)
        want.append((ref.tracker_step(b if not gf else xf_apply(fwd, b), ts, v, yaw), back, ref.tracker_dump()))
    ctx = _merging(pkg, rig, _params(pkg, gf, h_v))
    try:
        for f, ((ts, frames, _, _), (rows, b, _, _), (a, back, da)) in enumerate(zip(ticks, det, want)):
            check_tick(ctx.batch(frames, ts, *_ego(f)), rows, b, a, back, f)
            db = ctx.tracker_dump()
            assert np.array_equal(da[:, INTS], db[:, INTS]), f
            ok = _pd_tracks(da)
            err = _rel_err(da[ok][:, STATE], db[ok][:, STATE])
            assert err.size == 0 or err.max() < TOL, (f, float(err.max()))
    finally:
        ctx.close()
    ctx = _merging(pkg, rig, _params(pkg, gf, h_v))
    try:
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)
        with torch.cuda.stream(stream):
            dev = [[torch.from_numpy(p).cuda() for p in frames] for _, frames, _, _ in ticks]
            for f, ((ts, frames, _, _), d) in enumerate(zip(ticks, dev)):
                ctx.batch_dev([(t.data_ptr(), len(p)) for t, p in zip(d, frames)], ts, *_ego(f))
        for f, ((rows, b, _, _), (a, back, _)) in enumerate(zip(det, want)):
            check_tick(ctx.batch_collect(), rows, b, a, back, f)
        ctx.set_stream(None)
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ 2. sequences of three kinds
def test_sequences_merge_separate_and_tableless(pkg, synth):
    """sequence 0: a merging 4-sensor rig; 1: a separate 2-sensor rig; 2: no table.  lmot_seq, then lmot_seq_tick with a skip, a
    restart and a LISTS step; each sequence equals its twin context (merge + lmot_batch, lmot_batch, lmot_frame / lmot_track_step)"""
    rig0, rig1 = overlap_rig(4, heights=HEIGHTS[:4]), overlap_rig(2, heights=[1.3, 1.7])
    t0 = list(overlap_ticks(synth, rig0, 9, seed=21))
    t1 = list(overlap_ticks(synth, rig1, 9, seed=22))
    t2 = [p for _, p in synth.frames(synth.SceneConfig(seed=23, rings=32, azimuths=900), 9)]
    ctx = pkg.Lmot(_params(pkg))
    tw0, tw1, tw2 = _merging(pkg, rig0, _params(pkg)), _merging(pkg, rig1, _params(pkg), on=0), pkg.Lmot(_params(pkg))
    try:
        ctx.seq_open(3, ring=4)
        ctx.seq_set_sensors(0, **table_kw(rig0))
        ctx.seq_set_sensors(1, **table_kw(rig1))
        ctx.seq_set_rig_merge(0, 1)
        assert ctx.seq_get_rig_merge(0) and not ctx.seq_get_rig_merge(1) and not ctx.seq_get_rig_merge(2)
        for f in range(9):
            ts = [t0[f][0], t1[f][0] + 1e3, (f + 1) * 1e5 + 2e3]
            ego = [_ego(f), _ego(f + 1), _ego(f + 2)]
            if f < 4:
                got = ctx.seq([t0[f][1], t1[f][1], t2[f]], ts, [e[0] for e in ego], [e[1] for e in ego])
                kinds = ["F", "F", "F"]
            else:
                kinds = {4: ["F", None, "F"], 5: ["R", "F", "F"], 6: ["F", "F", "L"], 7: [None, "F", "L"], 8: ["F", "R", "F"]}[f]
                ent = []
                for k, kind in enumerate(kinds):
                    if kind is None:
                        ent.append(None)
                        continue
                    d = dict(timestamp=ts[k], v_gps=ego[k][0], yaw_gps=ego[k][1], restart=kind == "R")
                    if kind == "L":
                        d["lists"] = _some_boxes(f)
                    else:
                        d["frames"] = [t0[f][1], t1[f][1], t2[f]][k]
                    ent.append(d)
                got = ctx.seq_tick(ent)
            for k, kind in enumerate(kinds):
                if kind is None:
                    assert got[k] is None
                    continue
                tw = (tw0, tw1, tw2)[k]
                if kind == "R":
                    tw.tracker_reset()
                if k < 2:
                    w = tw.batch((t0, t1)[k][f][1], ts[k], *ego[k])
                    _seq_same(got[k], ctx.seq_frame_counts(k), w, _rows(w), (f, k))
                elif kind == "L":
                    w = dict(tw2.track_step(_some_boxes(f), ts[k], *ego[k]), boxes=_some_boxes(f))
                    _same(got[k], w, (f, k))
                else:
                    w = tw2.frame(t2[f], ts[k], *ego[k])
                    _same(got[k], w, (f, k))
                    assert (got[k]["n_elevated"], got[k]["num_cluster"]) == (w["n_elevated"], w["num_cluster"])
                assert ctx.seq_tracker_dump(k).tobytes() == tw.tracker_dump().tobytes(), (f, k)
        # a merging sequence's counts: n_elevated per sensor, the merged cloud's num_cluster / n_boxes in row 0 only
        rows = ctx.seq_frame_counts(0)
        assert len(rows) == 4 and all(r[2] == 0 and r[3] == 0 for r in rows[1:]) and rows[0][2] > 0
    finally:
        for c in (ctx, tw0, tw1, tw2):
            c.close()


def _some_boxes(f):
    """a small box list of step f (LISTS entries)"""
    b = np.zeros((3, 8, 3), f32)
    for i in range(3):
        cx, cy = 8.0 + 4 * i + 0.3 * f, -6.0 + 5 * i
        b[i, :, 0] = cx + np.array([1, 1, -1, -1, 1, 1, -1, -1], f32)
        b[i, :, 1] = cy + np.array([0.5, -0.5, -0.5, 0.5] * 2, f32)
        b[i, :, 2] = np.array([-1.7] * 4 + [-0.2] * 4, f32)
    return b


# ------------------------------------------------------------------------------------------------ 3. own detection values, deskew
def _timed(frames, f):
    """deskew's time field (column 3, seconds before the stamp) on every point of the sensor clouds"""
    out = []
    for p in frames:
        q = p.copy()
        q[:, 3] = (-0.1 * (np.arange(len(q)) / max(len(q), 1))).astype(f32)
        out.append(q)
    return out


def test_merge_with_own_detect_params_and_deskew(pkg, synth):
    rig = overlap_rig(4, heights=HEIGHTS[:4])
    ticks = list(overlap_ticks(synth, rig, 6, seed=31))
    own = dict(sensor_height=1.6, t_width_max=2.2, min_cluster_points=4)
    ctx = pkg.Lmot(_params(pkg))
    tw0 = _merging(pkg, rig, _params(pkg, **own))
    tw1 = _merging(pkg, rig, _params(pkg))
    try:
        tw1.set_deskew(on=1)
        ctx.seq_open(2, ring=2)
        for k in range(2):
            ctx.seq_set_sensors(k, **table_kw(rig))
            ctx.seq_set_rig_merge(k, 1)
        ctx.seq_set_detect_params(0, **own)
        ctx.seq_set_deskew(1, on=1)
        tw_boxes = [[], []]
        for f, (ts, frames, _, _) in enumerate(ticks):
            fr = _timed(frames, f)
            v, yaw = _ego(f)
            got = ctx.seq([fr, fr], [ts, ts], [v, v], [yaw, yaw])
            for k, tw in enumerate((tw0, tw1)):
                w = tw.batch(fr, ts, v, yaw)
                _seq_same(got[k], ctx.seq_frame_counts(k), w, _rows(w), (f, k))
                tw_boxes[k].append(w["boxes"].tobytes())
        # both variants really differ from plain merging
        plain = _merging(pkg, rig, _params(pkg))
        try:
            diff = [0, 0]
            for f, (ts, frames, _, _) in enumerate(ticks):
                fr = _timed(frames, f)
                p = plain.batch(fr, ts, *_ego(f))["boxes"]
                for k in range(2):
                    diff[k] += p.tobytes() != tw_boxes[k][f]
            assert all(diff), diff
        finally:
            plain.close()
    finally:
        for c in (ctx, tw0, tw1):
            c.close()


# ------------------------------------------------------------------------------------------------ 4. switching: no stale state
def test_switching_leaves_no_stale_state(pkg, synth):
    """one context switches merge on and off between ticks; every tick's detection equals a twin that never switched, and its tracker
    equals a twin fed the same lists through lmot_track_step"""
    import torch
    rig = overlap_rig(4, heights=HEIGHTS[:4])
    ticks = list(overlap_ticks(synth, rig, 12, seed=41))
    pattern = [1, 1, 0, 1, 0, 0, 1, 0, 1, 1, 0, 1]
    ctx, on, off = _merging(pkg, rig, _params(pkg), on=0), _merging(pkg, rig, _params(pkg)), _merging(pkg, rig, _params(pkg), on=0)
    trk = pkg.Lmot(_params(pkg))
    try:
        for f, ((ts, frames, _, _), m) in enumerate(zip(ticks, pattern)):
            ctx.set_rig_merge(m)
            v, yaw = _ego(f)
            if f % 3 == 2:                       # device frames as well
                d = [torch.from_numpy(p).cuda() for p in frames]
                torch.cuda.synchronize()
                ctx.batch_dev([(t.data_ptr(), len(p)) for t, p in zip(d, frames)], ts, v, yaw)
                r = ctx.batch_collect()
            else:
                r = ctx.batch(frames, ts, v, yaw)
            w = (on if m else off).batch(frames, ts, v, yaw)
            (off if m else on).batch(frames, ts, v, yaw)          # both twins see every tick
            assert _rows(r) == _rows(w), f
            assert r["boxes"].tobytes() == w["boxes"].tobytes(), f
            t = trk.track_step(w["boxes"], ts, v, yaw)
            for k in TRACK_KEYS:
                assert r[k].tobytes() == t[k].tobytes(), (f, k)
    finally:
        for c in (ctx, on, off, trk):
            c.close()


# ------------------------------------------------------------------------------------------------ 5. ticks in flight keep their setting
def test_in_flight_ticks_keep_their_setting(pkg, synth):
    rig = overlap_rig(4, heights=HEIGHTS[:4])
    ticks = list(overlap_ticks(synth, rig, 4, seed=51))
    plan = [1, 0, 1, 0]
    ctx, on, off = _merging(pkg, rig, _params(pkg), on=0), _merging(pkg, rig, _params(pkg)), _merging(pkg, rig, _params(pkg), on=0)
    trk = pkg.Lmot(_params(pkg))
    try:
        for (ts, frames, _, _), m in zip(ticks, plan):
            ctx.set_rig_merge(m)
            ctx.batch_submit(frames, ts)
        ctx.set_rig_merge(1)
        for (ts, frames, _, _), m in zip(ticks, plan):
            r = ctx.batch_collect()
            w = (on if m else off).batch(frames, ts)
            assert _rows(r) == _rows(w) and r["boxes"].tobytes() == w["boxes"].tobytes(), m
            t = trk.track_step(w["boxes"], ts)
            assert r["track_manage"].tobytes() == t["track_manage"].tobytes()
        # sequences: the tick keeps the setting it was submitted with
        ctx.seq_open(1, ring=4)
        ctx.seq_set_sensors(0, **table_kw(rig))
        tw_on, tw_off = _merging(pkg, rig, _params(pkg)), _merging(pkg, rig, _params(pkg), on=0)
        try:
            for (ts, frames, _, _), m in zip(ticks, plan):
                ctx.seq_set_rig_merge(0, m)
                ctx.seq_submit([frames], [ts])
            ctx.seq_set_rig_merge(0, 0)
            tw = pkg.Lmot(_params(pkg))
            try:
                for (ts, frames, _, _), m in zip(ticks, plan):
                    g = ctx.seq_collect()[0]
                    w = (tw_on if m else tw_off).batch(frames, ts)
                    t = tw.track_step(w["boxes"], ts)
                    _seq_same(g, ctx.seq_frame_counts(0), dict(w, **{k: t[k] for k in TRACK_KEYS}), _rows(w), m)
            finally:
                tw.close()
        finally:
            tw_on.close(); tw_off.close()
    finally:
        for c in (ctx, on, off, trk):
            c.close()


# ------------------------------------------------------------------------------------------------ 6. a merged cloud above max_points
def _raw_batch(ctx, frames, ts):
    ptrs, ns, F, stride, keep = ctx._batch_args(frames, False)
    bo, bufs = ctx._batch_out(ctx.params.max_tracks)
    st = ctx.lib.lmot_batch(ctx.h, ptrs, ns, F, stride, C.c_double(ts), C.c_double(0), C.c_double(0), C.byref(bo))
    return st, ctx._batch_result(bo, bufs)


def test_merged_cloud_above_max_points(pkg, ref_intended, synth):
    ref = ref_intended
    rig = overlap_rig(7, heights=HEIGHTS[:7])
    ticks = list(overlap_ticks(synth, rig, 4, seed=61))
    view = [p for _, p in synth.frames(synth.SceneConfig(seed=62, rings=16, azimuths=900), 4)]     # (each frame below max_points)
    biggest = max(len(p) for _, frames, _, _ in ticks for p in frames)
    full = merged_detection(ref, rig, ticks[0][1])[2]
    mp = biggest + 64
    assert len(full) > mp + 1000, (len(full), mp)                   # the merged cloud of every tick is cut
    prm = _params(pkg, max_points=mp)
    ctx = _merging(pkg, rig, prm)
    twin = _merging(pkg, rig, _params(pkg, max_points=mp))
    try:
        ref.tracker_reset()
        for f, (ts, frames, _, _) in enumerate(ticks):
            rows, b, E, cut = merged_detection(ref, rig, frames, max_points=mp)
            assert cut and len(E) == mp
            st, r = _raw_batch(ctx, frames, ts)
            assert st == pkg.ERR_CAPACITY, st
            a = ref.tracker_step(b, ts)
            check_tick(r, rows, b, a, None, f)
        # a sequence set: the merging sequence reports the capacity error, the table-less one is unaffected
        ctx.seq_open(2, ring=2)
        ctx.seq_set_sensors(0, **table_kw(rig))
        ctx.seq_set_rig_merge(0, 1)
        plain = pkg.Lmot(_params(pkg, max_points=mp))
        try:
            for f, (ts, frames, _, _) in enumerate(ticks):
                ptrs, ns, S, stride, keep = ctx._seq_args([frames, view[f]], False)
                so, sets = ctx._seq_out(ctx.params.max_tracks)
                tsa = ctx.seq_scalars(2, [ts, ts])
                zero = ctx.seq_scalars(2, 0.0)
                st = ctx.lib.lmot_seq(ctx.h, ptrs, ns, S, stride, tsa, zero, zero, C.byref(so))
                got = ctx._seq_result(so, sets)
                assert st == pkg.ERR_CAPACITY, st
                ws, w = _raw_batch(twin, frames, ts)
                assert ws == pkg.ERR_CAPACITY
                _seq_same(got[0], ctx.seq_frame_counts(0), w, _rows(w), f)
                _same(got[1], plain.frame(view[f], ts), f)
        finally:
            plain.close()
    finally:
        ctx.close(); twin.close()


# ------------------------------------------------------------------------------------------------ 7. off is today's path
_NAMES_SCRIPT = r"""
import importlib, json, sys
import torch
from torch.profiler import ProfilerActivity, profile
sys.path[:0] = sys.argv[1:3]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
from rig_merge_scenes import overlap_rig, overlap_ticks, table_kw
rig = overlap_rig(4, heights=[2.0, 1.2, 0.8, 1.8])
ticks = list(overlap_ticks(synth, rig, 3, seed=71))
out = {}
for arm in ("untouched", "toggled", "merging", "plain", "on_no_table", "seq_untouched", "seq_on_no_table"):
    ctx = pkg.Lmot(pkg.default_params())
    if arm in ("untouched", "toggled", "merging"):
        ctx.set_sensors(**table_kw(rig))
    if arm in ("toggled", "merging", "on_no_table"):
        ctx.set_rig_merge(1)
    if arm == "toggled":
        ctx.set_rig_merge(0)
    if arm.startswith("seq"):
        ctx.seq_open(2, ring=2)
        if arm == "seq_on_no_table":
            ctx.seq_set_rig_merge(0, 1); ctx.seq_set_rig_merge(1, 1)
    def run(f):
        ts, frames, _, _ = ticks[f]
        if arm.startswith("seq"):
            ctx.seq(frames[:2], [ts, ts])
        else:
            ctx.batch(frames, ts)
        torch.cuda.synchronize()
    run(0)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(1); run(2)
    out[arm] = [e.name for e in prof.events() if str(e.device_type).endswith("CUDA") and "Memcpy" not in e.name and "Memset" not in e.name]
    ctx.close()
print(json.dumps(out))
"""


def test_off_is_todays_path(pkg, synth):
    """results: never touched = switched on and off again (with a table), and merge on without a table = no table; launches by name
    (torch.profiler in a child process): the same, no rig_merge_kernel, and with merge on exactly one rig_merge_kernel and one CCL
    launch per tick"""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    rig = overlap_rig(4, heights=HEIGHTS[:4])
    ticks = list(overlap_ticks(synth, rig, 5, seed=71))
    untouched, toggled = _merging(pkg, rig, _params(pkg), on=0), _merging(pkg, rig, _params(pkg))
    plain, on_no_table = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        toggled.set_rig_merge(0)
        on_no_table.set_rig_merge(1)
        assert on_no_table.get_rig_merge() and not toggled.get_rig_merge()
        for f, (ts, frames, _, _) in enumerate(ticks):
            v, yaw = _ego(f)
            runs = {name: c.batch(frames, ts, v, yaw) for name, c in (("untouched", untouched), ("toggled", toggled), ("plain", plain),
                                                                      ("on_no_table", on_no_table))}
            for a, b in (("untouched", "toggled"), ("plain", "on_no_table")):
                assert _rows(runs[a]) == _rows(runs[b]), (f, a)
                _same(runs[a], runs[b], (f, a))
            assert untouched.tracker_dump().tobytes() == toggled.tracker_dump().tobytes()
            assert plain.tracker_dump().tobytes() == on_no_table.tracker_dump().tobytes()
    finally:
        for c in (untouched, toggled, plain, on_no_table):
            c.close()
    r = subprocess.run([sys.executable, "-c", _NAMES_SCRIPT, os.path.dirname(here), here], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    n = json.loads(r.stdout.strip().splitlines()[-1])
    # (kernels of different streams may interleave in any order in a trace: compared as multisets)
    for a, b in (("untouched", "toggled"), ("plain", "on_no_table"), ("seq_untouched", "seq_on_no_table")):
        assert n[a] and sorted(n[a]) == sorted(n[b]), (a, b)
        assert not any("rig_merge" in x for x in n[a] + n[b])
    assert sum("rig_merge_kernel" in x for x in n["merging"]) == 2                # one per tick
    assert sum("ccl_dense_kernel" in x for x in n["merging"]) == 2                # one CCL launch per tick: the merged cloud is its unit


# ------------------------------------------------------------------------------------------------ 8. validation
def test_validation(pkg, synth):
    rig = overlap_rig(2)
    frames = next(overlap_ticks(synth, rig, 1, seed=81))[1]
    ctx = pkg.Lmot(_params(pkg))
    try:
        for bad in (2, -1, 7):
            with pytest.raises(pkg.LmotError) as ei:
                ctx.set_rig_merge(bad)
            assert ei.value.status == pkg.ERR_INVALID
            assert ctx.get_rig_merge() is False
        with pytest.raises(pkg.LmotError) as ei:
            ctx.seq_set_rig_merge(0, 1)                              # no open set
        assert ei.value.status == pkg.ERR_INVALID
        ctx.seq_open(2, ring=2)
        for k, on in ((2, 1), (-1, 1), (0, 3)):
            with pytest.raises(pkg.LmotError) as ei:
                ctx.seq_set_rig_merge(k, on)
            assert ei.value.status == pkg.ERR_INVALID
        assert not ctx.seq_get_rig_merge(0)
        ctx.seq_set_rig_merge(1, 1)
        ctx.seq_tracker_reset(1)
        assert ctx.seq_get_rig_merge(1)                              # reset keeps it
        ctx.seq_open(2, ring=2)
        assert not ctx.seq_get_rig_merge(1)                          # reopening turns it off
        # timing mode: a merging submission is refused, a tick without a table is not merging
        ctx.set_rig_merge(1)
        ctx.enable_timing(True)
        ctx.batch(frames, 1e5)
        ctx.set_sensors(**table_kw(rig))
        with pytest.raises(pkg.LmotError) as ei:
            ctx.batch(frames, 2e5)
        assert ei.value.status == pkg.ERR_STATE
        ctx.set_rig_merge(0)
        ctx.batch(frames, 3e5)
        ctx.enable_timing(False)
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ 9. what merging is for
def test_merge_gives_one_box_per_object_and_fewer_tracks(pkg, ref_intended, synth):
    """30 ticks of the overlapping scene (every direction seen by two sensors at one height): separate detection gives many objects a
    second box; merged detection far fewer, and it spawns fewer tracks.  The second boxes merging leaves are not from the overlap: per
    object and tick the merged count equals the reference's on the vehicle's whole view with every elevated point twice (the merged
    cloud of this rig), where cells holding one return of the view become seeds of componentClustering's "more than one point" rule and
    can form an extra small component beside a sparse, far object (test_rig_merge_cpu.py)"""
    rig = overlap_rig(4)
    cfg = dict(seed=91, n_objects=30, rings=32, azimuths=900)
    ticks = list(overlap_ticks(synth, rig, 30, **cfg))
    views = [p for _, p in synth.frames(synth.SceneConfig(**cfg), 30)]           # the same renders, whole
    sep, mer = _merging(pkg, rig, _params(pkg), on=0), _merging(pkg, rig, _params(pkg))
    try:
        dup = dict(sep=0, mer=0)
        for f, ((ts, frames, pos, size), view) in enumerate(zip(ticks, views)):
            v, yaw = 0.0, 0.0                                         # the scene is rendered from a standing vehicle
            cs = boxes_per_object(sep.batch(frames, ts, v, yaw)["boxes"], pos, size)
            cm = boxes_per_object(mer.batch(frames, ts, v, yaw)["boxes"], pos, size)
            cd = boxes_per_object(doubled_view_detection(ref_intended, view), pos, size)
            assert np.array_equal(cm, cd), (f, cm, cd)
            dup["sep"] += int((cs > 1).sum()); dup["mer"] += int((cm > 1).sum())
        n_sep, n_mer = sep.tracker_num_tracks(), mer.tracker_num_tracks()
        print(f"30 ticks, 4 sensors: objects with a second box: separate {dup['sep']}, merged {dup['mer']} (= the doubled view's); "
              f"tracks spawned: separate {n_sep}, merged {n_mer}")
        assert dup["sep"] > 4 * max(dup["mer"], 1) and n_mer < n_sep, (dup, n_sep, n_mer)
    finally:
        sep.close(); mer.close()


# ------------------------------------------------------------------------------------------------ 10. the shared result ring
def test_frame_paths_after_merged_ticks(pkg, synth):
    """merged ticks fill every block of the context's result ring (result_ring 4, 10 ticks, the last one through
    lmot_batch_detect_dev); lmot_frame, lmot_frame_dev and lmot_track_step_lists_dev results that then land on those blocks equal a
    fresh twin's -- the merged ticks' per-sensor rows must not leak into their counts"""
    import torch
    rig = overlap_rig(4, heights=HEIGHTS[:4])
    ticks = list(overlap_ticks(synth, rig, 10, seed=101))
    views = [p for _, p in synth.frames(synth.SceneConfig(seed=102, rings=32, azimuths=900), 6)]
    ctx, twin = _merging(pkg, rig, _params(pkg, result_ring=4)), _merging(pkg, rig, _params(pkg, result_ring=4), on=0)
    ref = _merging(pkg, rig, _params(pkg))
    try:
        for f, (ts, frames, _, _) in enumerate(ticks[:9]):
            r, w = ctx.batch(frames, ts), ref.batch(frames, ts)
            assert _rows(r) == _rows(w) and r["boxes"].tobytes() == w["boxes"].tobytes(), f
        ts, frames, _, _ = ticks[9]
        d = [torch.from_numpy(p).cuda() for p in frames]
        torch.cuda.synchronize()
        ctx.batch_detect_dev([(t.data_ptr(), len(p)) for t, p in zip(d, frames)])
        r, w = ctx.batch_collect(), ref.batch(frames, ts)
        assert _rows(r) == _rows(w) and r["boxes"].tobytes() == w["boxes"].tobytes()
        assert sum(_rows(r)[0]) > 0 and len(_rows(r)) == 4
        ctx.tracker_reset()
        for f, view in enumerate(views):
            ts = 2e6 + 1e5 * f
            if f % 3 == 0:
                a, b = ctx.frame(view, ts), twin.frame(view, ts)
            elif f % 3 == 1:
                dv = torch.from_numpy(view).cuda()
                torch.cuda.synchronize()
                ctx.frame_dev(dv.data_ptr(), len(view), ts); twin.frame_dev(dv.data_ptr(), len(view), ts)
                a, b = ctx.frame_fetch(), twin.frame_fetch()
            else:
                lists = torch.from_numpy(np.stack([_some_boxes(f)] * 2)).cuda()
                cnt = torch.tensor([3, 2], dtype=torch.int32, device="cuda")
                torch.cuda.synchronize()
                ctx.track_step_lists_dev(lists.data_ptr(), cnt.data_ptr(), 2, 3, ts)
                twin.track_step_lists_dev(lists.data_ptr(), cnt.data_ptr(), 2, 3, ts)
                a, b = ctx.frame_fetch(), twin.frame_fetch()
                assert (a["n_elevated"], a["n_ground"], a["num_cluster"]) == (0, 0, 0), f
            assert (a["n_elevated"], a["n_ground"], a["num_cluster"]) == (b["n_elevated"], b["n_ground"], b["num_cluster"]), f
            _same(a, b, f)
    finally:
        for c in (ctx, twin, ref):
            c.close()
