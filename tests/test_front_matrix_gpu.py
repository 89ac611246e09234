"""The detection front end of sequence ticks across the configuration matrix of front_scenes: every combination of sensor table (none,
separate, merging), own detection values and deskew, mixed in one tick with LISTS entries, skips and a restart.

The front end picks its kernel variants tick-wide, as an OR over the tick's FRAMES streams (csrc/api.cu, detect_front and
seq_tick_common).  The contract is that a stream's outputs do not depend on what the other streams of its tick are.  Three checks:
  a. isolation: a context stepping the mixed ticks equals, bit for bit, a context with the same settings stepping each stream's entry
     of every tick alone (the others skip) -- counts, per-frame counts, boxes, every track field, track IDs and the track-table dump;
  b. the reference: per stream, the reference's detection of its configuration (deskewed clouds from test_deskew_gpu.deskew_np first)
     and the reference's tracker one stream at a time;
  c. the launch rule: the front-end kernels one tick launches, by name (torch.profiler in a child process), equal
     front_scenes.launch_rule for every distinct switch state of the matrix.
"""
import ctypes as C

import numpy as np
import pytest

import front_scenes as fs
from test_tracker_gpu import INTS, STATE, TOL, _pd_tracks, _rel_err

pytestmark = pytest.mark.gpu
f32 = np.float32
RING = 4
_STREAMS = {}


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8) if a.dtype.itemsize == 1 else a.view(f"u{a.dtype.itemsize}")


def _params(pkg, gf, max_points=1 << 16):
    p = pkg.default_params()
    p.max_points = max_points
    p.sensor_height = fs.H_VEHICLE
    p.global_frame = gf
    return p


def _streams(synth, key, layout, n_ticks, seed, sensors=None, view_seed=None):
    """the layout's streams, stream k from scene seed + 7 k (cached across parameters: the scenes are the costly part on the host);
    view_seed: the tableless stream of OVER_MAX, a 16-ring view"""
    if key not in _STREAMS:
        out = []
        for k, name in enumerate(layout):
            if view_seed is not None and name == "none":
                out.append(fs.Stream(synth, name, k, n_ticks, seed=view_seed, rings=16))
            else:
                out.append(fs.Stream(synth, name, k, n_ticks, seed=seed + 7 * k, n_sensors=sensors))
        _STREAMS[key] = out
    return _STREAMS[key]


def _layout_streams(synth, i):
    lay = fs.LAYOUTS[i]
    return _streams(synth, (i,), lay, len(fs.schedule(lay)), 300 + 31 * i)


def _configure(pkg, ctx, streams):
    """the streams' settings on an open set (identical for both contexts of a comparison)"""
    from rig_merge_scenes import table_kw
    for s in streams:
        if s.rig is not None:
            ctx.seq_set_sensors(s.k, **table_kw(s.rig))
            if s.table == "merge":
                ctx.seq_set_rig_merge(s.k, 1)
        if s.own:
            ctx.seq_set_detect_params(s.k, **fs.OWN)
        if s.dsk:
            ctx.seq_set_deskew(s.k, on=1)


def _entry(s, t, code, device, keep):
    """sequence s's entry at tick t for `code` (host arrays, or device copies kept alive in `keep`)"""
    v, yaw = s.ego(t)
    d = dict(timestamp=s.ts(t), v_gps=v, yaw_gps=yaw, restart=code == "R")
    tabled = s.rig is not None
    if code == "L":
        lists = s.lists_for(t)
        if not device:
            d["lists"] = lists if tabled else lists[0]
            return d
        import torch
        cap = max(len(x) for x in lists)
        buf = torch.zeros((len(lists), cap, 8, 3), dtype=torch.float32, device="cuda")
        for j, x in enumerate(lists):
            buf[j, : len(x)] = torch.from_numpy(x)
        cnt = torch.tensor([len(x) for x in lists], dtype=torch.int32, device="cuda")
        keep += [buf, cnt]
        d.update(lists=[buf.data_ptr() + j * cap * 96 for j in range(len(lists))], d_counts=cnt.data_ptr(), cap=cap)
        return d
    frames = s.frames_for(t, code)
    if device:
        import torch
        dev = []
        for p in frames:
            x = torch.from_numpy(np.ascontiguousarray(p)).cuda() if len(p) else None
            keep.append(x)
            dev.append((x.data_ptr() if x is not None else 0, len(p)))
        frames = dev
    d["frames"] = frames if tabled else frames[0]
    return d


def _snapshot(ctx, res, stepped):
    """a collected tick: per stepped sequence its result dict (copied), frame counts and track IDs"""
    out = {}
    for k in stepped:
        r = res[k]
        assert r is not None, k
        out[k] = ({key: np.array(v, copy=True) for key, v in r.items()}, ctx.seq_frame_counts(k), ctx.seq_track_ids(k))
    return out


def _collect(ctx):
    so, sets = ctx._seq_out(ctx.params.max_tracks)
    st = ctx.lib.lmot_seq_collect(ctx.h, C.byref(so))
    return st, ctx._seq_tick_result(so, sets)


class _Driver:
    """steps one context through ticks in one mode -- "sync" (lmot_seq_tick), "submit" (lmot_seq_tick_submit, RING ticks in flight)
    or "dev" (lmot_seq_tick_dev on float4 device frames and padded device lists) -- and records every tick's (status, snapshot) in
    submission order, through the raw calls so that an error status keeps its outputs"""

    def __init__(self, ctx, mode):
        self.ctx, self.mode, self.out, self.pending, self.keep = ctx, mode, [], [], []

    def tick(self, entries):
        c = self.ctx
        stepped = [k for k, e in enumerate(entries) if e is not None]
        if self.mode == "sync":
            arr, stride, keep = c._seq_entries(entries, False)
            so, sets = c._seq_out(c.params.max_tracks)
            st = c.lib.lmot_seq_tick(c.h, arr, len(entries), stride, C.byref(so))
            self.out.append((st, _snapshot(c, c._seq_tick_result(so, sets), stepped)))
            return
        if len(self.pending) == RING:
            self._collect_one()
        if self.mode == "submit":
            arr, stride, keep = c._seq_entries(entries, False)
            self.keep.append((arr, keep))
            st = c.lib.lmot_seq_tick_submit(c.h, arr, len(entries), stride)
        else:
            import torch
            torch.cuda.synchronize()
            arr, _, keep = c._seq_entries(entries, True)
            self.keep.append((arr, keep))
            st = c.lib.lmot_seq_tick_dev(c.h, arr, len(entries))
        assert st == 0, st
        self.pending.append(stepped)
        self.out.append(None)

    def _collect_one(self):
        stepped = self.pending.pop(0)
        st, res = _collect(self.ctx)
        self.out[self.out.index(None)] = (st, _snapshot(self.ctx, res, stepped))

    def finish(self):
        while self.pending:
            self._collect_one()
        return self.out


def _same_stream(a, b, what):
    """two snapshots of one stream's step bit for bit, and the per-frame rows agree with the step's totals (a merging rig reports the
    merged cloud's clusters and boxes in its row 0, behind nothing: rows written over by the concatenation break the sums)"""
    ra, fa, ia = a
    rb, fb, ib = b
    assert fa.sum(0)[1:].tolist() == [int(ra["n_ground"]), int(ra["num_cluster"]), len(ra["boxes"])], (what, fa)
    assert set(ra) == set(rb), what
    for key in ra:
        assert ra[key].shape == rb[key].shape and np.array_equal(_bits(ra[key]), _bits(rb[key])), (what, key)
    assert np.array_equal(fa, fb), (what, "frame counts", fa, fb)
    assert np.array_equal(ia, ib), (what, "track ids")


def _isolation(pkg, streams, key, ticks, gf, mode, max_points=1 << 16):
    """M steps the layout's mixed ticks; I steps every stepped entry of each tick as a tick of its own (the rest skip), in sequence
    order.  -> the number of (tick, stream) outputs compared"""
    S = len(streams)
    M, I = pkg.Lmot(_params(pkg, gf, max_points)), pkg.Lmot(_params(pkg, gf, max_points))
    try:
        for c in (M, I):
            c.seq_open(S, ring=RING)
            _configure(pkg, c, streams)
        dm, di = _Driver(M, mode), _Driver(I, mode)
        where = []                                     # (tick, stream) of every I tick
        for t, tk in enumerate(ticks):
            ent = [None if code == "-" else _entry(s, t, code, mode == "dev", dm.keep) for s, code in zip(streams, tk)]
            dm.tick(ent)
            for k, e in enumerate(ent):
                if e is not None:
                    di.tick([e if j == k else None for j in range(S)])
                    where.append((t, k))
            if mode == "sync":
                for k in range(S):
                    assert np.array_equal(_bits(M.seq_tracker_dump(k)), _bits(I.seq_tracker_dump(k))), (key, t, k, "dump")
        om, oi = dm.finish(), di.finish()
        n = 0
        for (t, k), (st_i, snap_i) in zip(where, oi):
            st_m, snap_m = om[t]
            # the tick's status: a capacity error belongs to the stream whose merged cloud was cut
            if st_i != 0:
                assert st_m == st_i, (key, t, k, st_m, st_i)
            _same_stream(snap_m[k], snap_i[k], (key, mode, gf, t, k, ticks[t]))
            n += 1
        for k in range(S):
            assert np.array_equal(_bits(M.seq_tracker_dump(k)), _bits(I.seq_tracker_dump(k))), (key, k, "dump")
        return n
    finally:
        M.close(); I.close()


@pytest.mark.parametrize("gf", [0, 1])
@pytest.mark.parametrize("mode", ["sync", "submit", "dev"])
def test_streams_are_isolated(pkg, synth, mode, gf):
    """Every layout of the matrix, mixed ticks against each stream stepped alone.  Catches a tick-wide switch taken from one group for
    all (the own-values OR read from group 0 only, the rig flag of box fitting dropped, CCL fused while a stream merges), a deskew
    table or count row indexed by stream instead of by frame (h_dsk / d_deskew by group, the merge unit's rows not behind its sensors'
    rows), the concatenation's row count taken from the header, and bank or merge-unit state leaking between the submitted ticks."""
    n = 0
    for i, lay in enumerate(fs.LAYOUTS):
        n += _isolation(pkg, _layout_streams(synth, i), (i,), fs.schedule(lay), gf, mode)
    assert n > 200, n


@pytest.mark.parametrize("mode", ["sync", "submit", "dev"])
def test_merged_cloud_above_max_points_is_isolated(pkg, synth, mode):
    """A 7-sensor merging rig whose merged cloud is cut at max_points next to a tableless stream: the capacity error and the cut cloud's
    outputs are the same whether the merging stream steps with the other one or alone, and the tableless stream is unaffected."""
    o = fs.OVER_MAX
    streams = _streams(synth, ("over",), o["layout"], len(o["ticks"]), o["seed"], o["sensors"], o["view_seed"])
    biggest = max(len(p) for s in streams if s.rig for fr in s.frames for p in fr)
    mp = biggest + 64
    total = sum(len(p) for p in streams[0].frames[0])
    assert total > mp + 1000 and max(len(fr[0]) for fr in streams[1].frames) <= mp, (total, mp)
    n = _isolation(pkg, streams, ("over",), o["ticks"], 0, mode, max_points=mp)
    assert n == sum(c != "-" for tk in o["ticks"] for c in tk)


# ------------------------------------------------------------------------------------------------ b. against the reference
REF_LAYOUTS = [0, 2, 4, 8]             # layouts whose streams cover every configuration the reference expresses (see the docstring)
REF_TICKS = 6


def _ref_detection(ref, ref_dt, pkg, s, frames, prev):
    """the reference's (rows, vehicle-frame boxes) for stream s's frames; prev: the stream's previous (stamp, yaw) for deskew's omega"""
    from rig_merge_scenes import merged_detection
    from test_deskew_gpu import deskew_np, omega_of
    from test_sensor_rig_gpu import expected_detection
    clouds = frames
    if s.dsk:
        t = prev[2]
        v, yaw = s.ego(t)
        om = omega_of(prev[:2] if prev[0] is not None else None, (s.ts(t), yaw))
        mounts = [p for p, _, _ in s.rig] if s.rig else [None]
        clouds = [deskew_np(pkg, P, v, om, m) for P, m in zip(frames, mounts)]
    clouds = [np.ascontiguousarray(c[:, :3]) for c in clouds]
    if s.table == "none":
        if s.own:
            with ref_dt.detect_params(fs.OWN):
                e, g = ref_dt.ground_remove(clouds[0])
                grid, k = ref_dt.component_clustering(e)
                b, _ = ref_dt.box_fitting(e, grid, k)
        else:
            e, g = ref.ground_remove(clouds[0])
            grid, k = ref.component_clustering(e)
            b, _ = ref.box_fitting(e, grid, k)
        return [(len(e), len(g), k, len(b))], np.asarray(b, f32).reshape(-1, 8, 3)
    if s.table == "sep":
        [(per, vlist)] = expected_detection(ref, [(p, h) for p, h, _ in s.rig], [(0.0, clouds)])
        return per, vlist.reshape(-1, 8, 3)
    rows, b, _, _ = merged_detection(ref, s.rig, clouds, fs.H_VEHICLE)
    return rows, np.asarray(b, f32).reshape(-1, 8, 3)


def test_streams_against_the_reference(pkg, synth, ref_intended):
    """Mixed all-FRAMES ticks of five layouts; each stream against the reference's detection of its own configuration and the
    reference's tracker stepped through that stream alone (tracker_reset between streams).  Bars: per-frame counts and boxes bit-exact,
    identical trackManage / static / visible flags and table integers, targets and UKF states within 1e-4 relative on positive-definite
    filters.  Catches a stream detected with another stream's values, mount or deskew table in a way (a) cannot see because both
    contexts share it, e.g. a setting dropped for every tick alike.
    A stream with its own values AND a sensor table has no single reference call (the reference has one set of globals, the library
    folds each sensor's four mount values over the stream's own); such streams are left to (a) and to the twin tests
    test_seq_detect_params_gpu.test_sensor_table_on_top_of_own_values and test_rig_merge_gpu.test_merge_with_own_detect_params_and_deskew."""
    from oracle import ref_detect_tunable
    ref = ref_intended
    ref_dt = ref_detect_tunable.RefDetectTunable() if ref_detect_tunable.have_ref("detect_tunable") else None
    covered = set()
    for i in REF_LAYOUTS:
        lay = fs.LAYOUTS[i]
        streams = _streams(synth, ("ref", i), lay, REF_TICKS, 900 + 31 * i)
        ctx = pkg.Lmot(_params(pkg, 0))
        try:
            ctx.seq_open(len(streams), ring=RING)
            _configure(pkg, ctx, streams)
            got = []
            for t in range(REF_TICKS):
                res = ctx.seq_tick([_entry(s, t, "F", False, []) for s in streams])
                got.append([(res[k], ctx.seq_frame_counts(k)) for k in range(len(streams))])
            for k, s in enumerate(streams):
                if s.own and s.rig is not None:
                    continue
                if s.own and ref_dt is None:
                    continue
                covered.add(s.name)
                ref.tracker_reset()
                prev = (None, None, 0)
                n_boxes = 0
                for t in range(REF_TICKS):
                    rows, boxes = _ref_detection(ref, ref_dt, pkg, s, s.frames[t], (prev[0], prev[1], t))
                    prev = (s.ts(t), s.ego(t)[1], t)
                    r, fc = got[t][k]
                    assert [tuple(int(x) for x in row) for row in fc] == [tuple(x) for x in rows], (i, s.name, t)
                    assert r["boxes"].shape == boxes.shape and np.array_equal(_bits(r["boxes"]), _bits(boxes)), (i, s.name, t)
                    n_boxes += len(boxes)
                    a = ref.tracker_step(boxes, s.ts(t), *s.ego(t))
                    for key in ("track_manage", "is_static", "is_vis"):
                        assert np.array_equal(r[key], a[key]), (i, s.name, t, key)
                    np.testing.assert_allclose(r["targets"], a["targets"], rtol=1e-4, atol=1e-4)
                assert n_boxes > 0, (i, s.name)
                da, db = ref.tracker_dump(), ctx.seq_tracker_dump(k)
                assert da.shape == db.shape and np.array_equal(da[:, INTS], db[:, INTS]), (i, s.name)
                ok = _pd_tracks(da)
                err = _rel_err(da[ok][:, STATE], db[ok][:, STATE])
                assert err.size == 0 or err.max() < TOL, (i, s.name, float(err.max()))
        finally:
            ctx.close()
    want = {n for n, c in fs.CONFIGS.items() if not (c["own"] and c["table"] != "none")}
    if ref_dt is None:
        want = {n for n in want if not fs.CONFIGS[n]["own"]}
    assert want <= covered, want - covered


# ------------------------------------------------------------------------------------------------ c. the launch rule
_NAMES_SCRIPT = r"""
import importlib, json, sys
import torch
from torch.profiler import ProfilerActivity, profile
sys.path[:0] = sys.argv[1:3]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
import front_scenes as fs
import test_front_matrix_gpu as T
out = []
for (sw, empty), (i, t, gf) in sorted(fs.switch_states().items(), key=lambda x: x[1]):
    ticks = fs.schedule(fs.LAYOUTS[i])
    streams = T._layout_streams(synth, i)
    ctx = pkg.Lmot(T._params(pkg, gf))
    ctx.seq_open(len(streams), ring=T.RING)
    T._configure(pkg, ctx, streams)
    ent = lambda: [None if c == "-" else T._entry(s, t, c, False, []) for s, c in zip(streams, ticks[t])]
    ctx.seq_tick(ent())
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.seq_tick(ent())
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if str(e.device_type).endswith("CUDA")]
    out.append(dict(layout=i, tick=t, gf=gf, names=sorted(k for k in map(fs.kernel_key, names) if k)))
    ctx.close()
print(json.dumps(out))
"""


def test_launches_follow_the_rule():
    """For every distinct switch state of the matrix (and all-empty ticks), the front-end kernels of one tick by name equal
    front_scenes.launch_rule.  Catches a wrong tick-wide switch directly: the own-values OR, the rig flag of box fitting (a merge-only
    tick runs box_fit_kernel<..., false>, merge next to a separate rig <..., true>), a CCL fused or launched twice, deskew launched for
    a tick without a deskewing stream, the concatenation skipped or issued without a table, and the segment pass of empty ticks."""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _NAMES_SCRIPT, os.path.dirname(here), here], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    runs = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(runs) == len(fs.switch_states())
    kinds = set()
    for run in runs:
        lay = fs.LAYOUTS[run["layout"]]
        cf, empty, lists = fs.tick_cfgs(lay, fs.schedule(lay)[run["tick"]])
        want = fs.launch_rule(cf, run["gf"], empty, lists)
        assert run["names"] == want, (run, cf, want)
        s = fs.switches(cf, run["gf"])
        if s["merging"] and not s["own_det"]:
            kinds.add("box_fit_kernel<true>" if s["rig_fit"] else "box_fit_kernel<false>")
    assert kinds == {"box_fit_kernel<true>", "box_fit_kernel<false>"}, kinds
