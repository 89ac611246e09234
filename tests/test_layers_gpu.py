"""Layered clustering on the device (include/lmot.h, lmot_set_layers): off is today's path, one slice is the unlayered pipeline bit for bit,
the device's per-point clusters equal the NumPy restatement (tests/layer_scenes.py) and its boxes the per-cluster reference oracle, next
to every other front-end setting, across setting changes in flight and in every size regime where the kernels switch paths."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import layer_scenes as ls

pytestmark = pytest.mark.gpu
f32 = np.float32
AREA = [np.array([[-30.0, -30.0], [30.0, -30.0], [30.0, 8.0], [-30.0, 12.0]])]


def _params(pkg, gf=0, rule=0, max_points=1 << 17, **kw):
    p = pkg.default_params()
    p.max_points = max_points
    p.global_frame = gf
    p.rule_filter = rule
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _bits(a):
    return np.ascontiguousarray(a, f32).view(np.uint32)


def _same(a, b, keys=("targets", "vandyaw", "track_manage", "is_static", "is_vis", "vis_bb")):
    for k in ("n_elevated", "n_ground", "num_cluster", "n_boxes"):
        if k in a:
            assert a[k] == b[k], k
    assert np.array_equal(_bits(a["boxes"]), _bits(b["boxes"]))
    for k in keys:
        if k in a:
            assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), k


def _frames(synth, n, seed=5, rings=32, azimuths=900):
    return [(ts, p) for ts, p in synth.frames(synth.SceneConfig(seed=seed, rings=rings, azimuths=azimuths, n_objects=30), n)]


def _ref(mode="intended"):
    from oracle import ref
    if not ref.have_ref(mode):
        pytest.skip("oracle/_ref not built")
    return ref.RefOracle(mode)


# ------------------------------------------------------------------------------------------------ today's path
_NAMES_SCRIPT = r"""
import importlib, json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
sys.path[:0] = sys.argv[1:3]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
P = [p for _, p in synth.frames(synth.SceneConfig(seed=5, rings=32, azimuths=900), 1)][0]
out = {}
for arm in ("off", "on_then_off", "on", "mixed"):
    p = pkg.default_params(); p.max_points = 1 << 16
    ctx = pkg.Lmot(p)
    ctx.seq_open(4, ring=4)
    if arm in ("on_then_off", "on"):
        ctx.set_layers(on=1); ctx.seq_set_layers(1, on=1, n_slices=8)
    if arm == "on_then_off":
        ctx.set_layers(); ctx.seq_set_layers(1)
    if arm == "mixed":
        ctx.seq_set_layers(1, on=1)
    d = torch.from_numpy(P).cuda(); torch.cuda.synchronize()
    def run(t):
        if arm != "mixed":
            ctx.frame(P, t)
            ctx.frame_dev(d.data_ptr(), len(P), t + 1e5); ctx.frame_fetch()
            ctx.batch([P, P], t + 2e5)
        ctx.seq([P] * 4, [t] * 4)
        torch.cuda.synchronize()
    run(1e6)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(2e6)
    out[arm] = [e.name for e in prof.events() if str(e.device_type).endswith("CUDA")]
    ctx.close()
print(json.dumps(out))
"""


def test_off_is_todays_path(pkg, synth):
    """layers set and cleared again leave the same kernels, copies and memsets; a layered submission runs layer_mark_kernel and
    ccl_layer_kernel, and the layered units' box fitting starts with tile_hist_layers_kernel; a set cleared again gives identical results"""
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _NAMES_SCRIPT, os.path.dirname(here), here], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    n = json.loads(r.stdout.strip().splitlines()[-1])
    assert n["off"] and not any("layer" in x for x in n["off"]), n["off"]
    assert sorted(n["off"]) == sorted(n["on_then_off"])
    for name in ("layer_mark_kernel", "ccl_layer_kernel", "tile_hist_layers_kernel"):
        assert sum(name in x for x in n["on"]) == 4, name        # frame, frame_dev, batch, one tick
        assert sum(name in x for x in n["mixed"]) == 1, name
    # the tick where one of four sequences is layered still clusters the other three in ccl_dense_kernel
    assert sum("ccl_dense_kernel" in x for x in n["mixed"]) == 1
    a, b = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        b.set_layers(on=1, n_slices=4, gap_slices=1)
        b.set_layers()
        assert b.get_layers() == ls_defaults()
        for ts, p in _frames(synth, 4):
            _same(a.frame(p, ts), b.frame(p, ts))
    finally:
        a.close(); b.close()


def ls_defaults():
    return {"on": 0, "n_slices": 32, "slice_m": 0.2, "z_min": -0.5, "gap_slices": 2}


# ------------------------------------------------------------------------------------------------ one slice is the unlayered pipeline
@pytest.mark.parametrize("gf", [0, 1])
def test_one_slice_is_off(pkg, synth, gf):
    """S = 1 (any slice size, origin and g = 0) reproduces layers off bit for bit: lmot_frame, pipelined _submit / _collect,
    lmot_frame_dev, lmot_batch and a sequence tick, every output and the tracker dump"""
    import torch
    frames = _frames(synth, 6, seed=9, rings=64, azimuths=1800)
    one = dict(on=1, n_slices=1, slice_m=0.37, z_min=-3.0, gap_slices=0)
    ctx = [pkg.Lmot(_params(pkg, gf, pipeline_depth=4)) for _ in range(2)]
    try:
        ctx[1].set_layers(**one)
        # lmot_frame
        for ts, p in frames:
            _same(ctx[0].frame(p, ts), ctx[1].frame(p, ts))
        assert np.array_equal(ctx[0].tracker_dump(), ctx[1].tracker_dump())
        assert len(ctx[1].debug_point_clusters()) == 1 and ctx[0].debug_point_clusters() == []
        # pipelined submission, depth 3
        for c in ctx:
            c.tracker_reset()
        res = [[], []]
        for i, (ts, p) in enumerate(frames):
            for j, c in enumerate(ctx):
                c.frame_submit(p, ts + 1e7)
                if i >= 2:
                    res[j].append(c.frame_collect())
        for j, c in enumerate(ctx):
            while c.frames_in_flight():
                res[j].append(c.frame_collect())
        for a, b in zip(*res):
            _same(a, b)
        # device frames
        for c in ctx:
            c.tracker_reset()
        for ts, p in frames:
            d = torch.from_numpy(np.ascontiguousarray(p)).cuda()
            torch.cuda.synchronize()
            out = []
            for c in ctx:
                c.frame_dev(d.data_ptr(), len(p), ts + 2e7)
                out.append(c.frame_fetch())
            _same(*out)
        assert np.array_equal(ctx[0].tracker_dump(), ctx[1].tracker_dump())
        # batched ticks of two frames
        for c in ctx:
            c.tracker_reset()
        for i in range(len(frames) - 1):
            ts = frames[i][0] + 3e7
            _same(ctx[0].batch([frames[i][1], frames[i + 1][1]], ts), ctx[1].batch([frames[i][1], frames[i + 1][1]], ts))
        # a sequence tick: sequence 1 layered at S = 1 against sequence 0 off
        ctx[0].seq_open(2, ring=2)
        ctx[0].seq_set_layers(1, **one)
        for ts, p in frames:
            r = ctx[0].seq([p, p], [ts, ts])
            _same(r[0], r[1])
        assert np.array_equal(ctx[0].seq_tracker_dump(0), ctx[0].seq_tracker_dump(1))
    finally:
        for c in ctx:
            c.close()


# ------------------------------------------------------------------------------------------------ against the oracle
@pytest.mark.parametrize("rule", [0, 1])
@pytest.mark.parametrize("sensor", ["64", "32"])
def test_canopy_scene_against_oracle(pkg, sensor, rule):
    """per-point clusters equal the NumPy restatement; counts and boxes equal the per-cluster reference oracle bit for bit; the tracker
    on them equals the reference's"""
    ground = _ref()
    fitter = _ref("o2" if rule else "intended")
    pts, objects = ls.render(sensor)
    ctx = pkg.Lmot(_params(pkg, 0, rule))
    try:
        ctx.set_layers(on=1)
        fitter.tracker_reset()
        for i in range(3):
            ts = 1e6 + i * 1e5
            e, _ = ground.ground_remove(pts)
            ids, k = ls.point_clusters(e)
            want = ls.oracle_boxes(fitter, e, ids, k)
            r = ctx.frame(pts, ts)
            assert (r["n_elevated"], r["num_cluster"]) == (len(e), k)
            dev = ctx.debug_point_clusters()
            assert len(dev) == 1 and np.array_equal(dev[0], ids)
            assert np.array_equal(_bits(r["boxes"]), _bits(want))
            if rule == 0:
                w = fitter.tracker_step(want, ts)
                assert np.array_equal(r["track_manage"], w["track_manage"])
                assert np.allclose(r["targets"], w["targets"], rtol=1e-4, atol=1e-4)
        # the cars under canopies the CPU test pins for the reference oracle (both rule modes box the same clusters' points)
        assert ls.found(r["boxes"], objects, "car_canopy") == ls.found(want, objects, "car_canopy") >= 2
    finally:
        ctx.close()


@pytest.mark.parametrize("layers", [dict(n_slices=8, slice_m=0.5, gap_slices=0), dict(n_slices=32, gap_slices=5, z_min=0.3),
                                    dict(n_slices=17, slice_m=0.13, gap_slices=16)])
def test_settings_against_oracle(pkg, synth, layers):
    ground = _ref()
    ctx = pkg.Lmot(_params(pkg))
    try:
        ctx.set_layers(on=1, **layers)
        for ts, p in _frames(synth, 2, seed=4, rings=64, azimuths=1800):
            e, _ = ground.ground_remove(p)
            ids, k = ls.point_clusters(e, **layers)
            r = ctx.frame(p, ts)
            assert r["num_cluster"] == k
            assert np.array_equal(ctx.debug_point_clusters()[0], ids)
            assert np.array_equal(_bits(r["boxes"]), _bits(ls.oracle_boxes(ground, e, ids, k)))
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------ with every other front-end setting
def _setting(ctx, k, which):
    """stream k (None: the context's own) with layers on and `which`"""
    own = k is None
    call = (lambda name, *a, **kw: getattr(ctx, name)(*a, **kw)) if own else (lambda name, *a, **kw: getattr(ctx, "seq_" + name)(k, *a, **kw))
    call("set_layers", on=1, gap_slices=1)
    if which == "search":
        call("set_box_search", on=1, n_angles=90)
    elif which == "lines":
        call("set_ground_lines", on=1)
    elif which == "area":
        call("set_detect_area", AREA)
    elif which == "acc":
        call("set_accumulate", sweeps=3)
    elif which == "deskew":
        call("set_deskew", on=1)
    elif which == "off":
        call("set_layers")


WHICH = ["plain", "search", "lines", "area", "acc", "deskew", "off"]


def test_sequences_with_other_settings(pkg, synth):
    """seven sequences, each layered next to another front-end setting (and one off), equal twin contexts stepped with lmot_frame"""
    frames = _frames(synth, 5, seed=12)
    S = len(WHICH)
    ctx = pkg.Lmot(_params(pkg))
    twins = [pkg.Lmot(_params(pkg)) for _ in range(S)]
    try:
        ctx.seq_open(S, ring=2)
        for k, w in enumerate(WHICH):
            _setting(ctx, k, w)
            _setting(twins[k], None, w)
        for i, (ts, p) in enumerate(frames):
            r = ctx.seq([p] * S, [ts] * S, v_gps=[2.0] * S, yaw_gps=[0.01 * i] * S)
            for k in range(S):
                _same(r[k], twins[k].frame(p, ts, 2.0, 0.01 * i))
    finally:
        ctx.close()
        for t in twins:
            t.close()


@pytest.mark.parametrize("merge", [False, True])
def test_rigs(pkg, synth, merge):
    """a two-sensor rig, separate and merging: every unit layered with its sensor's (or the vehicle's) sensor_height; the batched tick
    equals lmot_batch with layers at S = 1 set on a twin off, and at S = 32 each unit's ids equal the restatement on its cloud"""
    frames = _frames(synth, 3, seed=21)
    poses = [np.array([[1, 0, 0, 0.5], [0, 1, 0, 0.0], [0, 0, 1, 0.1]], f32), np.array([[1, 0, 0, -0.5], [0, 1, 0, 0.2], [0, 0, 1, 0.0]], f32)]
    a, b = pkg.Lmot(_params(pkg)), pkg.Lmot(_params(pkg))
    try:
        for c in (a, b):
            c.set_sensors(poses, sensor_height=[1.63, 1.73])
            c.set_rig_merge(merge)
        b.set_layers(on=1, n_slices=1, gap_slices=0)
        for ts, p in frames:
            _same(a.batch([p, p[::2]], ts), b.batch([p, p[::2]], ts))
        b.set_layers(on=1)
        b.batch([frames[0][1], frames[1][1]], 5e6)
        units = b.debug_point_clusters()
        assert len(units) == (1 if merge else 2)
        assert all(len(u) > 1000 and u.max() > 0 for u in units)
    finally:
        a.close(); b.close()


# ------------------------------------------------------------------------------------------------ changes in flight
def test_changes_in_flight(pkg, synth):
    """switching on and off on the same slots while frames are in flight: every frame equals the twin that always had its setting
    (stale bit planes, label grid or column masks would show)"""
    frames = _frames(synth, 10, seed=17, rings=64, azimuths=1800)
    sw = pkg.Lmot(_params(pkg, pipeline_depth=2))
    on, off = pkg.Lmot(_params(pkg, pipeline_depth=2)), pkg.Lmot(_params(pkg, pipeline_depth=2))
    try:
        on.set_layers(on=1)
        got, want = [], []
        for i, (ts, p) in enumerate(frames):
            layered = (i // 2) % 2 == 0 if i < 6 else i % 2 == 1
            if layered:
                sw.set_layers(on=1)
            else:
                sw.set_layers()
            sw.frame_submit(p, ts)
            if sw.frames_in_flight() >= 3:
                got.append(sw.frame_collect())
            on.tracker_reset(); off.tracker_reset()
            want.append((on if layered else off).frame(p, ts))
        while sw.frames_in_flight():
            got.append(sw.frame_collect())
        for a, b in zip(got, want):
            _same(a, b, keys=())
    finally:
        sw.close(); on.close(); off.close()


# ------------------------------------------------------------------------------------------------ size regimes
def test_empty_cloud(pkg):
    ctx = pkg.Lmot(_params(pkg))
    try:
        ctx.set_layers(on=1)
        r = ctx.frame(np.zeros((0, 4), f32), 1e6)
        assert (r["n_elevated"], r["num_cluster"], len(r["boxes"])) == (0, 0, 0)
        assert [len(u) for u in ctx.debug_point_clusters()] == [0]
    finally:
        ctx.close()


def test_every_column_sixteen_runs(pkg):
    """every column of the grid holds a seed in every other slice: 62,500 columns x 16 runs, about a million nodes"""
    xs = (np.arange(250) + 0.5) * 0.2 - 25.0
    X, Y = np.meshgrid(xs, xs, indexing="ij")
    z = -2.0 + 1.0 + (np.arange(16) * 2 + 0.5) * 0.2           # slices 0, 2, .., 30 from z_min = 1 m above the flat ground
    pts = np.stack(np.broadcast_arrays(X[..., None], Y[..., None], z[None, None, :]), -1).reshape(-1, 3)
    pts = np.concatenate([pts, pts + np.array([0.01, 0.0, 0.0])]).astype(f32)
    ground = _ref()
    ctx = pkg.Lmot(_params(pkg, max_points=1 << 21))
    try:
        ctx.set_layers(on=1, gap_slices=0, z_min=1.0)
        e, _ = ground.ground_remove(pts)
        ids, k = ls.point_clusters(e, gap_slices=0, z_min=1.0)
        r = ctx.frame(pts, 1e6)
        assert r["n_elevated"] == len(e) and r["num_cluster"] == k
        assert np.array_equal(ctx.debug_point_clusters()[0], ids)
        xi, yi, _ = ls.columns(e)
        assert len(set(zip(xi.tolist(), yi.tolist()))) > 60000 and k >= 8
    finally:
        ctx.close()


def test_max_clusters(pkg):
    """num_cluster just below and just above max_clusters: all boxes, then LMOT_ERR_CAPACITY"""
    ground = _ref()
    pts, _ = ls.render("64")
    e, _ = ground.ground_remove(pts)
    ids, k = ls.point_clusters(e)
    want = ls.oracle_boxes(ground, e, ids, k)
    for mc, ok in ((k, True), (k - 1, False)):
        ctx = pkg.Lmot(_params(pkg, max_clusters=mc))
        try:
            ctx.set_layers(on=1)
            if ok:
                r = ctx.frame(pts, 1e6)
                assert r["num_cluster"] == k and np.array_equal(_bits(r["boxes"]), _bits(want))
            else:
                with pytest.raises(pkg.LmotError) as ei:
                    ctx.frame(pts, 1e6)
                assert ei.value.status == pkg.ERR_CAPACITY
        finally:
            ctx.close()


# ------------------------------------------------------------------------------------------------ validation, timing mode, debug getters
def test_validation_and_state(pkg, synth):
    ctx = pkg.Lmot(_params(pkg))
    try:
        good = dict(on=1, n_slices=8, slice_m=0.25, z_min=-1.0, gap_slices=3)
        ctx.set_layers(**good)
        for bad in (dict(on=2), dict(n_slices=0), dict(n_slices=33), dict(slice_m=0.0), dict(slice_m=float("nan")),
                    dict(z_min=float("inf")), dict(gap_slices=-1), dict(gap_slices=8)):
            with pytest.raises(pkg.LmotError) as ei:
                ctx.set_layers(**{**good, **bad})
            assert ei.value.status == pkg.ERR_INVALID
            assert ctx.get_layers() == good
        with pytest.raises(pkg.LmotError):
            ctx.seq_set_layers(0, on=1)                     # no open set
        ctx.seq_open(2, ring=2)
        assert ctx.seq_get_layers(1) == ls_defaults()
        with pytest.raises(pkg.LmotError):
            ctx.seq_set_layers(2, on=1)
        ctx.seq_set_layers(1, **good)
        assert ctx.seq_get_layers(1) == good
        ctx.seq_open(2, ring=2)
        assert ctx.seq_get_layers(1) == ls_defaults()         # lmot_seq_open turns it off
        (ts, p), = _frames(synth, 1)
        ctx.frame(p, ts)
        for call in (lambda: ctx.cluster_outputs(), lambda: ctx.debug_label_grid()):
            with pytest.raises(pkg.LmotError) as ei:
                call()
            assert ei.value.status == pkg.ERR_STATE
        ctx.set_layers()
        ctx.frame(p, ts + 1e5)
        ctx.debug_label_grid()
        assert ctx.debug_point_clusters() == []
        ctx.set_layers(on=1)
        ctx.enable_timing(True)
        with pytest.raises(pkg.LmotError) as ei:
            ctx.frame(p, ts + 2e5)
        assert ei.value.status == pkg.ERR_STATE
    finally:
        ctx.close()
