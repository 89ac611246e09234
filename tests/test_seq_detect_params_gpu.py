"""Per-sequence detection parameters (lmot_seq_set_detect_params): each sequence of lmot_seq with its own ground-removal, clustering and
box-fitting values.

Contract (include/lmot.h): sequence k given values p gives bit for bit what a twin context gives that was created with the same
lmot_params except that its detection fields are p -- through lmot_frame without a sensor table, through lmot_set_sensors + lmot_batch
with one.  The twins are test_seq_rig_gpu's (_Twin, _run, _same_tables); a sequence's values go into its twin's lmot_params.  The
reference anchors the values themselves: oracle/_ref/libref_detect_tunable.so, the reference with its two detection literals
(ground tolerance, minimum cluster size) as globals, all its detection globals (rMin, roiM, ramPoints, ...) set through ctypes.
"""
import ctypes as C

import numpy as np
import pytest

from test_ground_gpu import _check_frame
from test_seq_rig_gpu import _RigSeq, _Twin, _bits, _params, _run, _same_tables
from test_sensor_rig_gpu import RIG
from test_tracker_gpu import INTS, STATE, TOL, _pd_tracks, _rel_err

pytestmark = pytest.mark.gpu
f32 = np.float32
N_TICKS = 30

# object_tracking0's values (its ground_removal.cpp / box_fitting.cpp / component_clustering.cpp)
OT0 = dict(t_hmin=-1.9, t_hmax=-1.0, h_sensor=1.73, roi_m=30.0, l_slope_dist=3, l_num_points=300, sensor_height=1.73,
           t_height_min=1.0, t_width_min=0.25, t_len_min=0.5, t_ratio_min=1.3, t_ratio_max=5.0, min_cluster_points=100)
# a short-range sparse sensor: 50 m window, few points per cluster, more L-shape draws than a batched box-fitting CTA has threads
SPARSE = dict(r_min=2.0, r_max=50.0, roi_m=40.0, t_pt_per_m3=2.0, ram_points=300, l_num_points=3, t_hdiff=0.3)
# every field of the reference's own globals moved; LITERALS moves the two that are literals in the reference
ALL_MOVED = dict(r_min=2.5, r_max=80.0, t_hmin=-2.2, t_hmax=-0.5, t_hdiff=0.35, h_sensor=1.9, roi_m=44.0, ram_points=120, l_slope_dist=2,
                 l_num_points=7, sensor_height=1.9, t_height_min=0.7, t_height_max=2.8, t_width_min=0.15, t_width_max=3.8, t_len_min=0.25,
                 t_len_max=12.0, t_area_max=24.0, t_ratio_min=1.1, t_ratio_max=7.0, min_len_ratio=2.5, t_pt_per_m3=6.0)
LITERALS = dict(ground_tolerance=0.3, min_cluster_points=12)
PREFILTER = dict(node_prefilter=1, filter_x_min=-40.0, filter_x_max=40.0, filter_y_min=-30.0, filter_y_max=30.0)
COMPAT = dict(rule_filter=1, t_height_min=0.6)
EIGHT = [None, OT0, SPARSE, {**ALL_MOVED, **LITERALS}, PREFILTER, COMPAT, dict(r_min=10.0, r_max=40.0, roi_m=60.0),
         dict(ram_points=1024, l_slope_dist=0, l_num_points=2, min_cluster_points=8)]


def _twin_params(pkg, values, global_frame=0):
    p = _params(pkg, global_frame=global_frame)
    if values:
        for k, v in values.items():
            setattr(p, k, v)
    return p


@pytest.fixture(scope="module")
def ref_dt():
    from oracle import ref_detect_tunable
    if not ref_detect_tunable.have_ref("detect_tunable"):
        pytest.skip("oracle/_ref/libref_detect_tunable.so not built (needs the reference checkout)")
    return ref_detect_tunable.RefDetectTunable()


def _seq_ctx(pkg, S, gf=0):
    ctx = pkg.Lmot(_params(pkg, global_frame=gf))
    ctx.seq_open(S, ring=32)
    return ctx


_NAMES_SCRIPT = r"""
import importlib, json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
sys.path[:0] = sys.argv[1:3]
pkg = importlib.import_module("3d-lidar-multi-object-tracking_b200")
synth = importlib.import_module("3d-lidar-multi-object-tracking_b200.synth")
frames = [p for _, p in synth.frames(synth.SceneConfig(seed=5, rings=32, azimuths=900), 1)] * 8
out = {}
for arm in ("default", "own"):
    p = pkg.default_params(); p.max_points = 1 << 16
    ctx = pkg.Lmot(p); ctx.seq_open(8, ring=4)
    if arm == "own":
        for k in range(8):
            ctx.seq_set_detect_params(k, **pkg.default_detect_params(ctx.params))
    ctx.seq(frames, [1e6] * 8)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.seq(frames, [1.1e6] * 8)
        torch.cuda.synchronize()
    out[arm] = [e.name for e in prof.events() if "ground_fused" in e.name or "box_fit" in e.name]
    ctx.close()
print(json.dumps(out))
"""


def _kernel_names():
    """names of the ground and box-fitting kernels one S = 8 tick launches, without and with every sequence given lmot_params' own
    values (torch.profiler, in a process of its own: profiler sessions in the test process disturb later tests' sessions)"""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-c", _NAMES_SCRIPT, os.path.dirname(here), here], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_defaults_are_todays_path(pkg, synth):
    """Catches an override path taken with no override set, and a per-frame variant that misreads a field of lmot_params' own values:
    a set given lmot_default_detect_params(ctx params) explicitly must run the frame variants with the same outputs and tables."""
    names = _kernel_names()
    assert names["default"] and not any("frame_kernel" in n for n in names["default"]), names
    assert any("ground_fused_frame_kernel" in n for n in names["own"]) and any("box_fit_frame_kernel" in n for n in names["own"]), names
    S = 8
    seqs = [_RigSeq(synth, k, None, n_ticks=10) for k in range(S)]
    a, b = _seq_ctx(pkg, S), _seq_ctx(pkg, S)
    try:
        for k in range(S):
            b.seq_set_detect_params(k, **pkg.default_detect_params(b.params))
            assert b.seq_get_detect_params(k) == pkg.default_detect_params(b.params)
        for f in range(10):
            entries = [s.frames[f][0] for s in seqs]
            ts = [s.ts(f) for s in seqs]
            v = [s.ego(f)[0] for s in seqs]
            y = [s.ego(f)[1] for s in seqs]
            ra, rb = [a.seq(entries, ts, v, y)], [b.seq(entries, ts, v, y)]
            for k in range(S):
                for key in ("n_elevated", "n_ground", "num_cluster", "boxes", "targets", "vandyaw", "track_manage", "vis_bb"):
                    assert np.array_equal(_bits(np.asarray(ra[0][k][key])), _bits(np.asarray(rb[0][k][key]))), (f, k, key)
                assert np.array_equal(a.seq_frame_counts(k), b.seq_frame_counts(k))
        for k in range(S):
            assert np.array_equal(_bits(a.seq_tracker_dump(k)), _bits(b.seq_tracker_dump(k))), k
    finally:
        a.close(); b.close()


@pytest.mark.parametrize("mode", ["sync", "dev"])
@pytest.mark.parametrize("gf", [0, 1])
def test_eight_sets_match_twin_contexts(pkg, synth, gf, mode):
    """Catches a frame reading another frame's entry, a field dropped between lmot_detect_params and the kernels' blocks (each set
    moves different fields: range window, ROI, L-shape gates, ram_points on both sides of the CTA size and at the bound, the rule
    window and mode, the literals, the node pre-filter), and values that leak into the following tick.  30 ticks."""
    S = len(EIGHT)
    seqs = [_RigSeq(synth, k, None, n_ticks=N_TICKS) for k in range(S)]
    ctx = _seq_ctx(pkg, S, gf)
    twins = [_Twin(pkg, _twin_params(pkg, vals, gf), None) for vals in EIGHT]
    try:
        for k, vals in enumerate(EIGHT):
            if vals:
                ctx.seq_set_detect_params(k, **vals)
        _run(ctx, seqs, lambda f: [None] * S, N_TICKS, mode, twins)
        _same_tables(ctx, twins, (gf, mode))
    finally:
        ctx.close()
        for t in twins:
            t.close()


@pytest.mark.parametrize("mode", ["sync", "dev"])
@pytest.mark.parametrize("gf", [0, 1])
def test_sensor_table_on_top_of_own_values(pkg, synth, gf, mode):
    """A sequence with a 3-sensor table and its own values: the twin is lmot_set_sensors + lmot_batch on a context created with those
    values (the table's mounting values replace the four of p).  Catches the fold of the sensor values into the frame entries."""
    from test_seq_rig_gpu import set_seq_rig
    rig = RIG[:3]
    layout = [rig, None, None, None, None, None]                       # 3 + 5 = 8 frames
    vals = [SPARSE, None, OT0, COMPAT, None, {**ALL_MOVED, **LITERALS}]
    S = len(layout)
    seqs = [_RigSeq(synth, k, r, n_ticks=N_TICKS) for k, r in enumerate(layout)]
    ctx = _seq_ctx(pkg, S, gf)
    twins = [_Twin(pkg, _twin_params(pkg, v, gf), r) for v, r in zip(vals, layout)]
    try:
        for k, (v, r) in enumerate(zip(vals, layout)):
            if r:
                set_seq_rig(ctx, k, r)
            if v:
                ctx.seq_set_detect_params(k, **v)
        _run(ctx, seqs, lambda f: layout, N_TICKS, mode, twins)
        _same_tables(ctx, twins, (gf, mode))
    finally:
        ctx.close()
        for t in twins:
            t.close()


@pytest.mark.parametrize("name", ["ot0", "sparse", "all_moved"])
def test_against_the_reference(pkg, synth, ref_dt, name):
    """Sequence 3 of an S = 8 tick with its own values: per-frame counts and boxes bit-exact against the reference's groundRemove /
    componentClustering / boxFitting with its globals set to those values (the two literals included), and the tracker on those boxes
    against the reference's immUkfJpdaf: identical trackManage, static and visible flags and table integers, targets and UKF states
    within 1e-4 relative.  Catches a value the kernels read from the wrong place, or a twin context that is itself wrong (this is the
    anchor of the twin tests)."""
    vals = {"ot0": OT0, "sparse": SPARSE, "all_moved": {**ALL_MOVED, **LITERALS}}[name]
    S, K, T = 8, 3, 20
    seqs = [_RigSeq(synth, k, None, n_ticks=T, n_objects=40) for k in range(S)]
    ctx = _seq_ctx(pkg, S)
    ref = ref_dt
    ref.tracker_reset()
    n_boxes = 0
    try:
        ctx.seq_set_detect_params(K, **vals)
        for f in range(T):
            got = ctx.seq([s.frames[f][0] for s in seqs], [s.ts(f) for s in seqs])
            pts = seqs[K].frames[f][0]
            with ref.detect_params(vals):
                e, g = ref.ground_remove(pts)
                grid, nc = ref.component_clustering(e)
                boxes, _ = ref.box_fitting(e, grid, nc)
            boxes = np.asarray(boxes, f32).reshape(-1, 8, 3)
            r = got[K]
            assert (r["n_elevated"], r["n_ground"], r["num_cluster"], len(r["boxes"])) == (len(e), len(g), nc, len(boxes)), (name, f)
            assert np.array_equal(r["boxes"].view(np.uint32), boxes.view(np.uint32)), (name, f)
            n_boxes += len(boxes)
            a = ref.tracker_step(boxes, seqs[K].ts(f))
            for key in ("track_manage", "is_static", "is_vis"):
                assert np.array_equal(r[key], a[key]), (name, f, key)
            np.testing.assert_allclose(r["targets"], a["targets"], rtol=1e-4, atol=1e-4)
        assert n_boxes > 0, name
        da, db = ref.tracker_dump(), ctx.seq_tracker_dump(K)
        assert da.shape == db.shape and np.array_equal(da[:, INTS], db[:, INTS]), name
        ok = _pd_tracks(da)
        err = _rel_err(da[ok][:, STATE], db[ok][:, STATE])
        assert err.size == 0 or err.max() < TOL, (name, float(err.max()))
    finally:
        ctx.close()


def _boundary_cloud(r_min, r_max, rng, n=4000):
    """points within 1e-6 m .. 1e-3 m of every bin boundary of [r_min, r_max] (and of the window's ends), and within 1e-7 .. 1e-4 rad
    of every channel boundary"""
    span = f32(r_max) - f32(r_min)
    d_b = [float(r_min) + k * float(span) / 120 for k in range(121)]
    eps = np.array([1e-6, 3e-6, 1e-5, 1e-4, 1e-3])
    rs = np.concatenate([np.add.outer(d_b, eps).ravel(), np.add.outer(d_b, -eps).ravel()])
    ang = rng.uniform(-np.pi, np.pi, len(rs))
    a_c = [-np.pi + j * 2 * np.pi / 80 for j in range(80)]
    ea = np.array([1e-7, 3e-7, 1e-6, 1e-4])
    angs = np.concatenate([np.add.outer(a_c, ea).ravel(), np.add.outer(a_c, -ea).ravel()])
    rr = rng.uniform(r_min, r_max, len(angs))
    R = np.concatenate([rs, rr]); A = np.concatenate([ang, angs])
    z = rng.uniform(-2.5, 0.5, len(R))
    return np.stack([R * np.cos(A), R * np.sin(A), z], 1).astype(f32)


@pytest.mark.parametrize("window", [(3.4, 120.0), (5.0, 60.0), (48.0, 60.0), (0.0, 30.0)])
def test_boundaries_under_a_moved_range(pkg, ref_dt, window):
    """Cell indices and labels of boundary-hugging points, bit-exact against the reference's cell_index with rMin / rMax set, for a
    context created with that window -- (48, 60) is the shortest window accepted for r_max 60 (r_max / 5)."""
    r_min, r_max = window
    assert (f32(r_max) - f32(r_min)) >= f32(r_max) / 5
    p = pkg.default_params()
    p.r_min, p.r_max = r_min, r_max
    lm = pkg.Lmot(p)
    rng = np.random.default_rng(int(r_max * 10 + r_min))
    try:
        with ref_dt.detect_params(dict(r_min=r_min, r_max=r_max)):
            for _ in range(2):
                _check_frame(lm, ref_dt, _boundary_cloud(r_min, r_max, rng))
    finally:
        lm.close()


def test_change_in_flight_open_and_reset(pkg, synth):
    """Ticks in flight keep their values, a change applies from the next submitted tick (detection outputs against twins created with
    the old and the new values); lmot_seq_tracker_reset keeps the values, lmot_seq_open resets them; tracking-only ticks ignore them."""
    import torch
    S = 2
    seqs = [_RigSeq(synth, k, None, n_ticks=12) for k in range(S)]
    ctx = _seq_ctx(pkg, S)
    det = {name: pkg.Lmot(_twin_params(pkg, v)) for name, v in (("none", None), ("sparse", SPARSE), ("ot0", OT0))}
    try:
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)
        keep, want = [], []
        ctx.seq_set_detect_params(1, **SPARSE)
        for f in range(12):
            if f == 6:
                ctx.seq_set_detect_params(1, **OT0)            # ticks 0..5 are still in flight with SPARSE
            with torch.cuda.stream(stream):
                dev = [torch.from_numpy(np.ascontiguousarray(s.frames[f][0])).cuda() for s in seqs]
                keep.append(dev)
                ctx.seq_dev([(t.data_ptr(), len(t)) for t in dev], [s.ts(f) for s in seqs])
            want.append([det["none"].frame(seqs[0].frames[f][0], seqs[0].ts(f)),
                         det["sparse" if f < 6 else "ot0"].frame(seqs[1].frames[f][0], seqs[1].ts(f))])
        for f in range(12):
            got = ctx.seq_collect()
            for k in range(S):
                w = want[f][k]
                assert (got[k]["n_elevated"], got[k]["n_ground"], got[k]["num_cluster"]) == (w["n_elevated"], w["n_ground"], w["num_cluster"])
                assert np.array_equal(got[k]["boxes"].view(np.uint32), w["boxes"].view(np.uint32)), (f, k)
        ctx.set_stream(None)
        kept = ctx.seq_get_detect_params(1)
        assert kept["roi_m"] == OT0["roi_m"] and kept["min_cluster_points"] == OT0["min_cluster_points"]
        ctx.seq_tracker_reset(1)
        assert ctx.seq_get_detect_params(1) == kept
        # a tracking-only tick does not read them: the same outputs as a set without them
        other = _seq_ctx(pkg, S)
        try:
            ctx.seq_tracker_reset(0)
            lists = [det["none"].frame(seqs[k].frames[0][0], 1e6)["boxes"] for k in range(S)]
            for t in range(3):
                a = ctx.seq_track(lists, [1e6 + 1e5 * t] * S)
                b = other.seq_track(lists, [1e6 + 1e5 * t] * S)
                for k in range(S):
                    for key in ("targets", "track_manage", "vis_bb"):
                        assert np.array_equal(_bits(a[k][key]), _bits(b[k][key])), (t, k, key)
        finally:
            other.close()
        ctx.seq_tracker_load(1, ctx.seq_tracker_dump(0), 1, seqs[0].ts(11))
        assert ctx.seq_get_detect_params(1) == kept
        ctx.seq_open(S, ring=4)
        assert ctx.seq_get_detect_params(1) == pkg.default_detect_params(ctx.params)
    finally:
        ctx.close()
        for c in det.values():
            c.close()


def test_validation(pkg):
    """Every rejection returns LMOT_ERR_INVALID and leaves every sequence's values as they were."""
    ctx = pkg.Lmot(_params(pkg))
    lib = pkg.load_library()
    try:
        d = pkg.DetectParams()
        lib.lmot_default_detect_params(None, C.byref(d))
        assert lib.lmot_seq_set_detect_params(ctx.h, 0, C.byref(d)) == pkg.ERR_INVALID        # no open set
        ctx.seq_open(3, ring=2)
        ctx.seq_set_detect_params(1, **SPARSE)
        before = [ctx.seq_get_detect_params(k) for k in range(3)]
        bad = [dict(r_max=float("nan")), dict(t_len_max=float("inf")), dict(ground_tolerance=float("nan")), dict(r_min=-0.1),
               dict(r_min=50.0, r_max=50.0), dict(r_min=60.0, r_max=50.0), dict(r_min=48.1, r_max=60.0), dict(roi_m=0.0),
               dict(roi_m=-5.0), dict(rule_filter=2), dict(rule_filter=-1), dict(ram_points=0), dict(ram_points=pkg.MAX_RAM_POINTS + 1)]
        for fields in bad:
            for k in (0, 1):
                with pytest.raises(pkg.LmotError) as e:
                    ctx.seq_set_detect_params(k, **fields)
                assert e.value.status == pkg.ERR_INVALID, fields
        for k in (-1, 3):
            assert lib.lmot_seq_set_detect_params(ctx.h, k, C.byref(d)) == pkg.ERR_INVALID
            assert lib.lmot_seq_get_detect_params(ctx.h, k, C.byref(d)) == pkg.ERR_INVALID
        assert [ctx.seq_get_detect_params(k) for k in range(3)] == before
        ctx.seq_set_detect_params(2, ram_points=pkg.MAX_RAM_POINTS, r_min=48.0, r_max=60.0)     # at the bounds: accepted
        ctx.seq_set_detect_params(1)                                                            # NULL: lmot_params again
        assert ctx.seq_get_detect_params(1) == pkg.default_detect_params(ctx.params)
    finally:
        ctx.close()
